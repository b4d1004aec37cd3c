"""Generate tests/golden/mag_gsp.pt by running the REFERENCE's own ``train()`` of mag_pyg/gnn_kd_and_aux.py (:174-268) with
``--training gpw`` for one step: the RGCN student (2 layers) learning from an RGCN teacher (3 layers, eval) through
``kd_criterion + beta * gpw_criterion(out, labels, model.out_feat[mask], teacher_model.out_feat[mask], kernel, beta,
max_samples)[2]`` (criterion.py:57-92), no projection heads, one Adam over the model.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_mag_gsp.py   (not run by the suite)

The stubs, the designed batch and the model states are make_golden_mag_lsp.py's (the same torch seed).  The reference's
forward hard-codes F.dropout(p=0.5); as there, the module's ``F`` multiplies by a recorded keep mask (``keep``), but the mask
is the one the engine itself draws at trainer seed 0, step 0 (oracle.dropout.mask, in batch node order), as in
make_golden_mag_gcrd.py, so that an RGCNTrainer(seed=0) step can be compared with the fixture directly.  Hyper-parameters
are the MAG script's (scripts/run_kd_and_aux.sh: gpw with beta 1; lr 0.005).  Cases:

    main/<kernel>   cosine, poly, l2 and rbf: train papers {0, 1, 2, 4, 5, 7}, max_samples 24576 >= 6, every row, no draw
    main/sampled    cosine on the same rows with max_samples 4: numpy is seeded before the step and the draw
                    np.random.choice makes inside gpw_criterion is recorded by wrapping it
    no_train        poly with no train row: KD, loss_cls and the mse over no pair are NaN and every gradient is zero.
                    train()'s final average divides by zero, so the ZeroDivisionError it raises after the step is caught,
                    and the losses are recorded from kd_criterion's and gpw_criterion's returns
    one_train       l2 with paper 4 the only train row: S = 1, both 1 x 1 similarities are 0, so loss_aux is 0.  train()
                    passes its labels as data.y[train_mask].squeeze(), a 0-d tensor for one row, which cross_entropy
                    refuses; the wrappers of kd_criterion and gpw_criterion pass that label as [1], so the step runs

Recorded per case: the kernel, max_samples, the sample (or None), the three losses, every gradient and every parameter
after Adam."""
from __future__ import annotations

import argparse
import importlib.util
import sys
from pathlib import Path

import numpy as np
import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; the stub modules have no __spec__ to scan)

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402
import make_golden_mag_lsp as mgl  # noqa: E402

from oracle import dropout as odrop  # noqa: E402

BETA, LR, ALPHA, KD_T = 1.0, 0.005, 0.9, 4.0
SEEDS = dict(numpy=11, dropout=0)
CASES = {"main/cosine": ("main", "cosine", 24576), "main/poly": ("main", "poly", 24576), "main/l2": ("main", "l2", 24576),
         "main/rbf": ("main", "rbf", 24576), "main/sampled": ("main", "cosine", 4),
         "no_train": ("no_train", "poly", 24576), "one_train": ("one_train", "l2", 24576)}
ONE_TRAIN = 4


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_mag_stubs()
    sys.path.insert(0, str(mg.REF / "mag_pyg"))
    spec = importlib.util.spec_from_file_location("mag_kd", mg.REF / "mag_pyg" / "gnn_kd_and_aux.py")
    mag = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mag)

    G = mgl.designed_graph()
    main_mask = G["train_mask"]["main"]
    one = torch.zeros_like(main_mask)
    one[ONE_TRAIN] = True
    assert bool(main_mask[ONE_TRAIN])
    G["train_mask"] = {"main": main_mask, "no_train": torch.zeros_like(main_mask), "one_train": one}
    G["keep"] = torch.from_numpy(odrop.mask(G["node_type"].numel(), mgl.H, 0.5, SEEDS["dropout"], 0))
    keep = {"mask": G["keep"]}

    class _F:
        def __getattr__(self, k):
            return getattr(torch.nn.functional, k)

        @staticmethod
        def dropout(x, p=0.5, training=True):
            return x * keep["mask"].to(x.dtype) / (1 - p) if training else x

    mag.F = _F()
    # the losses of the step as the criteria return them, and the rows np.random.choice draws inside gpw_criterion
    seen = {}
    kd, gpw, choice = mag.kd_criterion, mag.gpw_criterion, np.random.choice

    def labels_1d(a):
        # train() passes data.y[train_mask].squeeze(): with one train row a 0-d label, which cross_entropy refuses
        return (a[0], a[1].view(1)) + tuple(a[2:]) if a[1].dim() == 0 else a

    def kd_rec(*a, **k):
        seen["kd"] = r = kd(*labels_1d(a), **k)
        return r

    def gpw_rec(*a, **k):
        seen["gpw"] = r = gpw(*labels_1d(a), **k)
        return r

    def choice_rec(*a, **k):
        seen["sample"] = r = choice(*a, **k)
        return r

    mag.kd_criterion, mag.gpw_criterion, np.random.choice = kd_rec, gpw_rec, choice_rec

    F_IN, H, C, H_T, NN = mgl.F_IN, mgl.H, mgl.C, mgl.H_T, mgl.NUM_NODES
    torch.manual_seed(7)                                                   # make_golden_mag_lsp's model states
    student0 = mag.RGCN(F_IN, H, C, 2, 0.5, NN, [0], len(G["relations"]))
    teacher = mag.RGCN(F_IN, H_T, C, 3, 0.5, NN, [0], len(G["relations"]))
    teacher.eval()
    out = dict(G, num_nodes=NN, in_channels=F_IN, hidden=H, teacher_hidden=H_T, out_channels=C, beta=BETA, lr=LR,
               alpha=ALPHA, kd_T=KD_T, seeds=SEEDS,
               student_state={k: v.detach().clone() for k, v in student0.state_dict().items()},
               teacher_state={k: v.detach().clone() for k, v in teacher.state_dict().items()}, cases={})
    for name, (mask, kernel, max_samples) in CASES.items():
        m = mag.RGCN(F_IN, H, C, 2, 0.5, NN, [0], len(G["relations"]))
        m.load_state_dict(out["student_state"])
        opt = torch.optim.Adam(m.parameters(), lr=LR)
        b = mgl.Batch(edge_index=G["edge_index"], edge_attr=G["edge_type"], node_type=G["node_type"],
                      local_node_idx=G["local_node_idx"], y=G["y"], train_mask=G["train_mask"][mask])
        args = argparse.Namespace(training="gpw", kernel=kernel, beta=BETA, max_samples=max_samples, alpha=ALPHA, kd_T=KD_T,
                                  num_steps=1, batch_size=1)
        seen.clear()
        np.random.seed(SEEDS["numpy"])
        try:
            loss, loss_cls, loss_aux = mag.train(m, [b], {0: G["x"]}, opt, args, "cpu", teacher)
        except ZeroDivisionError:
            assert mask == "no_train"
            loss_aux = float(seen["gpw"][2].detach())
            loss, loss_cls = float(seen["kd"][0].detach()) + BETA * loss_aux, float(seen["kd"][1].detach())
        sample = torch.from_numpy(seen["sample"]).to(torch.int64) if "sample" in seen else None
        out["cases"][name] = dict(
            mask=mask, kernel=kernel, max_samples=max_samples, sample=sample,
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={k: (p.grad if p.grad is not None else torch.zeros_like(p)).detach().clone()
                   for k, p in m.named_parameters()},
            after={k: p.detach().clone() for k, p in m.named_parameters()})
    torch.save(out, mg.OUT / "mag_gsp.pt")
    print("wrote mag_gsp.pt", (mg.OUT / "mag_gsp.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
