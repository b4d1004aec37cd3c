"""Generate tests/golden/mag_gcrd.pt by running the REFERENCE's own ``train()`` of mag_pyg/gnn_kd_and_aux.py (:174-268) with
``--training nce`` for one step: the RGCN student (2 layers) and its projection head learning from an RGCN teacher (3 layers,
eval) through the teacher's projection head and ``kd_criterion + beta * nce_criterion(...)[2]`` (criterion.py:129-149), one
Adam over the model and both heads (:424-441).

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_mag_gcrd.py   (not run by the suite)

The stubs, the designed batch and the model states are make_golden_mag_lsp.py's (the same torch seed).  The reference's
forward hard-codes F.dropout(p=0.5); as there, the module's ``F`` multiplies by a recorded keep mask (``keep``), but the mask
is the one the engine itself draws at trainer seed 0, step 0 (oracle.dropout.mask, the CPU restatement of its Philox keep
decisions, in batch node order), so that an RGCNTrainer(seed=0) step can be compared with the fixture directly.  The heads are built as the reference's main() builds them, nn.Sequential(Linear, BatchNorm1d, ReLU), with the
teacher's Linear at the teacher's hidden width (12 here, 512 in the scripts), and start from
``oracle.ppi_gcrd.seeded_heads`` (seed 303), so no head state is stored.  Hyper-parameters are the MAG script's
(scripts/run_kd_and_aux.sh: beta 0.1, nce_T 0.075; lr 0.005) with proj_dim 64.  Cases:

    main/all       train papers {0, 1, 2, 4, 5, 7}, max_samples 24576 >= 6: every row, no draw
    main/sampled   the same rows, max_samples 4: numpy is seeded before the step and the draw np.random.choice makes
                   inside nce_criterion is recorded by wrapping it
    no_train       no train row: KD, loss_cls and the InfoNCE are means over nothing (NaN); every gradient is zero, the
                   heads' running statistics stay and num_batches_tracked advances.  train()'s final average divides by
                   zero, so the ZeroDivisionError it raises after the step is caught, and the losses are recorded from
                   kd_criterion's and nce_criterion's returns

Recorded per case: the three losses, every gradient of the model and of both heads, every parameter after Adam, and the
heads' running statistics and num_batches_tracked."""
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

from oracle import dropout as odrop, ppi_gcrd as opg  # noqa: E402

BETA, NCE_T, PROJ, LR, ALPHA, KD_T = 0.1, 0.075, 64, 0.005, 0.9, 4.0
SEEDS = dict(heads=303, numpy=11, dropout=0)
CASES = {"main/all": ("main", 24576), "main/sampled": ("main", 4), "no_train": ("no_train", 24576)}


def heads(hidden, teacher_hidden):
    """The reference main()'s heads (teacher Linear at the teacher's width), loaded from oracle.ppi_gcrd.seeded_heads."""
    s_sd, t_sd = opg.seeded_heads(hidden, teacher_hidden, PROJ, SEEDS["heads"])
    sp = torch.nn.Sequential(torch.nn.Linear(hidden, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    tp = torch.nn.Sequential(torch.nn.Linear(teacher_hidden, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    sp.load_state_dict(s_sd)
    tp.load_state_dict(t_sd)
    return sp, tp


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_mag_stubs()
    sys.path.insert(0, str(mg.REF / "mag_pyg"))
    spec = importlib.util.spec_from_file_location("mag_kd", mg.REF / "mag_pyg" / "gnn_kd_and_aux.py")
    mag = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mag)

    G = mgl.designed_graph()
    G["train_mask"] = {"main": G["train_mask"]["main"], "no_train": torch.zeros_like(G["train_mask"]["main"])}
    G["keep"] = torch.from_numpy(odrop.mask(G["node_type"].numel(), mgl.H, 0.5, SEEDS["dropout"], 0))
    keep = {"mask": G["keep"]}

    class _F:
        def __getattr__(self, k):
            return getattr(torch.nn.functional, k)

        @staticmethod
        def dropout(x, p=0.5, training=True):
            return x * keep["mask"].to(x.dtype) / (1 - p) if training else x

    mag.F = _F()
    # the losses of the step as the criteria return them, and the rows np.random.choice draws inside nce_criterion
    seen = {}
    kd, nce, choice = mag.kd_criterion, mag.nce_criterion, np.random.choice

    def kd_rec(*a, **k):
        seen["kd"] = r = kd(*a, **k)
        return r

    def nce_rec(*a, **k):
        seen["nce"] = r = nce(*a, **k)
        return r

    def choice_rec(*a, **k):
        seen["sample"] = r = choice(*a, **k)
        return r

    mag.kd_criterion, mag.nce_criterion, np.random.choice = kd_rec, nce_rec, choice_rec

    F_IN, H, C, H_T, NN = mgl.F_IN, mgl.H, mgl.C, mgl.H_T, mgl.NUM_NODES
    torch.manual_seed(7)                                                   # make_golden_mag_lsp's model states
    student0 = mag.RGCN(F_IN, H, C, 2, 0.5, NN, [0], len(G["relations"]))
    teacher = mag.RGCN(F_IN, H_T, C, 3, 0.5, NN, [0], len(G["relations"]))
    teacher.eval()
    out = dict(G, num_nodes=NN, in_channels=F_IN, hidden=H, teacher_hidden=H_T, out_channels=C, beta=BETA, nce_T=NCE_T,
               proj_dim=PROJ, lr=LR, alpha=ALPHA, kd_T=KD_T, seeds=SEEDS,
               student_state={k: v.detach().clone() for k, v in student0.state_dict().items()},
               teacher_state={k: v.detach().clone() for k, v in teacher.state_dict().items()}, cases={})
    for name, (mask, max_samples) in CASES.items():
        m = mag.RGCN(F_IN, H, C, 2, 0.5, NN, [0], len(G["relations"]))
        m.load_state_dict(out["student_state"])
        sp, tp = heads(H, H_T)
        opt = torch.optim.Adam([{"params": m.parameters(), "lr": LR}, {"params": sp.parameters(), "lr": LR},
                                {"params": tp.parameters(), "lr": LR}])
        b = mgl.Batch(edge_index=G["edge_index"], edge_attr=G["edge_type"], node_type=G["node_type"],
                      local_node_idx=G["local_node_idx"], y=G["y"], train_mask=G["train_mask"][mask])
        args = argparse.Namespace(training="nce", beta=BETA, nce_T=NCE_T, max_samples=max_samples, alpha=ALPHA, kd_T=KD_T,
                                  num_steps=1, batch_size=1)
        seen.clear()
        np.random.seed(SEEDS["numpy"])
        try:
            loss, loss_cls, loss_aux = mag.train(m, [b], {0: G["x"]}, opt, args, "cpu", teacher, sp, tp)
        except ZeroDivisionError:
            assert mask == "no_train"
            loss_aux = float(seen["nce"][2].detach())
            loss, loss_cls = float(seen["kd"][0].detach()) + BETA * loss_aux, float(seen["kd"][1].detach())
        sample = torch.from_numpy(seen["sample"]).to(torch.int64) if "sample" in seen else None
        groups = dict(model=m, sproj=sp, tproj=tp)
        out["cases"][name] = dict(
            max_samples=max_samples, sample=sample,
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={g: {k: p.grad.detach().clone() for k, p in mod.named_parameters()} for g, mod in groups.items()},
            after={g: {k: p.detach().clone() for k, p in mod.named_parameters()} for g, mod in groups.items()},
            running={g: {k: v.clone() for k, v in mod.state_dict().items() if "running" in k or "num_batches" in k}
                     for g, mod in (("sproj", sp), ("tproj", tp))})
    torch.save(out, mg.OUT / "mag_gcrd.pt")
    print("wrote mag_gcrd.pt", (mg.OUT / "mag_gcrd.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
