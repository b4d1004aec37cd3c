"""Generate tests/golden/ppi_gsp.pt by running the REFERENCE's own ``train()`` of ppi_pyg/gnn.py (:185-284) with
``--training gpw`` for one step: ``StudentNet`` learning from ``TeacherNet``'s ``out_feat`` through
``gpw_criterion(out, labels, model.out_feat, teacher_model.out_feat, kernel, beta, max_samples)`` (criterion.py:54-89:
BCE + beta * GSP, no projection heads).

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_ppi_gsp.py   (not run by the suite)

The stubs, the stand-in GATConv and the designed graph are make_golden_ppi.py's (n = 300: a hub, node 299 with no edge, the
self-loop 5 -> 5 and the duplicate edge 7 -> 8).  Both models start from ``oracle.ppi.seeded_state`` (student seed 101,
teacher seed 202), so no state is stored.  The teacher's 1024-wide out_feat is that of ppi_lsp.pt (the same seeded
TeacherNet on the same graph): the generator checks that its fingerprint equals the one ppi_lsp.pt records, and does not
store it again.  Cases, all at beta 100 and Adam lr 0.005:

    cosine, poly, l2, rbf   max_samples 8192 >= n: every row, no draw
    cosine_s128             cosine at max_samples 128: numpy is seeded before the step and the draw np.random.choice
                            makes inside gpw_criterion is recorded by repeating it after an identical seeding

(On this graph the rbf similarities of distinct rows underflow to about 1e-20 on both sides, so the rbf case pins the
classification term and the diagonal rule more than the GSP term; the sampled case therefore uses cosine.)

Recorded per case: the three losses train() returns, every gradient (``oracle.ppi.fingerprint`` with FP_SAMPLES sampled
entries) and, for the cases with every row, every parameter after the optimizer step at the ``after_entries`` entries
(the sampled case differs from them only in the loss's rows, not in the optimizer).  Every tensor of the file is a
view of one buffer per dtype (torch.save then writes each buffer once), which keeps the file under 0.5 MB."""
from __future__ import annotations

import argparse
import importlib
import sys
from pathlib import Path

import numpy as np
import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; the sklearn stub has no __spec__ to scan)

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402
import make_golden_ppi as mgp  # noqa: E402
from make_golden_ppi_lsp import Batch, after_entries  # noqa: E402

from oracle import ppi as oppi  # noqa: E402

BETA, LR = 100.0, 0.005
SEEDS = dict(student=101, teacher=202, numpy=11)
CASES = dict(cosine=("cosine", 8192), poly=("poly", 8192), l2=("l2", 8192), rbf=("rbf", 8192), cosine_s128=("cosine", 128))
FP_SAMPLES = 128


def consolidated(obj):
    """obj with every tensor replaced by a view of one flat buffer per dtype (same values, dtypes and shapes)."""
    leaves = []

    def walk(o):
        if isinstance(o, torch.Tensor):
            leaves.append(o)
        elif isinstance(o, dict):
            for v in o.values():
                walk(v)
    walk(obj)
    flat = {dt: torch.cat([t.reshape(-1) for t in leaves if t.dtype == dt]) for dt in {t.dtype for t in leaves}}
    offs = {dt: 0 for dt in flat}

    def rebuild(o):
        if isinstance(o, torch.Tensor):
            o0 = offs[o.dtype]
            offs[o.dtype] += o.numel()
            return flat[o.dtype][o0:o0 + o.numel()].view(o.shape)
        return {k: rebuild(v) for k, v in o.items()} if isinstance(o, dict) else o
    return rebuild(obj)


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mgp.install_stubs()
    sys.path.insert(0, str(mg.REF / "ppi_pyg"))
    gnn = importlib.import_module("gnn")
    ei = mgp.designed_edges()
    g = torch.Generator().manual_seed(41)                                    # make_golden_ppi's draws: the same x and y
    x = torch.randn(mgp.N, mgp.F_IN, generator=g)
    y = (torch.rand(mgp.N, mgp.C, generator=g) < 0.3).float()
    teacher = gnn.TeacherNet(mgp.F_IN, mgp.C)
    teacher.load_state_dict(oppi.seeded_state(oppi.layers_of("teacher", mgp.C), mgp.F_IN, SEEDS["teacher"]))
    teacher.eval()
    with torch.no_grad():
        teacher(x, ei)
    lsp = torch.load(mg.OUT / "ppi_lsp.pt")
    for k, v in oppi.fingerprint(teacher.out_feat).items():
        assert torch.equal(v, lsp["teacher_feat_fp"][k]), "the teacher features differ from ppi_lsp.pt's"
    out = dict(edge_index=ei.to(torch.int32), x=x, y=y.to(torch.uint8),
               in_channels=mgp.F_IN, out_channels=mgp.C, seeds=SEEDS, beta=BETA, lr=LR, fp_samples=FP_SAMPLES, cases={})
    for name, (kernel, max_samples) in CASES.items():
        m = gnn.StudentNet(mgp.F_IN, mgp.C)
        m.load_state_dict(oppi.seeded_state(oppi.layers_of("student", mgp.C), mgp.F_IN, SEEDS["student"]))
        opt = torch.optim.Adam(m.parameters(), lr=LR)
        args = argparse.Namespace(training="gpw", kernel=kernel, beta=BETA, max_samples=max_samples)
        np.random.seed(SEEDS["numpy"])
        loss, loss_cls, loss_aux = gnn.train(m, teacher, None, [Batch(x, y, ei)], opt, args, "cpu")
        np.random.seed(SEEDS["numpy"])
        sample = (torch.from_numpy(np.random.choice(mgp.N, max_samples, replace=False)).to(torch.int64)
                  if max_samples < mgp.N else None)
        out["cases"][name] = dict(
            kernel=kernel, max_samples=max_samples, sample=sample,
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={k: oppi.fingerprint(p.grad, n_sample=FP_SAMPLES) for k, p in m.named_parameters()})
        if sample is None:
            out["cases"][name]["after"] = {k: p.detach().reshape(-1)[after_entries(p.numel())].clone()
                                           for k, p in m.named_parameters()}
    torch.save(consolidated(out), mg.OUT / "ppi_gsp.pt")
    print("wrote ppi_gsp.pt", (mg.OUT / "ppi_gsp.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
