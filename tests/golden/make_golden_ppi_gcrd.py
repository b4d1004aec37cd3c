"""Generate tests/golden/ppi_gcrd.pt by running the REFERENCE's own ``train()`` of ppi_pyg/gnn.py (:185-284) with
``--training nce`` for one step: ``StudentNet`` and its projection head learning from ``TeacherNet``'s ``out_feat`` through
the teacher's projection head (gnn.py:355-372) and ``nce_criterion`` (criterion.py:126-146): BCE + beta * InfoNCE, one Adam
over the model and both heads.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_ppi_gcrd.py   (not run by the suite)

The stubs, the stand-in GATConv and the designed graph are make_golden_ppi.py's (n = 300: a hub, a node with no edge, a
self-loop and a duplicate edge).  Both models start from ``oracle.ppi.seeded_state`` (student seed 101, teacher seed 202)
and both heads from ``oracle.ppi_gcrd.seeded_heads`` (seed 303: the draws of gcrd.ProjectionHeads.reset_parameters), so no
state is stored; the teacher's 1024-wide out_feat is stored as its ``oracle.ppi.fingerprint`` only.  Hyper-parameters are
the scripts' (scripts/run.sh: beta 0.1, nce_T 0.075, proj_dim 256, Adam lr 0.005).  Two cases:

    full   max_samples 16384 >= n: every row, no draw
    s128   max_samples 128: numpy is seeded before the step and the draw np.random.choice makes inside nce_criterion is
           recorded by repeating it after an identical seeding

Recorded per case: the three losses train() returns, every gradient of the model and of both heads
(``oracle.ppi.fingerprint``), every parameter after the optimizer step at the ``after_entries`` entries, and the heads'
running statistics and num_batches_tracked."""
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

from oracle import ppi as oppi, ppi_gcrd as opg  # noqa: E402

BETA, NCE_T, PROJ, LR = 0.1, 0.075, 256, 0.005
SEEDS = dict(student=101, teacher=202, heads=303, numpy=11)
CASES = dict(full=16384, s128=128)


def heads():
    s_sd, t_sd = opg.seeded_heads(136, 1024, PROJ, SEEDS["heads"])
    sp = torch.nn.Sequential(torch.nn.Linear(136, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    tp = torch.nn.Sequential(torch.nn.Linear(1024, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    sp.load_state_dict(s_sd)
    tp.load_state_dict(t_sd)
    return sp, tp


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
    out = dict(edge_index=ei.to(torch.int32), x=x, y=y.to(torch.uint8), teacher_feat_fp=oppi.fingerprint(teacher.out_feat),
               in_channels=mgp.F_IN, out_channels=mgp.C, seeds=SEEDS, beta=BETA, nce_T=NCE_T, proj_dim=PROJ, lr=LR, cases={})
    for name, max_samples in CASES.items():
        m = gnn.StudentNet(mgp.F_IN, mgp.C)
        m.load_state_dict(oppi.seeded_state(oppi.layers_of("student", mgp.C), mgp.F_IN, SEEDS["student"]))
        sp, tp = heads()
        opt = torch.optim.Adam([{"params": m.parameters(), "lr": LR}, {"params": sp.parameters(), "lr": LR},
                                {"params": tp.parameters(), "lr": LR}])
        args = argparse.Namespace(training="nce", beta=BETA, nce_T=NCE_T, max_samples=max_samples)
        np.random.seed(SEEDS["numpy"])
        loss, loss_cls, loss_aux = gnn.train(m, teacher, None, [Batch(x, y, ei)], opt, args, "cpu", sp, tp)
        np.random.seed(SEEDS["numpy"])
        sample = (torch.from_numpy(np.random.choice(mgp.N, max_samples, replace=False)).to(torch.int64)
                  if max_samples < mgp.N else None)
        groups = dict(model=m, sproj=sp, tproj=tp)
        out["cases"][name] = dict(
            max_samples=max_samples, sample=sample,
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={gname: {k: oppi.fingerprint(p.grad) for k, p in mod.named_parameters()} for gname, mod in groups.items()},
            after={gname: {k: p.detach().reshape(-1)[after_entries(p.numel())].clone() for k, p in mod.named_parameters()}
                   for gname, mod in groups.items()},
            running={gname: {k: v.clone() for k, v in mod.state_dict().items() if k.startswith("1.") and "running" in k
                             or "num_batches" in k}
                     for gname, mod in (("sproj", sp), ("tproj", tp))})
    torch.save(out, mg.OUT / "ppi_gcrd.pt")
    print("wrote ppi_gcrd.pt", (mg.OUT / "ppi_gcrd.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
