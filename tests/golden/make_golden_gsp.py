"""Generate tests/golden/gsp_arxiv.pt by running the REFERENCE's own ``train()`` with ``--training gpw`` for one step:
arxiv_pyg/gnn.py (CE + beta * gpw) and arxiv_pyg/gnn_kd_and_aux.py (KD + beta * gpw), for the GCN and SAGE students, with the
projection heads and the three-group Adam of gnn_kd_and_aux.py:275-297, on the stand-in convs of make_golden.py.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_gsp.py   (not run by the suite)

The problem is make_golden_gcrd.py's: small graph of make_golden.small_graph (240 nodes), 16 input features, hidden 32,
8 classes, 3 layers, dropout 0, a 90-wide teacher feature matrix (not a multiple of 4, like the real 750), proj_dim 64,
max_samples 64 of the 150 training rows.  Cases: each script and student with the scripts' cosine at beta 10
(run_kd_and_aux.sh) or the argparse default rbf at beta 0.5, and l2 once.  numpy is seeded as the reference's seed() seeds it
before the step, and the draw np.random.choice makes inside gpw_criterion is recorded by repeating it between two identical
seedings.  Recorded per case: initial states of the model and both heads, the draw, the three losses, every gradient
(p.grad survives optimizer.step()) and the state after the step (parameters and running statistics)."""
from __future__ import annotations

import argparse
import importlib
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402

N_IN, HID, C, L, F_T, PROJ, S = 16, 32, 8, 3, 90, 64, 64
# case name -> (script, student, kernel, beta)
CASES = {"gnn_gcn_cosine": ("gnn", "gcn", "cosine", 10.0), "gnn_sage_rbf": ("gnn", "sage", "rbf", 0.5),
         "kd_and_aux_gcn_rbf": ("kd_and_aux", "gcn", "rbf", 0.5), "kd_and_aux_sage_cosine": ("kd_and_aux", "sage", "cosine", 10.0),
         "kd_and_aux_gcn_l2": ("kd_and_aux", "gcn", "l2", 0.5)}


def state(m):
    return {k: v.detach().clone() for k, v in m.state_dict().items()}


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_stubs()
    if "torch.utils.tensorboard" not in sys.modules:
        try:
            importlib.import_module("torch.utils.tensorboard")
        except Exception:                                    # the scripts only name SummaryWriter
            import types
            tb = types.ModuleType("torch.utils.tensorboard")
            tb.SummaryWriter = None
            sys.modules["torch.utils.tensorboard"] = tb
    sys.path.insert(0, str(mg.REF / "arxiv_pyg"))
    scripts = {"gnn": importlib.import_module("gnn"), "kd_and_aux": importlib.import_module("gnn_kd_and_aux")}
    n = 240
    ei, r, c, rowptr = mg.small_graph(n)
    g = torch.Generator().manual_seed(31)
    x = torch.randn(n, N_IN, generator=g)
    y = torch.randint(0, C, (n,), generator=g)
    train_idx = torch.randperm(n, generator=g)[:150].sort().values
    t_feat = torch.randn(n, F_T, generator=g).relu()
    t_logits = torch.randn(n, C, generator=g) * 2
    adj = mg._AdjT(torch.from_numpy(rowptr), torch.from_numpy(c), n)
    data = argparse.Namespace(x=x, adj_t=adj, y=y.view(-1, 1))
    cases = {}
    for name, (script, kind, kernel, beta) in CASES.items():
        mod = scripts[script]
        torch.manual_seed(7)
        model = (mod.GCN if kind == "gcn" else mod.SAGE)(N_IN, HID, C, L, 0.0)
        sproj = torch.nn.Sequential(torch.nn.Linear(HID, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
        tproj = torch.nn.Sequential(torch.nn.Linear(F_T, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
        opt = torch.optim.Adam([{"params": model.parameters(), "lr": 0.01}, {"params": sproj.parameters(), "lr": 0.01},
                                {"params": tproj.parameters(), "lr": 0.01}])
        init = dict(model=state(model), sproj=state(sproj), tproj=state(tproj))
        args = argparse.Namespace(training="gpw", beta=beta, kernel=kernel, max_samples=S, alpha=0.9, kd_T=4.0)
        np.random.seed(5)
        draw = torch.from_numpy(np.random.choice(train_idx.numel(), S, replace=False))
        np.random.seed(5)
        loss, loss_cls, loss_aux = mod.train(model, data, train_idx, opt, args, t_feat, t_logits, sproj, tproj)
        cases[name] = dict(
            kernel=kernel, beta=beta, init=init, draw=draw, loss=loss, loss_cls=loss_cls, loss_aux=loss_aux,
            grads=dict(model={k: p.grad.clone() for k, p in model.named_parameters()},
                       sproj={k: p.grad.clone() for k, p in sproj.named_parameters()},
                       tproj={k: p.grad.clone() for k, p in tproj.named_parameters()}),
            after=dict(model=state(model), sproj=state(sproj), tproj=state(tproj)))
    torch.save(dict(sym_row=torch.from_numpy(r), sym_col=torch.from_numpy(c), x=x, y=y, train_idx=train_idx, t_feat=t_feat,
                    t_logits=t_logits, hp=dict(hidden=HID, proj=PROJ, S=S, alpha=0.9, kd_T=4.0, lr=0.01, layers=L),
                    cases=cases), mg.OUT / "gsp_arxiv.pt")


if __name__ == "__main__":
    main()
