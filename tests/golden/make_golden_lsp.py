"""Generate tests/golden/lsp_arxiv.pt by running the REFERENCE's own ``train()`` with ``--training lpw`` for one step:
arxiv_pyg/gnn.py (CE + beta * lpw) and arxiv_pyg/gnn_kd_and_aux.py (KD + beta * lpw), for the GCN and SAGE students and the
cosine and rbf kernels, on the stand-in convs of make_golden.py.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_lsp.py   (not run by the suite)

Small graph of make_golden.small_graph (240 nodes), 16 input features, hidden 32, 8 classes, 3 layers, dropout 0 (the masks
are the one draw that cannot be shared), a 90-wide teacher feature matrix (not a multiple of 4, like the real 750).  The
edge list is the reference's ``subgraph(train_idx, stack(adj_t.coo()[:2]), relabel_nodes=True)[0]`` of the symmetric
adjacency (gnn_kd_and_aux.py:240-243).  cosine runs at the scripts' beta 100, rbf (the default kernel) at beta 0.5.
Recorded per case: the initial state of the model, the three losses, every gradient (p.grad survives optimizer.step())
and the state after the step."""
from __future__ import annotations

import argparse
import importlib
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402

N_IN, HID, C, L, F_T = 16, 32, 8, 3, 90
KERNELS = {"cosine": 100.0, "rbf": 0.5}


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
    g = torch.Generator().manual_seed(41)
    x = torch.randn(n, N_IN, generator=g)
    y = torch.randint(0, C, (n,), generator=g)
    train_idx = torch.randperm(n, generator=g)[:150].sort().values
    t_feat = torch.randn(n, F_T, generator=g).relu()
    t_logits = torch.randn(n, C, generator=g) * 2
    adj = mg._AdjT(torch.from_numpy(rowptr), torch.from_numpy(c), n)
    data = argparse.Namespace(x=x, adj_t=adj, y=y.view(-1, 1))
    subgraph = sys.modules["torch_geometric.utils"].subgraph
    edge_index = subgraph(train_idx, torch.from_numpy(np.stack([r, c])), relabel_nodes=True)[0]
    cases = {}
    for script, mod in scripts.items():
        for kind, cls in (("gcn", mod.GCN), ("sage", mod.SAGE)):
            for kernel, beta in KERNELS.items():
                torch.manual_seed(7)
                model = cls(N_IN, HID, C, L, 0.0)
                opt = torch.optim.Adam(model.parameters(), lr=0.01)
                init = state(model)
                args = argparse.Namespace(training="lpw", beta=beta, kernel=kernel, alpha=0.9, kd_T=4.0)
                loss, loss_cls, loss_aux = mod.train(model, data, train_idx, opt, args, t_feat, t_logits, None, None,
                                                     edge_index)
                cases[f"{script}_{kind}_{kernel}"] = dict(
                    init=init, beta=beta, loss=loss, loss_cls=loss_cls, loss_aux=loss_aux,
                    grads={k: p.grad.clone() for k, p in model.named_parameters()}, after=state(model))
    torch.save(dict(sym_row=torch.from_numpy(r), sym_col=torch.from_numpy(c), x=x, y=y, train_idx=train_idx, t_feat=t_feat,
                    t_logits=t_logits, edge_index=edge_index,
                    hp=dict(hidden=HID, alpha=0.9, kd_T=4.0, lr=0.01, layers=L), cases=cases), mg.OUT / "lsp_arxiv.pt")


if __name__ == "__main__":
    main()
