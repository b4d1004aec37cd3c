"""Generate tests/golden/ppi_model.pt by running the REFERENCE's own ``StudentNet`` and ``TeacherNet`` classes
(ppi_pyg/gnn.py:24-83), unmodified, on a plain-torch CPU restatement of PyG 1.7 ``GATConv``.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_ppi.py   (not run by the test suite)

The module-level imports of gnn.py / criterion.py are stubbed as make_golden.py does.  On a designed graph (n = 300, not a
multiple of 128): node 0 receives 280 edges (a hub above the engine's HUB_THRESHOLD of 256 once its self-loop is added),
node 299 has no edge but the self-loop GATConv adds, edge 5 -> 5 is a self-loop already present, 7 -> 8 appears twice.  10
input features (stored padded to 12) and 19 classes (a head width stored padded to 20) keep the file small.  The state is
``oracle.ppi.seeded_state`` (every parameter non-trivial), so it is not stored; tensors above 8192 entries are stored as
``oracle.ppi.fingerprint`` summaries.  Recorded per model: eval logits and out_feat, one supervised step's loss and every
parameter gradient, one kd step's loss and gradients with fixed teacher logits."""
from __future__ import annotations

import importlib
import sys
import types
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402

from oracle import ppi as oppi  # noqa: E402

N, F_IN, C = 300, 10, 19


class GATConv(torch.nn.Module):
    """PyG 1.7 GATConv (int in_channels, add_self_loops=True, dropout 0), restated with scatter ops."""

    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, bias=True):
        super().__init__()
        self.heads, self.out_channels, self.concat, self.negative_slope = heads, out_channels, concat, negative_slope
        self.lin_l = torch.nn.Linear(in_channels, heads * out_channels, bias=False)
        self.lin_r = self.lin_l
        self.att_l = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        self.att_r = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        self.bias = torch.nn.Parameter(torch.zeros(heads * out_channels if concat else out_channels))

    def reset_parameters(self):
        pass

    def forward(self, x, edge_index):
        H, D, n = self.heads, self.out_channels, x.shape[0]
        src, dst = edge_index
        keep = src != dst                                                    # remove_self_loops
        loop = torch.arange(n)
        src, dst = torch.cat([src[keep], loop]), torch.cat([dst[keep], loop])   # add_self_loops
        xl = self.lin_l(x).view(-1, H, D)
        alpha_l, alpha_r = (xl * self.att_l).sum(-1), (xl * self.att_r).sum(-1)
        alpha = torch.nn.functional.leaky_relu(alpha_l[src] + alpha_r[dst], self.negative_slope)
        idx = dst.view(-1, 1).expand_as(alpha)
        amax = torch.full((n, H), float("-inf")).scatter_reduce(0, idx, alpha, "amax", include_self=True)
        ex = (alpha - amax[dst]).exp()                                       # torch_geometric.utils.softmax
        alpha = ex / (torch.zeros(n, H).scatter_add(0, idx, ex)[dst] + 1e-16)
        out = torch.zeros(n, H, D).index_add(0, dst, xl[src] * alpha.unsqueeze(-1))
        out = out.reshape(n, H * D) if self.concat else out.mean(dim=1)
        return out + self.bias


def designed_edges():
    g = torch.Generator().manual_seed(31)
    s, d = torch.randint(1, N - 1, (1800,), generator=g), torch.randint(1, N - 1, (1800,), generator=g)
    hub_src = torch.arange(1, 281)
    src = torch.cat([s, hub_src, torch.tensor([5, 7, 7])])
    dst = torch.cat([d, torch.zeros(280, dtype=torch.long), torch.tensor([5, 8, 8])])
    return torch.stack([src, dst])                                           # PyG convention: row 0 source, row 1 target


def install_stubs():
    mg.install_stubs()
    tg = sys.modules["torch_geometric"]
    na = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError("stub"))  # noqa: E731
    tg.nn.GATConv = GATConv
    tg.utils.subgraph = na
    tg.datasets = types.ModuleType("torch_geometric.datasets")
    tg.datasets.PPI = na
    sys.modules["torch_geometric.datasets"] = tg.datasets
    tg.data = types.ModuleType("torch_geometric.data")
    tg.data.DataLoader = na
    sys.modules["torch_geometric.data"] = tg.data
    for name, attrs in (("sklearn", {}), ("sklearn.metrics", {"f1_score": na}), ("torch.utils.tensorboard", {"SummaryWriter": None})):
        if name == "torch.utils.tensorboard":
            try:
                importlib.import_module(name)
                continue
            except Exception:
                pass
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    install_stubs()
    sys.path.insert(0, str(mg.REF / "ppi_pyg"))
    gnn = importlib.import_module("gnn")
    crit = importlib.import_module("criterion")
    ei = designed_edges()
    g = torch.Generator().manual_seed(41)
    x = torch.randn(N, F_IN, generator=g)
    y = (torch.rand(N, C, generator=g) < 0.3).float()
    t_logits = torch.randn(N, C, generator=g) * 2
    out = dict(edge_index=ei.to(torch.int32), x=x, y=y.to(torch.uint8), teacher_logits=t_logits, in_channels=F_IN,
               out_channels=C, models={})
    for kind, cls, seed in (("student", gnn.StudentNet, 101), ("teacher", gnn.TeacherNet, 202)):
        m = cls(F_IN, C)
        state = oppi.seeded_state(oppi.layers_of(kind, C), F_IN, seed)
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == {k: tuple(v.shape) for k, v in state.items()}
        m.load_state_dict(state)
        case = dict(seed=seed)
        m.eval()
        with torch.no_grad():
            case["logits_eval"] = oppi.fingerprint(m(x, ei))
            case["out_feat_eval"] = oppi.fingerprint(m.out_feat)
        m.train()
        for mode in ("supervised", "kd"):
            m.zero_grad()
            logits = m(x, ei)
            if mode == "supervised":
                loss = torch.nn.functional.binary_cross_entropy_with_logits(logits, y)
                losses = (loss, loss, loss * 0)
            else:
                losses = crit.kd_criterion(logits, y, t_logits, 0.5, 1)
            losses[0].backward()
            case[mode] = dict(loss=torch.stack([v.detach() for v in losses]),
                              grads={k: oppi.fingerprint(p.grad) for k, p in m.named_parameters()})
        out["models"][kind] = case
    torch.save(out, mg.OUT / "ppi_model.pt")
    print("wrote ppi_model.pt", (mg.OUT / "ppi_model.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
