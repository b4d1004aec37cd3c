"""Generate golden fixtures by running the REFERENCE's own Python files, unmodified, in the build container.

    python tests/golden/make_golden.py        REFERENCE=<checkout of the reference repository>   (not run by the test suite)

The reference's hot-path arithmetic lives in torch_geometric / torch_sparse, which are not installed,
so `arxiv_pyg/criterion.py` and `arxiv_pyg/gnn.py` are imported on top of minimal stand-in modules whose
operators come from oracle/ (the CPU restatement).  What the fixtures therefore pin:
  * criterion_*.pt  — outputs/gradients of the reference's six criteria (kd, fitnet, at, gpw, lpw, nce)
    computed BY THE REFERENCE FILE; only `softmax` (lpw) is a restated dependency.
  * model_*.pt      — logits / out_feat / parameter gradients of the reference's `GCN` and `SAGE` classes
    computed BY THE REFERENCE FILE on restated GCNConv / SAGEConv operators.
  * gat_arxiv.pt    — output / gradients of the reference's own DGL `GATConv` class (arxiv_dgl/models.py:95-236) computed
    BY THE REFERENCE FILE on a stand-in `dgl` whose four graph primitives (apply_edges(u_add_v|copy_u), edge_softmax,
    update_all(u_mul_e, sum), in/out_degrees) are restated with plain torch index ops.
  * sign_arxiv.pt   — `neighbor_average_features` of arxiv_dgl/sign.py:175-201 (R chained mean aggregations) run BY THE
    REFERENCE FILE on the same `dgl` stand-in, on the directed graph (zero in-degree rows included).
  * rgcn_mag.pt     — the reference's own `RGCNConv` / `RGCN` classes (mag_pyg/gnn.py:26-171): `forward` (per-relation
    MessagePassing with mean aggregation + per-type root Linear, `group_input` embedding assembly) and `inference`
    (per-relation SparseTensor.matmul(reduce='mean')) on a small 3-type / 5-relation graph, computed BY THE REFERENCE
    FILE on restated `MessagePassing.propagate` / `SparseTensor.matmul`.
Both oracle/ (tests, -m "not gpu") and the CUDA path (tests, -m gpu) must reproduce them.
Regenerating is deterministic up to the summation order of torch's multi-threaded CPU index_add_/scatter_add_ backward
(differences at the 1e-7 level in a few gradient entries), far inside the tolerances the tests apply.
"""
from __future__ import annotations

import importlib
import importlib.util
import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
REF = Path(os.environ.get("REFERENCE", "reference"))
OUT = Path(__file__).resolve().parent

from oracle import graph as og, ops as oo  # noqa: E402


# ----------------------------------------------------------------------------- stand-in modules
class _AdjT:
    """What the restated convs need from a SparseTensor: CSR arrays (+ cached GCN normalisation)."""

    def __init__(self, rowptr, col, n):
        self.rowptr, self.col, self.n = rowptr, col, n
        self._gcn = None

    def gcn(self):
        if self._gcn is None:
            row = np.repeat(np.arange(self.n), np.diff(self.rowptr.numpy()))
            r, c, v = og.gcn_norm(row, self.col.numpy(), self.n)
            self._gcn = (torch.from_numpy(og.ind2ptr(r, self.n)), torch.from_numpy(c), torch.from_numpy(v))
        return self._gcn


class GCNConv(torch.nn.Module):
    def __init__(self, in_channels, out_channels, cached=False):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.empty(in_channels, out_channels))
        self.bias = torch.nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        a = (6.0 / (self.weight.size(0) + self.weight.size(1))) ** 0.5
        torch.nn.init.uniform_(self.weight, -a, a)
        torch.nn.init.zeros_(self.bias)

    def forward(self, x, adj_t):
        rowptr, col, val = adj_t.gcn()
        return oo.spmm_scatter(torch.repeat_interleave(torch.arange(adj_t.n), rowptr[1:] - rowptr[:-1]), col, val,
                               x @ self.weight, adj_t.n, "sum") + self.bias


class SAGEConv(torch.nn.Module):
    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.lin_l = torch.nn.Linear(in_channels, out_channels, bias=True)
        self.lin_r = torch.nn.Linear(in_channels, out_channels, bias=False)

    def reset_parameters(self):
        self.lin_l.reset_parameters()
        self.lin_r.reset_parameters()

    def forward(self, x, adj_t):
        row = torch.repeat_interleave(torch.arange(adj_t.n), adj_t.rowptr[1:] - adj_t.rowptr[:-1])
        agg = oo.spmm_scatter(row, adj_t.col, None, x, adj_t.n, "mean")
        return self.lin_l(agg) + self.lin_r(x)


def install_stubs():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    na = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError("stub"))  # noqa: E731
    tg = mod("torch_geometric")
    tg.utils = mod("torch_geometric.utils", softmax=oo.segment_softmax, to_dense_adj=na, negative_sampling=na,
                   add_self_loops=na,
                   subgraph=lambda s, ei, relabel_nodes=False: (torch.from_numpy(
                       og.subgraph(s.numpy(), ei.numpy(), relabel_nodes)[0]), None))
    tg.nn = mod("torch_geometric.nn", GCNConv=GCNConv, SAGEConv=SAGEConv)
    tg.transforms = mod("torch_geometric.transforms", ToSparseTensor=na)
    ogb = mod("ogb")
    ogb.nodeproppred = mod("ogb.nodeproppred", PygNodePropPredDataset=na, Evaluator=na)


class _DGLGraph:
    """Homogeneous graph stand-in: edges src[e] -> dst[e]; the primitives GATConv.forward uses, in plain torch."""

    is_block = False

    def __init__(self, src, dst, n):
        self.src, self.dst, self.n = src, dst, n
        self.ndata, self.edata = {}, {}
        self.srcdata = self.dstdata = self.ndata

    def local_scope(self):
        import contextlib

        @contextlib.contextmanager
        def scope():
            nd, ed = dict(self.ndata), dict(self.edata)
            try:
                yield
            finally:
                self.ndata.clear(); self.ndata.update(nd); self.edata.clear(); self.edata.update(ed)
        return scope()

    def in_degrees(self): return torch.bincount(self.dst, minlength=self.n)
    def out_degrees(self): return torch.bincount(self.src, minlength=self.n)
    def number_of_edges(self): return int(self.src.numel())
    def number_of_dst_nodes(self): return self.n

    def apply_edges(self, f):
        if f[0] == "u_add_v":
            self.edata[f[3]] = self.srcdata[f[1]][self.src] + self.dstdata[f[2]][self.dst]
        elif f[0] == "copy_u":
            self.edata[f[2]] = self.srcdata[f[1]][self.src]
        else:
            raise NotImplementedError(f)

    def update_all(self, msg, red):
        if msg[0] == "copy_u" and red[0] == "mean":          # sign.py:182-183 (mean over in-edges, zero if none)
            assert msg[2] == red[1]
            self.dstdata[red[2]] = oo.scatter(self.srcdata[msg[1]][self.src], self.dst, self.n, "mean")
            return
        assert msg[0] == "u_mul_e" and red[0] == "sum" and msg[3] == red[1]
        m = self.srcdata[msg[1]][self.src] * self.edata[msg[2]]
        self.dstdata[red[2]] = torch.zeros((self.n,) + tuple(m.shape[1:]), dtype=m.dtype).index_add_(0, self.dst, m)


def install_dgl_stubs():
    def mod(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        sys.modules[name] = m
        return m

    dgl = mod("dgl")
    dgl.function = mod("dgl.function", u_add_v=lambda a, b, o: ("u_add_v", a, b, o), copy_u=lambda u, o: ("copy_u", u, o),
                       u_mul_e=lambda u, e, o: ("u_mul_e", u, e, o), sum=lambda m, o: ("sum", m, o),
                       mean=lambda m, o: ("mean", m, o))
    dgl.nn = mod("dgl.nn")
    dgl.nn.pytorch = mod("dgl.nn.pytorch", GraphConv=None)
    dgl.nn.pytorch.utils = mod("dgl.nn.pytorch.utils", Identity=torch.nn.Identity)
    dgl._ffi = mod("dgl._ffi")
    dgl._ffi.base = mod("dgl._ffi.base", DGLError=RuntimeError)
    dgl.ops = mod("dgl.ops", edge_softmax=lambda g, e, eids=None: oo.segment_softmax(e, g.dst, g.n))
    dgl.utils = mod("dgl.utils", expand_as_pair=lambda x: x if isinstance(x, tuple) else (x, x))


class _MessagePassing(torch.nn.Module):
    """PyG MessagePassing as RGCNConv uses it: x_j = x[edge_index[0]], message(x_j, **extras), aggr over edge_index[1]."""

    def __init__(self, aggr="add"):
        super().__init__()
        self.aggr = aggr

    def propagate(self, edge_index, x=None, **kw):
        msg = self.message(x_j=x[edge_index[0]], **kw)
        return oo.scatter(msg, edge_index[1], x.size(0), self.aggr)


class _SparseTensor:
    """torch_sparse.SparseTensor(row=, col=) with inferred sizes, .to(), .matmul(x, reduce)."""

    def __init__(self, row, col):
        self.row, self.col = row, col
        self.m = int(row.max()) + 1

    def to(self, *a, **k):
        return self

    def matmul(self, x, reduce="sum"):
        return oo.scatter(x[self.col], self.row, self.m, reduce)


def install_mag_stubs():
    install_stubs()
    na = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError("stub"))  # noqa: E731
    sys.modules["torch_sparse"] = types.ModuleType("torch_sparse")
    sys.modules["torch_sparse"].SparseTensor = _SparseTensor
    tg = sys.modules["torch_geometric"]
    tg.utils.to_undirected = na
    tg.nn.MessagePassing = _MessagePassing
    tg.data = types.ModuleType("torch_geometric.data")
    tg.data.Data, tg.data.GraphSAINTRandomWalkSampler = na, na
    sys.modules["torch_geometric.data"] = tg.data
    het = types.ModuleType("torch_geometric.utils.hetero")
    het.group_hetero_graph = na
    sys.modules["torch_geometric.utils.hetero"] = het
    tg.utils.hetero = het


def small_graph(n=240, e=1400, seed=3):
    from efficient_gnns_b200.synthetic import skewed_edges
    ei = skewed_edges(n, e, seed).numpy()
    row, col, _ = og.to_sparse_adj_t(ei, n)
    r, c = og.to_symmetric(row, col, n)
    return ei, r, c, og.ind2ptr(r, n)


def main():
    assert REF.exists(), "set REFERENCE to a checkout of the reference repository to regenerate the fixtures"
    install_stubs()
    sys.path.insert(0, str(REF / "arxiv_pyg"))
    crit = importlib.import_module("criterion")
    gnn = importlib.import_module("gnn")

    torch.manual_seed(0)
    g = torch.Generator().manual_seed(11)
    n, C, Fs, Ft = 240, 8, 24, 40
    ei, r, c, rowptr = small_graph(n)
    edge_index = torch.from_numpy(np.stack([r, c]))          # = torch.stack(adj_t.coo()[:2]) of the symmetric adj
    train_idx = torch.randperm(n, generator=g)[:150].sort().values
    sub_ei = torch.from_numpy(og.subgraph(train_idx.numpy(), edge_index.numpy(), True)[0])
    nt = train_idx.numel()

    logits = torch.randn(nt, C, generator=g)
    labels = torch.randint(0, C, (nt,), generator=g)
    t_logits = torch.randn(nt, C, generator=g) * 2
    feat = torch.randn(nt, Fs, generator=g).relu() + 0.01
    t_feat = torch.randn(nt, Ft, generator=g).relu() + 0.01
    same_t_feat = torch.randn(nt, Fs, generator=g)          # fitnet / nce / gpw need equal widths after projection
    inds = torch.randperm(nt, generator=g)[:64]

    cases = {}

    def run(name, fn, feats_need_grad=True):
        z = logits.clone().requires_grad_(True)
        f = feat.clone().requires_grad_(feats_need_grad)
        out = fn(z, f)
        loss = out[0]
        grads = torch.autograd.grad(loss, [z] + ([f] if feats_need_grad else []), allow_unused=True)
        cases[name] = dict(loss=out[0].detach(), loss_cls=out[1].detach(), loss_aux=out[2].detach(),
                           d_logits=grads[0], d_feat=grads[1] if feats_need_grad else None)

    run("kd", lambda z, f: crit.kd_criterion(z, labels, t_logits, 0.9, 4.0), False)
    run("fitnet", lambda z, f: crit.fitnet_criterion(z, labels, f, same_t_feat, 1000))
    run("at", lambda z, f: crit.at_criterion(z, labels, f, t_feat, 1000))
    for k in ("cosine", "poly", "l2", "rbf"):
        run(f"gpw_{k}", lambda z, f, k=k: crit.gpw_criterion(z, labels, f, t_feat, k, 1.0, 10 ** 9))
        run(f"lpw_{k}", lambda z, f, k=k: crit.lpw_criterion(z, labels, f, t_feat, sub_ei, k, 100))
    # sampled variants: seed numpy exactly like the reference's seed() does, record the draw
    np.random.seed(5)
    draw = torch.from_numpy(np.random.choice(nt, 64, replace=False))
    np.random.seed(5)
    run("gpw_cosine_sampled", lambda z, f: crit.gpw_criterion(z, labels, f, t_feat, "cosine", 1.0, 64))
    np.random.seed(5)
    run("nce_sampled", lambda z, f: crit.nce_criterion(z, labels, f, same_t_feat, 0.5, 0.075, 64))
    run("nce_full", lambda z, f: crit.nce_criterion(z, labels, f, same_t_feat, 0.5, 0.075, 10 ** 9))

    torch.save(dict(inputs=dict(logits=logits, labels=labels, t_logits=t_logits, feat=feat, t_feat=t_feat,
                                same_t_feat=same_t_feat, sub_edge_index=sub_ei, np_seed=5, np_draw=draw),
                    cases=cases), OUT / "criterion_arxiv.pt")

    # ---- models: the reference's GCN / SAGE classes
    x = torch.randn(n, 16, generator=g)
    adj = _AdjT(torch.from_numpy(rowptr), torch.from_numpy(c), n)
    models = {}
    for name, cls in (("gcn", gnn.GCN), ("sage", gnn.SAGE)):
        torch.manual_seed(1)
        m = cls(16, 32, C, 3, 0.0)  # dropout 0: the mask is the only thing that cannot be shared
        m.train()
        out = m(x, adj)
        y = torch.randint(0, C, (n,), generator=g)
        loss = torch.nn.functional.cross_entropy(out[train_idx], y[train_idx])
        loss.backward()
        models[name] = dict(state={k: v.detach().clone() for k, v in m.state_dict().items()},
                            logits_train=out.detach(), out_feat=m.out_feat.detach(), y=y, loss=loss.detach(),
                            grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})
        m.eval()
        models[name]["logits_eval"] = m(x, adj).detach()
    # ---- the reference's ProjectionGCD head (gnn.py:88-99): relu(BN(Linear(x) + GCNConv(x, adj_t))), non-cached conv
    torch.manual_seed(2)
    pg = gnn.ProjectionGCD(16, 12)
    pg.train()
    xin = x.clone().requires_grad_(True)
    wout = torch.randn(n, 12, generator=g)
    pout = pg(xin, adj)
    (pout * wout).sum().backward()
    models["proj_gcd"] = dict(state={k: v.detach().clone() for k, v in pg.state_dict().items()}, out_train=pout.detach(),
                              w=wout, d_x=xin.grad.detach().clone(),
                              grads={k: p.grad.detach().clone() for k, p in pg.named_parameters()})
    torch.save(dict(edge_index_directed=torch.from_numpy(ei), sym_row=torch.from_numpy(r), sym_col=torch.from_numpy(c),
                    x=x, train_idx=train_idx, sub_edge_index=sub_ei, models=models), OUT / "model_arxiv.pt")
    # ---- the reference's DGL GATConv layer (arxiv_dgl/models.py:95-236) on the symmetric graph + self-loops
    install_dgl_stubs()
    sys.path.insert(0, str(REF / "arxiv_dgl"))
    dgl_models = importlib.import_module("models")
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)       # row = destination, col = source
    graph = _DGLGraph(torch.from_numpy(cs), torch.from_numpy(rs), n)
    gat = {}
    for name, kw in (("attn_dst", dict(use_attn_dst=True)), ("no_attn_dst", dict(use_attn_dst=False))):
        torch.manual_seed(3)
        layer = dgl_models.GATConv(16, 8, num_heads=3, residual=True, use_symmetric_norm=True, **kw)
        layer.train()
        xin = x.clone().requires_grad_(True)
        wout = torch.randn(n, 3, 8, generator=g)
        out = layer(graph, xin)
        (out * wout).sum().backward()
        gat[name] = dict(state={k: v.detach().clone() for k, v in layer.state_dict().items()}, out=out.detach(), w=wout,
                         d_x=xin.grad.detach().clone(),
                         grads={k: p.grad.detach().clone() for k, p in layer.named_parameters()})
    torch.save(dict(row=torch.from_numpy(rs), col=torch.from_numpy(cs), x=x, layers=gat), OUT / "gat_arxiv.pt")
    # ---- SIGN precompute: the reference's neighbor_average_features (arxiv_dgl/sign.py:175-201)
    ogbm = sys.modules["ogb.nodeproppred"]
    ogbm.DglNodePropPredDataset = None
    if "torch.utils.tensorboard" not in sys.modules:
        try:
            importlib.import_module("torch.utils.tensorboard")
        except Exception:                                    # tensorboard is not installed everywhere: sign.py only names it
            tb = types.ModuleType("torch.utils.tensorboard")
            tb.SummaryWriter = None
            sys.modules["torch.utils.tensorboard"] = tb
    sign = importlib.import_module("sign")
    row_d, col_d, _ = og.to_sparse_adj_t(ei, n)              # directed: row = destination, col = source
    gd = _DGLGraph(torch.from_numpy(col_d), torch.from_numpy(row_d), n)
    gd.ndata["feat"] = x
    hops = sign.neighbor_average_features(gd, types.SimpleNamespace(R=3, dataset="ogbn-arxiv"))
    torch.save(dict(row=torch.from_numpy(row_d), col=torch.from_numpy(col_d), x=x, hops=[h.clone() for h in hops]),
               OUT / "sign_arxiv.pt")

    # ---- the reference's RGCN (mag_pyg/gnn.py): forward (MessagePassing formulation) and inference (SparseTensor formulation)
    install_mag_stubs()
    sys.path.insert(0, str(REF / "mag_pyg"))
    spec = importlib.util.spec_from_file_location("mag_gnn", REF / "mag_pyg" / "gnn.py")
    mag = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mag)
    gm = torch.Generator().manual_seed(21)
    nn_t = {0: 60, 1: 50, 2: 20}                              # node type -> count (0 carries features, 1/2 get embeddings)
    rels = [(1, 2, 90), (2, 1, 90), (1, 0, 200), (0, 1, 200), (0, 0, 240)]   # (src type, dst type, #edges)
    off = {0: 0, 1: 60, 2: 110}
    edge_index_dict, key2int, eis, ets = {}, {0: 0, 1: 1, 2: 2}, [], []
    for i, (sT, dT, e) in enumerate(rels):
        src = torch.randint(0, nn_t[sT], (e,), generator=gm)
        dst = torch.randint(0, nn_t[dT], (e,), generator=gm)
        src[-1], dst[-1] = nn_t[sT] - 1, nn_t[dT] - 1         # upstream infers sizes from the max index: make it exact
        key = (sT, f"r{i}", dT)
        edge_index_dict[key] = (src, dst)
        key2int[key] = i
        eis.append(torch.stack([src + off[sT], dst + off[dT]]))
        ets.append(torch.full((e,), i, dtype=torch.long))
    edge_index, edge_type = torch.cat(eis, 1), torch.cat(ets)
    node_type = torch.cat([torch.full((nn_t[t],), t, dtype=torch.long) for t in range(3)])
    local_idx = torch.cat([torch.arange(nn_t[t]) for t in range(3)])
    x_paper = torch.randn(nn_t[0], 16, generator=gm)
    torch.manual_seed(4)
    rg = mag.RGCN(16, 24, 5, 2, 0.5, nn_t, [0], len(rels))
    rg.eval()                                                 # no dropout: forward and inference must agree
    out_f = rg({0: x_paper}, edge_index, edge_type, node_type, local_idx)
    wout = torch.randn(130, 5, generator=gm)
    (out_f * wout).sum().backward()
    grads = {k: p.grad.detach().clone() for k, p in rg.named_parameters()}
    with torch.no_grad():
        inf = rg.inference({0: x_paper}, edge_index_dict, key2int)
    torch.save(dict(num_nodes=nn_t, rels=rels, edge_index_dict={k: torch.stack(v) for k, v in edge_index_dict.items()},
                    key2int=key2int, edge_index=edge_index, edge_type=edge_type, node_type=node_type,
                    local_node_idx=local_idx, x_paper=x_paper, state={k: v.detach().clone() for k, v in rg.state_dict().items()},
                    out_forward=out_f.detach(), out_feat=rg.out_feat.detach(), w=wout, grads=grads,
                    out_inference={k: v.clone() for k, v in inf.items()}), OUT / "rgcn_mag.pt")
    print("wrote", [p.name for p in OUT.glob("*.pt")])


if __name__ == "__main__":
    main()
