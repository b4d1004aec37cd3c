"""Host-side mirrors of the PyG layer surface the reference uses (SURVEY.md §8b), backed by b200gnn kernels.

    GCNConv(in, out, cached=)            arxiv_pyg/gnn.py:28-35, ppi_pyg/gnn.py:125
    SAGEConv(in, out)                    arxiv_pyg/gnn.py:61-67
    MessagePassing(aggr=).propagate      mag_pyg/gnn.py:26-68 (custom RGCNConv)
    utils.softmax / subgraph / to_undirected

Parameter names and shapes follow PyG 1.6/1.7 (``GCNConv.weight`` is [in, out], ``SAGEConv.lin_l/lin_r`` are
``nn.Linear``), so ``state_dict``s are interchangeable with the reference's checkpoints.
Dense contractions run on the wgmma 3xTF32 GEMMs, aggregations on the CSR SpMM; both are differentiable.
"""
from __future__ import annotations

import inspect
import math
from typing import Optional

import torch

from . import lib, ops
from .engine import gcn_norm
from .sparse import SparseTensor


# ----------------------------------------------------------------------------------------- dense: y = x W^T (+b)
class _LinearTC(torch.autograd.Function):
    """x[M,in] @ weight[out,in]^T + bias on the tensor cores with fp32 fidelity; all three gradients too."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        x, weight = x.contiguous(), weight.contiguous()
        hi, lo = ops.split_tf32(weight)                                  # B[N=out, K=in]
        y = ops.gemm_tf32x3(x, hi, lo, bias=None if bias is None else bias.contiguous())
        ctx.save_for_backward(x, weight)
        ctx.has_bias = bias is not None
        return y

    @staticmethod
    def backward(ctx, gy):
        x, weight = ctx.saved_tensors
        gy = gy.contiguous()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            if gy.shape[1] % 4 == 0:
                hi, lo = ops.split_tf32(weight, transpose=True)          # B[N=in, K=out]
                gx = ops.gemm_tf32x3(gy, hi, lo)
            else:
                gx = torch.mm(gy, weight)                                # contraction width (out) off the TMA 16-byte pitch
        if ctx.needs_input_grad[1]:
            out_f, in_f = weight.shape
            if ops.wgrad_supported(out_f, in_f):
                gw = ops.gemm_wgrad_tf32x3(gy, x)                        # gy^T x : [out, in]
            else:
                gw = torch.mm(gy.t(), x)                                 # shapes outside the tensor-core tiling
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = ops.col_sum(gy) if gy.shape[1] % 4 == 0 and gy.shape[1] <= 1024 else gy.sum(0)
        return gx, gw, gb


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """F.linear on the b200gnn GEMMs when the layout allows (feature widths multiples of 4), cuBLAS otherwise."""
    if x.dim() == 2 and x.shape[0] == 0:          # an empty node-type mask / relation (mag_pyg/gnn.py:61-66): F.linear semantics
        return torch.nn.functional.linear(x, weight, bias)
    if x.is_cuda and x.dim() == 2 and x.shape[1] % 4 == 0 and x.dtype == torch.float32:
        return _LinearTC.apply(x, weight, bias)
    return torch.nn.functional.linear(x, weight, bias)


class Linear(torch.nn.Linear):
    def forward(self, x):
        return linear(x, self.weight, self.bias)


def glorot(t: torch.Tensor):
    a = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
    with torch.no_grad():
        t.uniform_(-a, a)


# ----------------------------------------------------------------------------------------- adjacency handling
def _as_adj(edge_index_or_adj, num_nodes: int) -> SparseTensor:
    """SparseTensor adj_t as is; a Tensor edge_index [2,E] (source -> target) becomes adj_t (row = target, col = source)."""
    if isinstance(edge_index_or_adj, SparseTensor):
        return edge_index_or_adj
    ei = edge_index_or_adj
    return SparseTensor(row=ei[1], col=ei[0], sparse_sizes=(num_nodes, num_nodes), is_sorted=False)


class GCNConv(torch.nn.Module):
    """out = D^-1/2 (A+I) D^-1/2 (x W) + b  (PyG GCNConv, SURVEY Appendix A.2)."""

    def __init__(self, in_channels, out_channels, improved=False, cached=False, add_self_loops=True, normalize=True,
                 bias=True, **kwargs):
        super().__init__()
        if improved or not add_self_loops or not normalize:
            raise NotImplementedError("the reference only uses GCNConv defaults (+cached)")
        self.in_channels, self.out_channels, self.cached = in_channels, out_channels, cached
        self.weight = torch.nn.Parameter(torch.empty(in_channels, out_channels))
        self.bias = torch.nn.Parameter(torch.empty(out_channels)) if bias else None
        self._cached_adj_t = None
        self.reset_parameters()

    def reset_parameters(self):
        glorot(self.weight)
        if self.bias is not None:
            torch.nn.init.zeros_(self.bias)
        self._cached_adj_t = None

    def forward(self, x, edge_index, edge_weight=None):
        if edge_weight is not None:
            raise NotImplementedError
        adj = self._cached_adj_t
        if adj is None:
            adj = gcn_norm(_as_adj(edge_index, x.size(0)))
            if self.cached:
                self._cached_adj_t = adj
        h = linear(x, self.weight.t())                 # x @ weight  (weight stored [in,out] like PyG 1.x)
        out = ops.matmul(adj, h, "add")
        return out if self.bias is None else out + self.bias

    def __repr__(self):
        return f"GCNConv({self.in_channels}, {self.out_channels})"


class SAGEConv(torch.nn.Module):
    """out = lin_l(mean_j x_j) + lin_r(x_i)  (PyG SAGEConv, Appendix A.3)."""

    def __init__(self, in_channels, out_channels, normalize=False, root_weight=True, bias=True, **kwargs):
        super().__init__()
        if normalize or not root_weight:
            raise NotImplementedError("the reference only uses SAGEConv defaults")
        self.in_channels, self.out_channels = in_channels, out_channels
        self.lin_l = Linear(in_channels, out_channels, bias=bias)
        self.lin_r = Linear(in_channels, out_channels, bias=False)

    def reset_parameters(self):
        self.lin_l.reset_parameters()
        self.lin_r.reset_parameters()

    def forward(self, x, edge_index):
        adj = _as_adj(edge_index, x.size(0))
        if adj.has_value():
            adj = adj.set_value(None)
        return self.lin_l(ops.matmul(adj, x, "mean")) + self.lin_r(x)

    def __repr__(self):
        return f"SAGEConv({self.in_channels}, {self.out_channels})"


class GINConv(torch.nn.Module):
    """out = nn((1 + eps) * x_i + sum_j x_j)  (PyG GINConv; BASELINE.json north_star names it beside GCN/SAGE — the
    reference's mol_pyg/ students — and it is the sum-aggregation SpMM followed by the caller's MLP)."""

    def __init__(self, nn: torch.nn.Module, eps: float = 0.0, train_eps: bool = False, **kwargs):
        super().__init__()
        self.nn = nn
        self.initial_eps = float(eps)
        if train_eps:
            self.eps = torch.nn.Parameter(torch.tensor([float(eps)]))
        else:
            self.register_buffer("eps", torch.tensor([float(eps)]))

    def reset_parameters(self):
        for m in self.nn.modules():
            if m is not self.nn and hasattr(m, "reset_parameters"):
                m.reset_parameters()
        self.eps.data.fill_(self.initial_eps)

    def forward(self, x, edge_index):
        adj = _as_adj(edge_index, x.size(0))
        if adj.has_value():
            adj = adj.set_value(None)
        return self.nn(ops.matmul(adj, x, "sum") + (1.0 + self.eps) * x)

    def __repr__(self):
        return f"GINConv(nn={self.nn})"


class DGLGraphConv(torch.nn.Module):
    """DGL ``GraphConv(in, out, norm='both')`` as the reference's DGL student uses it (arxiv_dgl/models.py:46-92, ctor :65):
    ``out = D_in^-1/2 A D_out^-1/2 x W + b`` with degrees clamped to >= 1 and no self-loops added (the script adds them to the
    graph).  Called as ``conv(adj_t, feat)`` with a SparseTensor (row = destination, col = source) in place of the DGL graph.
    The two degree scalings are folded into the edge values once per adjacency, so the layer is one weighted SpMM and one
    wgmma GEMM; like DGL the narrower side is aggregated (W first iff in > out)."""

    def __init__(self, in_feats, out_feats, norm="both", weight=True, bias=True, activation=None):
        super().__init__()
        if norm != "both" or not weight:
            raise NotImplementedError("the reference only uses GraphConv(norm='both') with a weight")
        self._in, self._out, self._activation = in_feats, out_feats, activation
        self.weight = torch.nn.Parameter(torch.empty(in_feats, out_feats))
        self.bias = torch.nn.Parameter(torch.empty(out_feats)) if bias else None
        self._norm_adj = (None, None)
        self.reset_parameters()

    def reset_parameters(self):
        torch.nn.init.xavier_uniform_(self.weight)
        if self.bias is not None:
            torch.nn.init.zeros_(self.bias)

    def _normalised(self, adj_t: SparseTensor) -> SparseTensor:
        if self._norm_adj[0] is not adj_t:
            st = adj_t.storage
            row, col = st.row(), st.col()
            d_in = st.rowcount().clamp(min=1).to(torch.float32).pow(-0.5)
            d_out = torch.bincount(col, minlength=adj_t.size(1)).clamp(min=1).to(torch.float32).pow(-0.5)
            val = d_in[row] * d_out[col]
            if st.value() is not None:
                val = val * st.value()
            self._norm_adj = (adj_t, adj_t.set_value(val, layout="coo"))
        return self._norm_adj[1]

    def forward(self, adj_t: SparseTensor, feat: torch.Tensor) -> torch.Tensor:
        A = self._normalised(adj_t)
        if self._in > self._out:
            rst = ops.matmul(A, linear(feat, self.weight.t()), "add")
        else:
            rst = linear(ops.matmul(A, feat, "add"), self.weight.t())
        if self.bias is not None:
            rst = rst + self.bias
        return rst if self._activation is None else self._activation(rst)


def neighbor_average_features(adj_t: SparseTensor, feat: torch.Tensor, R: int):
    """SIGN precompute (arxiv_dgl/sign.py:175-183): ``feat_r = mean over in-neighbours of feat_{r-1}`` for r = 1..R
    (DGL ``update_all(copy_u, mean)``; nodes without in-edges get zeros).  Returns ``[feat_0, ..., feat_R]`` —
    R chained mean-SpMMs on the same CSR plan."""
    A = adj_t.set_value(None) if adj_t.has_value() else adj_t
    res = [feat]
    for _ in range(R):
        res.append(ops.matmul(A, res[-1], "mean"))
    return res


# ----------------------------------------------------------------------------------------- generic message passing
def scatter(src: torch.Tensor, index: torch.Tensor, dim: int = 0, dim_size: Optional[int] = None, reduce: str = "sum"):
    """torch_scatter.scatter(src, index, dim=0, dim_size, reduce in {sum, add, mean}) as one SpMM: the [dim_size x E]
    selection matrix has a single non-zero per column, so out = S @ src is the scatter — deterministic, no atomics."""
    if dim != 0 or src.dim() != 2:
        raise NotImplementedError("scatter: the reference path only reduces [E, F] messages over dim 0")
    if reduce not in ("sum", "add", "mean"):
        raise NotImplementedError(f"scatter reduce={reduce!r}")
    n = int(index.max()) + 1 if dim_size is None else dim_size
    return ops.matmul(_selection_matrix(index, n), src, "mean" if reduce == "mean" else "sum")


_SEL_CACHE: dict = {}


def _selection_matrix(index: torch.Tensor, n: int) -> SparseTensor:
    """The [n x E] selection matrix of a scatter index, with its sort, CSR/CSC views and chunk/hub plans, cached per index
    tensor (RGCNConv scatters over the same 7 relation masks every layer and every step: mag_pyg/gnn.py:54-68).  The cache
    keeps a reference to the index tensor, so its address cannot be recycled for different contents while the entry lives."""
    key = (index.data_ptr(), int(index.numel()), index._version, n, str(index.device))
    hit = _SEL_CACHE.get(key)
    if hit is not None and hit[0] is index:
        return hit[1]
    E = index.numel()
    sel = SparseTensor(row=index, col=torch.arange(E, device=index.device), sparse_sizes=(n, E), is_sorted=False)
    if len(_SEL_CACHE) > 64:
        _SEL_CACHE.clear()
    _SEL_CACHE[key] = (index, sel)
    return sel


class MessagePassing(torch.nn.Module):
    """The slice of PyG's MessagePassing the reference's custom RGCNConv needs (mag_pyg/gnn.py:26-68):
    ``propagate(edge_index, x=..., **extras)`` -> ``message(x_j, **extras)`` -> scatter(aggr) onto the targets."""

    def __init__(self, aggr: str = "add", flow: str = "source_to_target", node_dim: int = 0):
        super().__init__()
        if flow != "source_to_target" or node_dim != 0:
            raise NotImplementedError
        self.aggr = aggr

    def propagate(self, edge_index, size=None, **kwargs):
        x = kwargs.get("x")
        if isinstance(edge_index, SparseTensor):
            row, col, _ = edge_index.coo()
            src, dst, n = col, row, edge_index.size(0)
        else:
            src, dst = edge_index[0], edge_index[1]
            n = x.size(0) if x is not None else int(dst.max()) + 1
        params = inspect.signature(self.message).parameters
        if dst.numel() == 0 and x is not None:        # empty relation: nothing to gather, message() never sees an empty batch
            return self.update(x.new_zeros(n, self._empty_out_width(x, kwargs)))
        args = {}
        for name in params:
            if name.endswith("_j"):
                args[name] = kwargs[name[:-2]].index_select(0, src)
            elif name.endswith("_i"):
                args[name] = kwargs[name[:-2]].index_select(0, dst)
            elif name in kwargs:
                args[name] = kwargs[name]
        msg = self.message(**args)
        if dst.numel() == 0:
            return msg.new_zeros(n, msg.shape[1])
        return self.update(scatter(msg, dst, 0, n, self.aggr))

    def message(self, x_j):
        return x_j

    def _empty_out_width(self, x, kwargs) -> int:
        """Output width of message() for an empty edge set, probed with a zero-row batch on the CPU-free meta path."""
        params = inspect.signature(self.message).parameters
        args = {}
        for name in params:
            if name.endswith("_j") or name.endswith("_i"):
                args[name] = kwargs[name[:-2]][:0]
            elif name in kwargs:
                args[name] = kwargs[name]
        return int(self.message(**args).shape[1])

    def update(self, inputs):
        return inputs


# ----------------------------------------------------------------------------- hetero input assembly (a14)
class _GroupInput(torch.autograd.Function):
    """h[i] = table[node_type[i]][local_node_idx[i]]; backward = deterministic typed scatter into the tables that need a
    gradient (b200gnn_typed_gather_f32 / b200gnn_typed_scatter_f32)."""

    @staticmethod
    def forward(ctx, node_type, local_node_idx, in_channels, keys, *tables):
        dev = node_type.device
        if not node_type.is_cuda:
            raise lib.B200GnnError("group_input: CUDA tensors only (no CPU fallback)")
        n_tables = (max(keys) + 1) if keys else 1
        # the reference indexes with any integer tensor; the kernels read int64
        nt, li = node_type.reshape(-1).long().contiguous(), local_node_idx.reshape(-1).long().contiguous()
        out = torch.empty(nt.numel(), in_channels, device=dev)
        ops.typed_gather(dict(zip(keys, tables)), n_tables, nt, li, out)   # raises on an index outside its table
        ctx.keys, ctx.shapes, ctx.n_tables = keys, [tuple(t.shape) for t in tables], n_tables
        ctx.save_for_backward(nt, li)
        return out

    @staticmethod
    def backward(ctx, d_out):
        nt, li = ctx.saved_tensors
        n = d_out.shape[0]
        needs = ctx.needs_input_grad[4:]
        grads = [torch.zeros(sh, device=d_out.device) if need else None for sh, need in zip(ctx.shapes, needs)]
        if any(needs) and n:
            # every index of a type with a table is below big (the forward checked it); clamping the others, which the
            # scatter skips, keeps their keys from landing inside a table type's run and splitting it in two
            big = int(max(sh[0] for sh in ctx.shapes)) + 1
            order = torch.argsort(nt * big + li.clamp(0, big - 1), stable=True)
            ops.typed_scatter(d_out.contiguous(), nt, li, order,
                              {k: g for k, g in zip(ctx.keys, grads) if g is not None}, ctx.n_tables)
        return (None, None, None, None, *grads)


def group_input(x_dict, emb_dict, node_type: torch.Tensor, local_node_idx: torch.Tensor, in_channels: int) -> torch.Tensor:
    """RGCN.group_input (mag_pyg/gnn.py:111-124): the [n, in_channels] input of the sampled / full heterogeneous graph,
    row i taken from the feature table (x_dict, int keys) or the embedding table (emb_dict, str keys as in the reference's
    ParameterDict) of node_type[i] at local_node_idx[i].  Types without a table give zero rows, as in the reference."""
    keys, tables = [], []
    for k, x in x_dict.items():
        keys.append(int(k)); tables.append(x)
    for k, e in emb_dict.items():
        keys.append(int(k)); tables.append(e)
    return _GroupInput.apply(node_type, local_node_idx, int(in_channels), tuple(keys), *tables)


# ----------------------------------------------------------------------------------------- utils
def subgraph(subset, edge_index, edge_attr=None, relabel_nodes=False, num_nodes=None):
    """torch_geometric.utils.subgraph (SURVEY A.7): induced subgraph, edge order preserved, ids = positions in subset."""
    n = num_nodes if num_nodes is not None else int(edge_index.max()) + 1
    if subset.dtype == torch.bool:
        n_mask = subset
        subset = subset.nonzero().view(-1)
    else:
        n = max(n, int(subset.max()) + 1) if subset.numel() else n
        n_mask = torch.zeros(n, dtype=torch.bool, device=edge_index.device)
        n_mask[subset] = True
    mask = n_mask[edge_index[0]] & n_mask[edge_index[1]]
    ei = edge_index[:, mask]
    if relabel_nodes:
        n_idx = torch.zeros(n_mask.numel(), dtype=torch.long, device=edge_index.device)
        n_idx[subset] = torch.arange(subset.numel(), device=edge_index.device)
        ei = n_idx[ei]
    return ei, (edge_attr[mask] if edge_attr is not None else None)


def to_undirected(edge_index, num_nodes=None):
    n = num_nodes if num_nodes is not None else int(edge_index.max()) + 1
    r, c, _ = SparseTensor(row=edge_index[0], col=edge_index[1], sparse_sizes=(n, n)).to_symmetric().coo()
    return torch.stack([r, c])


def softmax(src, index, ptr=None, num_nodes=None):
    """torch_geometric.utils.softmax(src, index): e / (sum_e + 1e-16) with the max subtracted per group.
    Composed from differentiable torch scatter primitives on the device (index plumbing); the LSP criterion in
    efficient_gnns_b200.criterion fuses this with the similarity and the KL terms instead."""
    n = int(index.max()) + 1 if num_nodes is None else num_nodes
    shape = (n,) + tuple(src.shape[1:])
    idx = index.view(-1, *([1] * (src.dim() - 1))).expand_as(src)
    m = torch.full(shape, float("-inf"), dtype=src.dtype, device=src.device).scatter_reduce_(0, idx, src.detach(), "amax")
    e = (src - m.index_select(0, index)).exp()
    s = torch.zeros(shape, dtype=src.dtype, device=src.device).scatter_add_(0, idx, e)
    return e / (s.index_select(0, index) + 1e-16)


# ----------------------------------------------------------------------------------------- graph attention
class _GatAggregate(torch.autograd.Function):
    """out[i,h,:] = sum_{j->i} softmax_j(leaky_relu(el[j,h] + er[i,h])) * ft[j,h,:]   (DGL apply_edges + edge_softmax +
    update_all, arxiv_dgl/models.py:202-217; PyG GATConv's message/aggregate) with its hand-written backward."""

    @staticmethod
    def forward(ctx, ft, el, er, adj: SparseTensor, H: int, D: int, slope: float, eps: float, edge_keep=None, attn_scale=None):
        ft, el = ft.contiguous(), el.contiguous()
        er = None if er is None else er.contiguous()
        st = adj.storage
        G = st.engine_csr_unweighted() if st.value() is None else st.engine_csr()
        L, s = lib.load(), lib.stream_ptr()
        n = G.n_rows
        a = torch.empty(G.nnz, H, dtype=torch.float32, device=ft.device)
        lib.check(L.b200gnn_gat_edge_softmax_f32(G.rowptr.data_ptr(), G.col.data_ptr(), el.data_ptr(),
                                                 None if er is None else er.data_ptr(), n, H, slope, eps, a.data_ptr(),
                                                 None if edge_keep is None else edge_keep.data_ptr(), s),
                  "gat_edge_softmax_f32")
        a_used = a if attn_scale is None else a * attn_scale        # attention dropout (models.py:211-214)
        out = torch.empty(n, H * D, dtype=torch.float32, device=ft.device)
        _gat_aggregate(G, None, a_used, ft, out, H, D)
        ctx.adj, ctx.dims, ctx.slope = adj, (H, D), slope
        ctx.save_for_backward(ft, el, er if er is not None else el, a, a_used if attn_scale is not None else a,
                              attn_scale if attn_scale is not None else a)
        ctx.has_er, ctx.has_scale = er is not None, attn_scale is not None
        return out

    @staticmethod
    def backward(ctx, dout):
        ft, el, er, a, a_used, scale = ctx.saved_tensors
        H, D = ctx.dims
        er = er if ctx.has_er else None
        scale = scale if ctx.has_scale else None
        dout = dout.contiguous()
        st = ctx.adj.storage
        G = st.engine_csr_unweighted() if st.value() is None else st.engine_csr()
        L, s = lib.load(), lib.stream_ptr()
        dpre = torch.empty_like(a)
        der = torch.empty(G.n_rows, H, dtype=torch.float32, device=ft.device) if er is not None else None
        lib.check(L.b200gnn_gat_bwd_rows_f32(G.rowptr.data_ptr(), G.col.data_ptr(), a.data_ptr(), ft.data_ptr(), ft.stride(0),
                                             dout.data_ptr(), dout.stride(0), el.data_ptr(),
                                             None if er is None else er.data_ptr(), G.n_rows, H, D, ctx.slope, dpre.data_ptr(),
                                             None if der is None else der.data_ptr(), G.chunk_rowptr.data_ptr(), G.n_chunks,
                                             *_hub_args(G, H), None if scale is None else scale.data_ptr(), s),
                  "gat_bwd_rows_f32")
        Gt = st.engine_csc("value")                              # transposed graph as CSR (rows = sources)
        perm = _csr2csc_i32(st)
        dft = torch.empty(Gt.n_rows, H * D, dtype=torch.float32, device=ft.device)
        _gat_aggregate(Gt, perm, a_used, dout, dft, H, D)
        d_el = torch.empty(Gt.n_rows, H, dtype=torch.float32, device=ft.device)
        lib.check(L.b200gnn_segment_sum_heads_f32(Gt.rowptr.data_ptr(), perm.data_ptr(), dpre.data_ptr(), Gt.n_rows, H,
                                                  d_el.data_ptr(), s), "segment_sum_heads_f32")
        return dft, d_el, der, None, None, None, None, None, None, None


def _csr2csc_i32(st) -> torch.Tensor:
    p = st._engine.get("csr2csc_i32")
    if p is None:
        p = st._engine["csr2csc_i32"] = st.csr2csc().to(torch.int32).contiguous()
    return p


def _gat_aggregate(G, eidx, a, ft, out, H, D):
    lib.check(lib.load().b200gnn_gat_aggregate_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), None if eidx is None else eidx.data_ptr(), a.data_ptr(), ft.data_ptr(),
        ft.stride(0), out.data_ptr(), out.stride(0), G.n_rows, H, D, G.chunk_rowptr.data_ptr(), G.n_chunks,
        *_hub_args(G, H * D), lib.stream_ptr()), "gat_aggregate_f32")


def _hub_args(G, ws_width: int):
    """(hub_threshold, seg_len, hub_rows, hub_segptr, n_hub, n_seg, workspace[n_seg * ws_width]) of a CsrGraph plan."""
    if not G.n_hub:
        return G.hub_threshold, G.seg_len, None, None, 0, 0, None
    return (G.hub_threshold, G.seg_len, G.hub_rows.data_ptr(), G.hub_segptr.data_ptr(), G.n_hub, G.n_seg,
            G.hub_workspace(ws_width).data_ptr())


def gat_aggregate(ft, el, er, adj: SparseTensor, heads: int, negative_slope: float = 0.2, softmax_eps: float = 0.0,
                  edge_keep: Optional[torch.Tensor] = None, attn_scale: Optional[torch.Tensor] = None):
    """ft [N, heads*D], el [N, heads], er [N_dst, heads] or None, adj rows = destinations -> [N_dst, heads*D].
    edge_keep [nnz] uint8 (CSR order): dropped edges leave the softmax (edge_drop); attn_scale [nnz, heads] = keep/(1-p)
    multiplies the attention coefficients after the softmax (attention dropout)."""
    return _GatAggregate.apply(ft, el, er, adj, heads, ft.shape[1] // heads, float(negative_slope), float(softmax_eps),
                               edge_keep, attn_scale)


def _attention_masks(nnz: int, heads: int, edge_drop: float, attn_drop: float, training: bool, device):
    """(edge_keep, attn_scale) of one training forward (arxiv_dgl/models.py:206-214): a random permutation drops the first
    int(nnz*edge_drop) edges; nn.Dropout(attn_drop) on the coefficients.  torch's generator draws the decisions."""
    keep = scale = None
    if training and edge_drop > 0:
        perm = torch.randperm(nnz, device=device)
        keep = torch.ones(nnz, dtype=torch.uint8, device=device)
        keep[perm[:int(nnz * edge_drop)]] = 0
    if training and attn_drop > 0:
        scale = (torch.rand(nnz, heads, device=device) >= attn_drop).float() / (1.0 - attn_drop)
    return keep, scale


class DGLGATConv(torch.nn.Module):
    """The reference's DGL GATConv (arxiv_dgl/models.py:95-236) on a SparseTensor adjacency (rows = destinations):
    same parameters (fc, attn_l, attn_r, res_fc), symmetric degree normalisation, optional residual / activation.
    edge_drop / attn_drop (teacher training, models.py:206-214) are applied inside the fused kernels (edge keep-mask in the
    softmax, coefficient scaling in the aggregation and its backward); the random draws come from torch's generator."""

    def __init__(self, in_feats, out_feats, num_heads=1, feat_drop=0.0, attn_drop=0.0, edge_drop=0.0, negative_slope=0.2,
                 use_attn_dst=True, residual=False, activation=None, allow_zero_in_degree=False, use_symmetric_norm=False):
        super().__init__()
        self.attn_drop_p, self.edge_drop = float(attn_drop), float(edge_drop)
        self._num_heads, self._out_feats, self._slope = num_heads, out_feats, negative_slope
        self._use_symmetric_norm, self._activation = use_symmetric_norm, activation
        self.fc = Linear(in_feats, out_feats * num_heads, bias=False)
        self.attn_l = torch.nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.attn_r = torch.nn.Parameter(torch.empty(1, num_heads, out_feats)) if use_attn_dst else None
        self.feat_drop = torch.nn.Dropout(feat_drop)
        self.res_fc = Linear(in_feats, num_heads * out_feats, bias=False) if residual else None
        self.reset_parameters()

    def reset_parameters(self):
        gain = torch.nn.init.calculate_gain("relu")
        torch.nn.init.xavier_normal_(self.fc.weight, gain=gain)
        torch.nn.init.xavier_normal_(self.attn_l, gain=gain)
        if self.attn_r is not None:
            torch.nn.init.xavier_normal_(self.attn_r, gain=gain)
        if self.res_fc is not None:
            torch.nn.init.xavier_normal_(self.res_fc.weight, gain=gain)

    def forward(self, adj_t: SparseTensor, feat):
        H, D = self._num_heads, self._out_feats
        h = self.feat_drop(feat)
        ft = self.fc(h).view(-1, H, D)
        ft_dst = ft                    # models.py:187-188: the destination side keeps the raw projection (er is not degree-scaled)
        st = adj_t.storage
        if self._use_symmetric_norm:
            out_deg = torch.bincount(st.col(), minlength=adj_t.size(1)).float().clamp(min=1)
            ft = ft * out_deg.pow(-0.5).view(-1, 1, 1)
        el = (ft * self.attn_l).sum(-1)
        er = (ft_dst * self.attn_r).sum(-1) if self.attn_r is not None else None
        keep, scale = _attention_masks(st.col().numel(), H, self.edge_drop, self.attn_drop_p, self.training, feat.device)
        rst = gat_aggregate(ft.reshape(-1, H * D), el, er, adj_t, H, self._slope, 0.0, keep, scale).view(-1, H, D)
        if self._use_symmetric_norm:
            rst = rst * st.rowcount().float().clamp(min=1).pow(0.5).view(-1, 1, 1)
        if self.res_fc is not None:
            rst = rst + self.res_fc(h).view(h.shape[0], -1, D)
        return self._activation(rst) if self._activation is not None else rst


class GATConv(torch.nn.Module):
    """PyG 1.6/1.7 GATConv as used by ppi_pyg/gnn.py:27-31,53-61: shared ``lin`` (no bias), att_l / att_r, self-loops
    re-added, PyG softmax (eps 1e-16), concat or head-mean, bias."""

    def __init__(self, in_channels, out_channels, heads=1, concat=True, negative_slope=0.2, dropout=0.0, add_self_loops=True,
                 bias=True, **kwargs):
        super().__init__()
        self.dropout = float(dropout)          # PyG: F.dropout on the attention coefficients in training
        self.in_channels, self.out_channels, self.heads, self.concat = in_channels, out_channels, heads, concat
        self.negative_slope, self.add_self_loops = negative_slope, add_self_loops
        self.lin_l = Linear(in_channels, heads * out_channels, bias=False)
        self.lin_r = self.lin_l
        self.att_l = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        self.att_r = torch.nn.Parameter(torch.empty(1, heads, out_channels))
        self.bias = torch.nn.Parameter(torch.empty(heads * out_channels if concat else out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        glorot(self.lin_l.weight); glorot(self.att_l); glorot(self.att_r)
        if self.bias is not None:
            torch.nn.init.zeros_(self.bias)

    def forward(self, x, edge_index):
        H, C = self.heads, self.out_channels
        n = x.size(0)
        adj = _as_adj(edge_index, n)
        if self.add_self_loops:
            adj = adj.set_value(None).fill_diag(1.0) if adj.has_value() else _fill_diag_pattern(adj)
        xl = self.lin_l(x).view(-1, H, C)
        al, ar = (xl * self.att_l).sum(-1), (xl * self.att_r).sum(-1)
        _, scale = _attention_masks(adj.storage.col().numel(), H, 0.0, self.dropout, self.training, x.device)
        # The aggregation kernels move whole 128-bit vectors inside a head: a head width that is not a multiple of 4 (PPI's 121
        # classes, ppi_pyg/gnn.py:31,61) is zero-padded per head for the kernel and the padding sliced off again (exact).
        Cp = (C + 3) // 4 * 4
        ft = xl if Cp == C else torch.nn.functional.pad(xl, (0, Cp - C))
        out = gat_aggregate(ft.reshape(-1, H * Cp), al, ar, adj, H, self.negative_slope, 1e-16, None, scale).view(-1, H, Cp)
        if Cp != C:
            out = out[..., :C]
        out = out.reshape(-1, H * C) if self.concat else out.mean(dim=1)
        return out if self.bias is None else out + self.bias


def _fill_diag_pattern(adj: SparseTensor) -> SparseTensor:
    """remove_self_loops + add_self_loops on a value-less adjacency."""
    row, col, _ = adj.coo()
    off = row != col
    d = torch.arange(min(adj.sparse_sizes()), device=row.device)
    return SparseTensor(row=torch.cat([row[off], d]), col=torch.cat([col[off], d]), sparse_sizes=adj.sparse_sizes(), is_sorted=False)
