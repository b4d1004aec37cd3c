"""The lane-copy column-slab SpMM kernel (spmm_rows_slab_kernel), which the automatic dispatch picks for K = 128 and 256 when
X is larger than the L2 budget (b200gnn_spmm_csr_f32): where it runs, and that it reproduces spmm_rows_bulk_kernel bit for
bit — every Y element and every statistics slot, on random non-dyadic data as well as on the exact dyadic data of
test_sparse_exact_gpu.py, and through three training steps of the engine."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops, synthetic
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.sparse import CsrGraph, SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
SUM, MEAN = lib.REDUCE_SUM, lib.REDUCE_MEAN
CANARY = 0x7FC0DEAD
NAN_BITS = 0x7FC00000
BULK_VARIANT = {256: 5, 128: 4}       # the bulk-copy kernel with 256- / 128-float slabs: the automatic choice below the budget


def _gcn_graph(n: int, e: int, seed: int = 0) -> CsrGraph:
    """Symmetric, self-looped, GCN-normalised skewed graph (the benchmark's construction) as an engine CSR."""
    ei = synthetic.skewed_edges(n, e, seed).to(DEV)
    row, col = ei
    perm = (col * n + row).argsort()
    adj = SparseTensor(row=col[perm], col=row[perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    adj = adj.fill_value(1.0).fill_diag(1.0)
    dis = adj.sum(1).pow(-0.5)
    dis[torch.isinf(dis)] = 0
    r, c, v = adj.coo()
    return adj.set_value(dis[r] * v * dis[c]).storage.engine_csr()


_GRAPHS = {}


def graph(name: str) -> CsrGraph:
    """arxiv: the benchmark's shape (169,343 nodes); mid: 60,000 / 120,000 sources, X still beyond the budget at K = 256 /
    128; small: 24,000 sources (24.6 MB at K = 256), below it."""
    if name not in _GRAPHS:
        S = synthetic.ARXIV
        n, e = {"arxiv": (S["num_nodes"], S["num_edges"]), "mid256": (60_000, 400_000), "mid128": (120_000, 800_000),
                "small": (24_000, 160_000)}[name]
        _GRAPHS[name] = _gcn_graph(n, e)
    return _GRAPHS[name]


def _spmm_c(G: CsrGraph, val, xv, yv, K, reduce, bias, part) -> int:
    ws = G.hub_workspace(K)
    return lib.load().b200gnn_spmm_csr_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), None if val is None else val.data_ptr(), xv.data_ptr(), xv.stride(0),
        yv.data_ptr(), yv.stride(0), G.n_rows, G.n_cols, K, reduce, None if bias is None else bias.data_ptr(),
        None if part is None else part.data_ptr(), G.chunk_rowptr.data_ptr(), G.n_chunks, G.hub_threshold, G.seg_len,
        G.hub_rows.data_ptr() if G.n_hub else None, G.hub_segptr.data_ptr() if G.n_hub else None, G.n_hub, G.n_seg,
        None if ws is None else ws.data_ptr(), lib.stream_ptr())


@pytest.fixture
def spmm_variant():
    yield ops.set_spmm_variant
    ops.set_spmm_variant(0)


def _kernels(fn) -> set:
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages()}


# ================================================================================================================ dispatch
@pytest.mark.parametrize("name,K,kernel", [("arxiv", 256, "spmm_rows_slab_kernel"), ("arxiv", 128, "spmm_rows_slab_kernel"),
                                           ("small", 256, "spmm_rows_bulk_kernel")])
def test_dispatch(name, K, kernel):
    G = graph(name)
    x = torch.randn(G.n_cols, K, device=DEV)
    out = torch.empty(G.n_rows, K, device=DEV)
    part = torch.empty(int(lib.load().b200gnn_spmm_stat_slots(G.n_chunks, G.n_hub)), 2, K, device=DEV)
    ops.spmm_csr(G, x, "sum", out=out)                                  # warm-up outside the profiler
    names = _kernels(lambda: ops.spmm_csr(G, x, "sum", out=out, stat_partial=part))
    spmm = [k for k in names if "spmm_rows" in k]
    assert spmm and all(kernel in k for k in spmm), spmm


# ================================================================================ bit identity with the bulk kernel
class Poisoned:
    """X as a [n_src, K] view with pitch K + 4 (NaN in the padding), Y as a [n_rows, K] view inside a buffer of NaN canaries,
    a NaN-filled statistics buffer."""

    def __init__(self, G: CsrGraph, K: int, seed: int):
        g = torch.Generator(device=DEV).manual_seed(seed)
        self.G, self.K = G, K
        xbuf = torch.full((G.n_cols, K + 4), float("nan"), device=DEV)
        xbuf[:, :K] = torch.randn(G.n_cols, K, generator=g, device=DEV) * torch.exp2(
            torch.randint(-6, 7, (G.n_cols, 1), generator=g, device=DEV).float())
        self.X = xbuf[:, :K]
        self.bias = torch.randn(K, generator=g, device=DEV)
        self.ybuf = torch.empty((G.n_rows + 4) * (K + 8), dtype=torch.int32, device=DEV)
        self.Y = self.ybuf.view(torch.float32)[3 * (K + 8):].view(-1, K + 8)[:G.n_rows, :K]
        slots = int(lib.load().b200gnn_spmm_stat_slots(G.n_chunks, G.n_hub))
        self.part = torch.empty(slots * 2 * K, dtype=torch.int32, device=DEV)

    def run(self, val, reduce, use_bias, stats):
        self.ybuf.fill_(CANARY)
        self.Y.view(torch.int32).fill_(NAN_BITS)
        self.part.fill_(NAN_BITS)
        lib.check(_spmm_c(self.G, val, self.X, self.Y, self.K, reduce, self.bias if use_bias else None,
                          self.part.view(torch.float32) if stats else None), "spmm_csr_f32")
        torch.cuda.synchronize()
        return self.ybuf.clone(), self.part.clone()


@pytest.mark.parametrize("name,K", [("arxiv", 256), ("arxiv", 128), ("mid256", 256), ("mid128", 128)])
def test_slab_matches_bulk_bitwise(name, K, spmm_variant):
    """Sum and mean, weighted and unweighted, with and without bias and statistics: the whole Y buffer (canaries included)
    and every statistics slot equal to the bulk kernel's, bit for bit."""
    G = graph(name)
    case = Poisoned(G, K, seed=K)
    val = G.val
    for reduce in (SUM, MEAN):
        for weights in (val, None):
            for use_bias in (False, True):
                for stats in (False, True):
                    spmm_variant(0)
                    y, part = case.run(weights, reduce, use_bias, stats)
                    spmm_variant(BULK_VARIANT[K])
                    y_ref, part_ref = case.run(weights, reduce, use_bias, stats)
                    what = (name, K, reduce, weights is not None, use_bias, stats)
                    assert torch.equal(y, y_ref), what
                    assert torch.equal(part, part_ref), what
                    if stats:
                        assert not bool((part == NAN_BITS).any()), what
                    assert bool((y != CANARY).sum() == G.n_rows * K), what


# ============================================================================================ exact on dyadic data
N_SRC = 140_000                       # X beyond the budget at K = 128 (72 MB) and K = 256 (143 MB)
PLANS = [(256, 256, 128, 4), (31, 7, 5, 1), (255, 257, 33, 2)]   # (hub_threshold, seg_len, chunk_nnz, row_cost)
EMPTY_RUNS = (1, 31, 32, 33, 100)
# 1-9, 15-17, 31-33, 63-65: the 8-edge commit groups, the 32- and 64-row rings, the 32-edge windows
BOUNDARY_DEGS = list(range(1, 10)) + [15, 16, 17, 31, 32, 33, 63, 64, 65]


def designed(plan, seed: int):
    """Hubs as the first and the last row, rows at hub_threshold ± 1, the degrees above, empty runs (leading, trailing and
    inside), columns uniform over N_SRC sources."""
    rng = np.random.default_rng(seed)
    thr = plan[0]
    body = []
    for i, d in enumerate(BOUNDARY_DEGS + [thr - 1, thr, thr + 1]):
        body += rng.integers(0, 24, size=6).tolist() + [d]
        if i % 3 == 0:
            body += [0] * EMPTY_RUNS[(i // 3) % len(EMPTY_RUNS)]
    filler = rng.integers(0, 30, size=3000)
    filler[rng.random(3000) < 0.15] = 0
    body += filler.tolist()
    degs = np.asarray([2000] + [0] * 33 + body + [0] * 100 + [3000], dtype=np.int64)
    rowptr = np.concatenate([[0], np.cumsum(degs)])
    col = rng.integers(0, N_SRC, size=int(rowptr[-1]))
    return rowptr, col, degs.size


@pytest.mark.parametrize("plan", PLANS, ids=["default", "31-7-5-1", "255-257-33-2"])
@pytest.mark.parametrize("K", [256, 128])
def test_slab_exact_dyadic(plan, K, spmm_variant):
    """X in {-1, 0, 1}, values in 2^-2 Z ∩ (0, 2], bias in 2^-2 Z: every partial sum is exact in fp32, so Y must equal the fp64
    scatter sum rounded once (mean: S / deg rounded, then + bias rounded); the statistics equal the bulk kernel's."""
    rowptr, col, n_rows = designed(plan, seed=K + plan[2])
    G = CsrGraph(torch.from_numpy(rowptr).to(DEV, torch.int32), torch.from_numpy(col).to(DEV, torch.int32), None, n_rows,
                 N_SRC).build_plan(*plan)
    assert G.n_hub >= 2
    g = torch.Generator(device=DEV).manual_seed(K)
    val = torch.randint(1, 9, (int(rowptr[-1]),), generator=g, device=DEV).float() / 4
    x = torch.randint(-4, 5, (N_SRC, K), generator=g, device=DEV).div(4, rounding_mode="trunc").float()
    bias = torch.randint(-8, 9, (K,), generator=g, device=DEV).float() / 4
    rows = torch.from_numpy(np.repeat(np.arange(n_rows), np.diff(rowptr))).to(DEV)
    cols = torch.from_numpy(col).to(DEV)
    deg = torch.from_numpy(np.diff(rowptr)).to(DEV).double().clamp(min=1)[:, None]
    case = Poisoned(G, K, seed=0)
    case.X.copy_(x)
    case.bias = bias
    for reduce, w in ((SUM, val), (MEAN, None)):
        terms = x.double()[cols] * (w.double()[:, None] if w is not None else 1.0)
        S = torch.zeros(n_rows, K, dtype=torch.float64, device=DEV).index_add_(0, rows, terms)
        assert float(torch.zeros_like(S).index_add_(0, rows, terms.abs()).max()) * 4 < 2 ** 24
        del terms
        ref = (S if reduce == SUM else S / deg).float()
        for use_bias in (False, True):
            for stats in (False, True):
                spmm_variant(0)
                ybuf, part = case.run(w, reduce, use_bias, stats)
                assert torch.equal(case.Y, ref + bias if use_bias else ref), (plan, K, reduce, use_bias, stats)
                spmm_variant(BULK_VARIANT[K])
                ybuf_ref, part_ref = case.run(w, reduce, use_bias, stats)
                assert torch.equal(ybuf, ybuf_ref) and torch.equal(part, part_ref), (plan, K, reduce, use_bias, stats)


# ================================================================================================================ engine
def make_trainer(n=120_000, e=900_000, dims=(128, 256, 256, 40)):
    ei = skewed_edges(n, e, 0)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    tr = GCNStudentTrainer(adj, list(dims), dropout=0.5, seed=0)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, dims[0], generator=g).cuda()
    y = torch.randint(0, dims[-1], (n,), generator=g).cuda()
    t = (torch.randn(n, dims[-1], generator=g) * 2).cuda()
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values.cuda()
    return tr, (x, y, idx, t)


@pytest.mark.parametrize("graph_replay", [False, True])
def test_engine_slab_matches_bulk(graph_replay, spmm_variant):
    """Three training steps (120,000 nodes: every K = 128 and K = 256 aggregation beyond the budget) with the automatic
    choice and with the bulk kernel: losses, outputs, gradients and parameters bit-identical."""
    runs = []
    for variant in (0, 5):
        spmm_variant(variant)
        tr, inputs = make_trainer()
        if graph_replay:
            tr.capture(*inputs, warmup=1)
        losses = [(tr.replay() if graph_replay else tr.train_step(*inputs)).clone() for _ in range(3)]
        torch.cuda.synchronize()
        runs.append((tr, torch.stack(losses)))
    (got, l_got), (ref, l_ref) = runs
    assert torch.equal(l_got, l_ref)
    assert torch.equal(got.Y[-1], ref.Y[-1])
    assert torch.equal(got.grads, ref.grads)
    assert torch.equal(got.params, ref.params)
    assert torch.equal(got.out_feat(), ref.out_feat())
