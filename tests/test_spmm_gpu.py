"""CUDA SpMM (through the C ABI) vs the CPU oracle: forward, backward, fused epilogues, edge cases.

Tolerance: max-norm relative error <= 1e-5 on fp32 (BASELINE.json north_star / SURVEY.md §8c)."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import fro_err, rel_err
from efficient_gnns_b200 import lib, ops
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og, ops as oo

pytestmark = pytest.mark.gpu
TOL = 1e-5


def sym_graph(n, e, seed):
    ei = skewed_edges(n, e, seed).numpy()
    row, col, _ = og.to_sparse_adj_t(ei, n)
    r, c = og.to_symmetric(row, col, n)
    return torch.from_numpy(r), torch.from_numpy(c)


def make_adj(r, c, n_rows, n_cols, val=None, device="cuda"):
    return SparseTensor(row=r.to(device), col=c.to(device), value=None if val is None else val.to(device),
                        sparse_sizes=(n_rows, n_cols), is_sorted=True)


@pytest.mark.parametrize("K", [1, 3, 4, 8, 31, 32, 33, 40, 64, 100, 128, 250, 256, 512, 750])
@pytest.mark.parametrize("reduce,weighted", [("sum", True), ("sum", False), ("mean", False)])
def test_spmm_forward_widths(K, reduce, weighted):
    n = 3000
    r, c = sym_graph(n, 20_000, 0)
    g = torch.Generator().manual_seed(K)
    x = torch.randn(n, K, generator=g)
    val = torch.rand(r.numel(), generator=g) if weighted else None
    ref = oo.spmm_scatter(r, c, val, x.double(), n, reduce) if val is None else \
        oo.spmm_scatter(r, c, val.double(), x.double(), n, reduce)
    adj = make_adj(r, c, n, n, val)
    out = adj.matmul(x.cuda(), reduce)
    assert out.shape == (n, K)
    assert rel_err(out, ref) < TOL and fro_err(out, ref) < TOL


@pytest.mark.parametrize("K", [40, 256])
def test_spmm_hub_rows_and_plan(K):
    """A hub of degree ~1.2e4 plus empty rows: the split path must agree with the oracle and the plan must be exact."""
    n = 20_000
    g = torch.Generator().manual_seed(5)
    hub_nbrs = torch.randperm(n, generator=g)[:12_345]
    mid_nbrs = torch.randperm(n, generator=g)[:700]
    row = torch.cat([torch.full((12_345,), 7), torch.full((700,), 4000), torch.randint(100, n - 50, (30_000,), generator=g)])
    col = torch.cat([hub_nbrs, mid_nbrs, torch.randint(0, n, (30_000,), generator=g)])
    r, c, _ = og.coalesce(row.numpy(), col.numpy(), n)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    val = torch.rand(r.numel(), generator=g)
    x = torch.randn(n, K, generator=g)
    adj = make_adj(r, c, n, n, val)
    G = adj.storage.engine_csr()
    deg = np.diff(og.ind2ptr(r.numpy(), n))
    hubs = np.nonzero(deg > G.hub_threshold)[0]
    assert G.n_hub == hubs.size and G.hub_rows[:G.n_hub].cpu().tolist() == hubs.tolist()
    segs = -(-deg[hubs] // G.seg_len)
    assert G.hub_segptr.cpu().tolist() == [0] + np.cumsum(segs).tolist() and G.n_seg == int(segs.sum())
    for reduce in ("sum", "mean"):
        a = adj if reduce == "sum" else adj.set_value(None)
        ref = oo.spmm_scatter(r, c, val.double() if reduce == "sum" else None, x.double(), n, reduce)
        out = a.matmul(x.cuda(), reduce)
        assert rel_err(out, ref) < TOL
        assert rel_err(out[7], ref[7]) < TOL and rel_err(out[4000], ref[4000]) < TOL
        assert torch.count_nonzero(out[:7]) == 0  # rows 0..6 are empty -> exactly 0


def test_spmm_rectangular_and_empty():
    g = torch.Generator().manual_seed(1)
    n_rows, n_cols, K = 500, 1300, 64
    row = torch.randint(0, n_rows, (4000,), generator=g)
    col = torch.randint(0, n_cols, (4000,), generator=g)
    r, c, _ = og.coalesce(row.numpy(), col.numpy(), n_cols)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    x = torch.randn(n_cols, K, generator=g)
    adj = make_adj(r, c, n_rows, n_cols)
    ref = oo.spmm_scatter(r, c, None, x.double(), n_rows, "mean")
    assert rel_err(adj.matmul(x.cuda(), "mean"), ref) < TOL
    # empty matrix: all-zero output, and zero rows: empty output
    e = torch.zeros(0, dtype=torch.long)
    out = make_adj(e, e, 10, 10).matmul(torch.randn(10, 8).cuda())
    assert out.shape == (10, 8) and torch.count_nonzero(out) == 0


@pytest.mark.parametrize("reduce,weighted", [("sum", True), ("mean", False)])
def test_spmm_backward_matches_autograd_oracle(reduce, weighted):
    n, K = 2500, 96
    ei = skewed_edges(n, 15_000, 3).numpy()          # directed => non-symmetric: exercises the CSC view
    r, c, _ = og.to_sparse_adj_t(ei, n)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    g = torch.Generator().manual_seed(2)
    val = torch.rand(r.numel(), generator=g) if weighted else None
    x = torch.randn(n, K, generator=g)
    w = torch.randn(n, K, generator=g)
    xr = x.double().requires_grad_(True)
    ref = oo.spmm_scatter(r, c, None if val is None else val.double(), xr, n, reduce)
    (ref * w.double()).sum().backward()
    xc = x.cuda().requires_grad_(True)
    out = make_adj(r, c, n, n, val).matmul(xc, reduce)
    (out * w.cuda()).sum().backward()
    assert rel_err(out, ref) < TOL
    assert rel_err(xc.grad, xr.grad) < TOL


def test_spmm_fused_bias_and_column_statistics():
    n, K = 5000, 256
    r, c = sym_graph(n, 40_000, 7)
    g = torch.Generator().manual_seed(3)
    val = torch.rand(r.numel(), generator=g)
    x, bias = torch.randn(n, K, generator=g), torch.randn(K, generator=g)
    adj = make_adj(r, c, n, n, val)
    G = adj.storage.engine_csr()
    assert G.n_hub > 0  # the skewed generator gives hubs; their statistics come from the finalize kernel
    part = torch.full((ops.stat_slots(G), 2, K), float("nan"), device="cuda")
    out = ops.spmm_csr(G, x.cuda(), "sum", bias=bias.cuda(), stat_partial=part)
    ref = oo.spmm_scatter(r, c, val.double(), x.double(), n, "sum") + bias.double()
    assert rel_err(out, ref) < TOL
    s = part.double().sum(0).cpu()
    assert rel_err(s[0], ref.sum(0)) < TOL
    assert rel_err(s[1], (ref * ref).sum(0)) < TOL
    # determinism: bitwise identical on a second run
    part2 = torch.empty_like(part)
    out2 = ops.spmm_csr(G, x.cuda(), "sum", bias=bias.cuda(), stat_partial=part2)
    assert torch.equal(out, out2) and torch.equal(part, part2)


def test_spmm_strided_operand_and_unaligned_views():
    n, K = 1000, 40
    r, c = sym_graph(n, 5000, 9)
    g = torch.Generator().manual_seed(4)
    big = torch.randn(n, 2 * K + 3, generator=g)
    adj = make_adj(r, c, n, n)
    G = adj.storage.engine_csr()
    xs = big.cuda()[:, 3:3 + K]                      # ld = 83 floats, base misaligned for float4
    with pytest.raises(lib.B200GnnError):
        ops.spmm_csr(G, xs)                          # non-contiguous views are rejected explicitly
    ref = oo.spmm_scatter(r, c, None, big[:, 3:3 + K].double(), n, "sum")
    assert rel_err(ops.spmm_csr(G, xs.contiguous()), ref) < TOL


def test_large_arxiv_shape_properties():
    """Full ARXIV-shape graph: no oracle run; size-independent properties instead.
    (1) linearity  A(ax+by) = aAx + bAy ; (2) A·1 = row sums ; (3) <Ax, y> = <x, A^T y> via the backward kernel."""
    from efficient_gnns_b200.synthetic import ARXIV
    n, K = ARXIV["num_nodes"], 128
    r, c = sym_graph(n, ARXIV["num_edges"], 0)
    g = torch.Generator().manual_seed(0)
    val = torch.rand(r.numel(), generator=g)
    adj = make_adj(r, c, n, n, val)
    x, y = torch.randn(n, K, generator=g).cuda(), torch.randn(n, K, generator=g).cuda()
    ax, ay = adj.matmul(x), adj.matmul(y)
    lin = adj.matmul(2.0 * x - 0.5 * y)
    assert rel_err(lin, 2.0 * ax - 0.5 * ay) < TOL
    ones = adj.matmul(torch.ones(n, 4, device="cuda"))
    rowsum = torch.zeros(n, dtype=torch.float64).index_add_(0, r, val.double())
    assert rel_err(ones[:, 0], rowsum) < TOL
    xg = x.clone().requires_grad_(True)
    (adj.matmul(xg) * y).sum().backward()            # grad = A^T y
    lhs = (ax.double() * y.double()).sum()
    rhs = (x.double() * xg.grad.double()).sum()
    assert abs(lhs - rhs) / abs(lhs) < 1e-6


# ---------------------------------------------------------------------------------------------- round 2: bulk-copy kernel
# variant word: 2 = cp.async ring, 3 = bulk (slab min(K,256)), 4 = bulk 128-float slabs, 5 = bulk 256-float slabs,
# 6 / 7 = bulk-copy ring over 128-float slabs with 8 / 4 edges per barrier, +16 evict_last gathers, +32 other barrier-group
# size, +64 two CTAs per SM (efficient-gnns_b200/csrc/spmm.cu)
BULK_VARIANTS = [0, 1, 2, 3, 4, 5, 6, 7, 3 + 16, 4 + 16, 3 + 32, 4 + 32, 5 + 16 + 32, 3 + 64]


@pytest.fixture
def spmm_variant():
    yield ops.set_spmm_variant
    ops.set_spmm_variant(0)


@pytest.mark.parametrize("K", [128, 256, 384, 512])
@pytest.mark.parametrize("variant", BULK_VARIANTS)
def test_spmm_bulk_variants_hubs_stats_bias(K, variant, spmm_variant):
    """Every SpMM kernel family on a graph with a 12k hub, a 700-edge row, empty rows and runs that cross the 32-edge
    windows; forward, fused bias + per-CTA column statistics, mean reduction; bitwise repeatable."""
    n = 20_000
    g = torch.Generator().manual_seed(11)
    hub_nbrs = torch.randperm(n, generator=g)[:12_345]
    mid_nbrs = torch.randperm(n, generator=g)[:700]
    row = torch.cat([torch.full((12_345,), 7), torch.full((700,), 4000), torch.randint(100, n - 50, (150_000,), generator=g)])
    col = torch.cat([hub_nbrs, mid_nbrs, torch.randint(0, n, (150_000,), generator=g)])
    r, c, _ = og.coalesce(row.numpy(), col.numpy(), n)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    val = torch.rand(r.numel(), generator=g)
    x, bias = torch.randn(n, K, generator=g), torch.randn(K, generator=g)
    adj = make_adj(r, c, n, n, val)
    G = adj.storage.engine_csr()
    Gu = adj.set_value(None).storage.engine_csr_unweighted()
    spmm_variant(variant)
    ref = oo.spmm_scatter(r, c, val.double(), x.double(), n, "sum") + bias.double()
    part = torch.full((ops.stat_slots(G), 2, K), float("nan"), device="cuda")
    out = ops.spmm_csr(G, x.cuda(), "sum", bias=bias.cuda(), stat_partial=part)
    assert rel_err(out, ref) < TOL and fro_err(out, ref) < TOL
    s = part.double().sum(0).cpu()
    assert rel_err(s[0], ref.sum(0)) < TOL and rel_err(s[1], (ref * ref).sum(0)) < TOL
    part2 = torch.empty_like(part)
    out2 = ops.spmm_csr(G, x.cuda(), "sum", bias=bias.cuda(), stat_partial=part2)
    assert torch.equal(out, out2) and torch.equal(part, part2)
    refm = oo.spmm_scatter(r, c, None, x.double(), n, "mean")
    outm = ops.spmm_csr(Gu, x.cuda(), "mean")
    assert rel_err(outm, refm) < TOL
    assert torch.count_nonzero(outm[:7]) == 0            # empty rows -> exactly 0
    assert rel_err(outm[7], refm[7]) < TOL and rel_err(outm[4000], refm[4000]) < TOL


@pytest.mark.parametrize("variant", [3, 4, 4 + 16, 6, 7])
def test_spmm_bulk_tiny_and_ragged(variant, spmm_variant):
    """Degenerate shapes on the bulk kernel: a single edge, rows of degree exactly G / ring depth, a graph smaller than one
    chunk, and a rectangular matrix whose sources are never referenced beyond n_src."""
    spmm_variant(variant)
    K = 256
    g = torch.Generator().manual_seed(12)
    for n_rows, n_cols, degs in [(1, 1, [1]), (5, 9, [0, 1, 0, 9, 2]), (40, 64, [4] * 8 + [8] * 8 + [16] * 8 + [0] * 8 + [33] * 8)]:
        row = torch.cat([torch.full((d,), i) for i, d in enumerate(degs)]).long()
        col = torch.cat([torch.randperm(n_cols, generator=g)[:d].sort().values for d in degs]).long()
        x = torch.randn(n_cols, K, generator=g)
        val = torch.rand(row.numel(), generator=g)
        ref = oo.spmm_scatter(row, col, val.double(), x.double(), n_rows, "sum")
        out = make_adj(row, col, n_rows, n_cols, val).matmul(x.cuda(), "sum")
        assert rel_err(out, ref) < TOL


@pytest.mark.parametrize("K", [8, 16, 32, 40, 64])
def test_spmm_narrow_deep_pipeline_variant(K, spmm_variant):
    """variant +128: the multi-row-per-warp narrow kernel with 8 instead of 4 gathers in flight per lane group (the widths the
    multi-GPU engine's column slices and the 40 logits use): identical results, hub rows and ragged tails included."""
    n = 20_000
    g = torch.Generator().manual_seed(K)
    row = torch.cat([torch.full((9000,), 5), torch.randint(0, n, (120_000,), generator=g)])
    col = torch.cat([torch.randperm(n, generator=g)[:9000], torch.randint(0, n, (120_000,), generator=g)])
    r, c, _ = og.coalesce(row.numpy(), col.numpy(), n)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    val = torch.rand(r.numel(), generator=g)
    x = torch.randn(n, K, generator=g)
    G = make_adj(r, c, n, n, val).storage.engine_csr()
    ref = oo.spmm_scatter(r, c, val.double(), x.double(), n, "sum")
    spmm_variant(0)
    a = ops.spmm_csr(G, x.cuda(), "sum")
    spmm_variant(128)
    b = ops.spmm_csr(G, x.cuda(), "sum")
    assert rel_err(a, ref) < TOL and rel_err(b, ref) < TOL
