"""Producer kernels with the multi-GPU engine's layout exchange fused into their epilogue (hybrid.py), exercised on ONE GPU
with local destination buffers standing in for the peers': the scattered result must equal the plain kernel's output
re-arranged (bitwise — same arithmetic, different addresses)."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import ops
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = pytest.mark.gpu


def _offsets(n, world):
    base, rem = divmod(n, world)
    off = [0]
    for q in range(world):
        off.append(off[-1] + base + (1 if q < rem else 0))
    return off


@pytest.mark.parametrize("world,N,K", [(2, 256, 128), (4, 256, 256), (8, 256, 64)])
def test_gemm_epilogue_r2c_scatter(world, N, K):
    """b200gnn_gemm_tf32x3_scatter_f32: column block q of A·B^T lands in buffer q at rows row_off + m."""
    M, n_nodes, row_off = 1000, 5000, 777
    g = torch.Generator().manual_seed(0)
    a, b = torch.randn(M, K, generator=g).cuda(), torch.randn(N, K, generator=g).cuda()
    hi, lo = ops.split_tf32(b)
    ref = ops.gemm_tf32x3(a, hi, lo)
    kc = N // world
    dst = [torch.full((n_nodes, kc), float("nan"), device="cuda") for _ in range(world)]
    ops.gemm_tf32x3_scatter(a, hi, lo, [d.data_ptr() for d in dst], row_off)
    for q in range(world):
        assert torch.equal(dst[q][row_off:row_off + M], ref[:, q * kc:(q + 1) * kc])
        assert torch.isnan(dst[q][:row_off]).all() and torch.isnan(dst[q][row_off + M:]).all()


@pytest.mark.parametrize("world,K", [(2, 128), (4, 256), (8, 32), (8, 16), (2, 64), (2, 1152), (4, 2048)])
def test_spmm_epilogue_c2r_scatter(world, K):
    """b200gnn_spmm_csr_scatter_f32 on the TMA kernels (K % 128 == 0) and the narrow kernel, hub rows included: row i goes to
    the buffer of the rank owning it at (i - off[q], col_dst ...).  K = 1152 / 2048 (> 1024) finish the hub rows on the hub
    finalize's scalar path."""
    n = 20_000
    gen = torch.Generator().manual_seed(5)
    hub = torch.randperm(n, generator=gen)[:5000]
    row = torch.cat([torch.full((5000,), 3), torch.randint(0, n, (150_000,), generator=gen)])
    col = torch.cat([hub, torch.randint(0, n, (150_000,), generator=gen)])
    r, c, _ = og.coalesce(row.numpy(), col.numpy(), n)
    r, c = torch.from_numpy(r), torch.from_numpy(c)
    val = torch.rand(r.numel(), generator=gen)
    adj = SparseTensor(row=r.cuda(), col=c.cuda(), value=val.cuda(), sparse_sizes=(n, n), is_sorted=True)
    G = adj.storage.engine_csr()
    assert G.n_hub > 0
    x = torch.randn(n, K, generator=gen).cuda()
    bias = torch.randn(K, generator=gen).cuda()
    ref = ops.spmm_csr(G, x, "sum", bias=bias)
    off = _offsets(n, world)
    k_total, rank = K * world, world - 1
    block = max(off[q + 1] - off[q] for q in range(world))
    dst = [torch.full((block, k_total), float("nan"), device="cuda") for _ in range(world)]
    ops.spmm_csr_scatter(G, x, [d.data_ptr() for d in dst], off, k_total, rank * K, "sum", bias=bias)
    for q in range(world):
        rows = off[q + 1] - off[q]
        assert torch.equal(dst[q][:rows, rank * K:(rank + 1) * K], ref[off[q]:off[q + 1]])
        assert torch.isnan(dst[q][:rows, :rank * K]).all()


def test_activation_pass_c2r_scatter():
    n, kc, world = 9001, 32, 8
    K = kc * world
    g = torch.Generator().manual_seed(2)
    y = torch.randn(n, kc, generator=g).cuda()
    scale, shift = torch.rand(kc, generator=g).cuda() + 0.5, torch.randn(kc, generator=g).cuda()
    rowmap = torch.randperm(n, generator=g).to(torch.int32).cuda()
    rank = 3
    ref = ops.affine_relu_dropout_mapped(y, scale, shift, True, 0.5, 7, 1, rowmap=rowmap, k_global=K, col_offset=rank * kc)
    off = _offsets(n, world)
    block = max(off[q + 1] - off[q] for q in range(world))
    dst = [torch.full((block, K), float("nan"), device="cuda") for _ in range(world)]
    out = torch.empty_like(y)
    ops.affine_relu_dropout_scatter(y, scale, shift, True, 0.5, 7, 1, out, None, 0, rowmap, K, rank * kc,
                                    [d.data_ptr() for d in dst], off, K)
    assert torch.equal(out, ref)
    for q in range(world):
        rows = off[q + 1] - off[q]
        assert torch.equal(dst[q][:rows, rank * kc:(rank + 1) * kc], ref[off[q]:off[q + 1]])


@pytest.mark.parametrize("N,K", [(40, 256), (160, 64)])
def test_gemm_epilogue_row_allgather_broadcast(N, K):
    """b200gnn_gemm_tf32x3_bcast_f32: the [M, N] result lands in every destination buffer at rows row_off + m (narrow tile
    shape with its ragged last column chunk, and the wide one)."""
    M, n_nodes, row_off, world = 1500, 4000, 123, 4
    g = torch.Generator().manual_seed(1)
    a, b = torch.randn(M, K, generator=g).cuda(), torch.randn(N, K, generator=g).cuda()
    hi, lo = ops.split_tf32(b)
    ref = ops.gemm_tf32x3(a, hi, lo)
    dst = [torch.full((n_nodes, N), float("nan"), device="cuda") for _ in range(world)]
    ops.gemm_tf32x3_bcast(a, hi, lo, [d.data_ptr() for d in dst], row_off, N)
    for q in range(world):
        assert torch.equal(dst[q][row_off:row_off + M], ref)
        assert torch.isnan(dst[q][:row_off]).all() and torch.isnan(dst[q][row_off + M:]).all()
