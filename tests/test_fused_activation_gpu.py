"""Hidden activations recomputed inside their consumers (packed dropout keep bits + Y + BatchNorm scale / shift) against
the materialised activation of affine_relu_dropout: every comparison is bit for bit."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = pytest.mark.gpu


def unpack(bits, K):
    """int32 [..., W] keep bits -> bool [..., 32 W] (column 32 w + b = bit b of word w)."""
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    return ((bits.unsqueeze(-1) >> sh) & 1).bool().flatten(-2)


def bits_for(n, K, p, seed, offset, n_layers=1):
    bits = torch.empty(n_layers, n, (K + 31) // 32, dtype=torch.int32, device="cuda")
    return ops.dropout_bits(bits, p, seed, offset, K=K)


def bn_operands(n, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    y = torch.randn(n, K, device="cuda", generator=g) * 2 + 0.3
    scale = torch.rand(K, device="cuda", generator=g) + 0.5
    shift = torch.randn(K, device="cuda", generator=g) * 0.5
    return y, scale, shift


@pytest.mark.parametrize("p", [0.5, 0.3])
@pytest.mark.parametrize("n,K", [(1001, 256), (777, 40), (513, 100)])
def test_keep_bits_match_dropout_mask(p, n, K):
    step = torch.tensor([5], dtype=torch.int32, device="cuda")
    bits = torch.full((2, n, (K + 31) // 32), -1, dtype=torch.int32, device="cuda")
    ops.dropout_bits(bits, p, 7, 3, step_dev=step, step_mul=2, K=K)
    u = unpack(bits, K)
    for l in range(2):
        mask = ops.dropout_mask(n, K, p, 7, 3 + l + 5 * 2).bool()
        assert torch.equal(u[l, :, :K], mask)
    assert not u[:, :, K:].any()


@pytest.mark.parametrize("p", [0.5, 0.3])
def test_affine_relu_bits_matches_affine_relu_dropout(p):
    n, K = 1001, 100
    y, scale, shift = bn_operands(n, K, 1)
    ref = ops.affine_relu_dropout(y, scale, shift, True, p, 11, 4)
    got = ops.affine_relu_bits(y, bits_for(n, K, p, 11, 4)[0], scale, shift, p)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("N", [40, 256])
@pytest.mark.parametrize("K", [64, 128, 256])
def test_act_gemm_matches_gemm_on_materialised_activation(N, K):
    M, p = 1000, 0.5
    y, scale, shift = bn_operands(M, K, 2)
    a = ops.affine_relu_dropout(y, scale, shift, True, p, 5, 1)
    w = torch.randn(K, N, device="cuda") / K ** 0.5
    bias = torch.randn(N, device="cuda")
    hi, lo = ops.split_tf32(w, transpose=True)
    ref = ops.gemm_tf32x3(a, hi, lo, bias=bias)
    got = ops.gemm_tf32x3_act(y, scale, shift, bits_for(M, K, p, 5, 1)[0], p, hi, lo, bias=bias)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("k_in,n_out", [(256, 256), (256, 40), (128, 256)])
def test_act_wgrad_matches_wgrad_on_materialised_activation(k_in, n_out):
    nn_, p = 3001, 0.5
    y, scale, shift = bn_operands(nn_, k_in, 3)
    a = ops.affine_relu_dropout(y, scale, shift, True, p, 9, 0)
    g = torch.randn(nn_, n_out, device="cuda")
    ref = ops.gemm_wgrad_tf32x3(a, g)
    got = ops.gemm_wgrad_tf32x3_act(y, scale, shift, bits_for(nn_, k_in, p, 9, 0)[0], p, g)
    assert torch.equal(got, ref)


@pytest.mark.parametrize("variant", [1, 2])          # the TMA-staged and the register epilogue
@pytest.mark.parametrize("K", [40, 256])
@pytest.mark.parametrize("accumulate", [False, True])
def test_bnbwd_bits_matches_bnbwd_xout(variant, K, accumulate):
    M, N, p = 1000, 256, 0.5
    y, scale, shift = bn_operands(M, N, 4)
    x_out = ops.affine_relu_dropout(y, scale, shift, True, p, 13, 2)
    mean, invstd = torch.randn(N, device="cuda"), torch.rand(N, device="cuda") + 0.5
    a = torch.randn(M, K, device="cuda")
    hi, lo = ops.split_tf32(torch.randn(N, K, device="cuda") / K ** 0.5)
    start = torch.randn(M, N, device="cuda")
    slots = ops.gemm_stat_slots(M, N)
    L = lib.load()
    try:
        L.b200gnn_gemm_set_bnbwd_variant(variant)
        out_ref, part_ref = start.clone(), torch.zeros(slots, 2, N, device="cuda")
        ops.gemm_tf32x3_bnbwd(a, hi, lo, out_ref, x_out, y, mean, invstd, p, part_ref, accumulate=accumulate)
        out, part = start.clone(), torch.zeros(slots, 2, N, device="cuda")
        ops.gemm_tf32x3_bnbwd_bits(a, hi, lo, out, bits_for(M, N, p, 13, 2)[0], y, mean, invstd, scale, shift, p, part,
                                   accumulate=accumulate)
    finally:
        L.b200gnn_gemm_set_bnbwd_variant(0)
    assert torch.equal(out, out_ref)
    assert torch.equal(part, part_ref)


def make_trainer(fuse, n=4000, e=30_000, dims=(128, 256, 256, 40)):
    ei = skewed_edges(n, e, 0)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    tr = GCNStudentTrainer(adj, list(dims), dropout=0.5, seed=0, fuse_activations=fuse)
    assert tr.fuse_act == fuse
    g = torch.Generator().manual_seed(9)
    x = torch.randn(n, dims[0], generator=g).cuda()
    y = torch.randint(0, dims[-1], (n,), generator=g).cuda()
    t = (torch.randn(n, dims[-1], generator=g) * 2).cuda()
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values.cuda()
    return tr, (x, y, idx, t)


@pytest.mark.parametrize("graph", [False, True])
def test_fused_engine_matches_unfused_engine(graph):
    runs = []
    for fuse in (False, True):
        tr, inputs = make_trainer(fuse)
        if graph:
            tr.capture(*inputs, warmup=1)
        losses = []
        for _ in range(3):
            losses.append((tr.replay() if graph else tr.train_step(*inputs)).clone())
        torch.cuda.synchronize()
        runs.append((tr, torch.stack(losses)))
    (ref, l_ref), (got, l_got) = runs
    assert torch.equal(l_got, l_ref)
    assert torch.equal(got.Y[-1], ref.Y[-1])
    assert torch.equal(got.grads, ref.grads)
    assert torch.equal(got.params, ref.params)
    for a, b in zip(got.A, ref.A):
        assert torch.equal(a, b)
    assert torch.equal(got.out_feat(), ref.out_feat())
