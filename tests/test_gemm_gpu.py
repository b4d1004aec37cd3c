"""wgmma 3xTF32 GEMM (through the C ABI) vs fp64: fp32-level accuracy on the tensor cores."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(120)]


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (128, 128, 128), (1000, 256, 128), (5000, 256, 256), (777, 40, 256),
                                   (3000, 256, 40), (129, 130, 36), (20_000, 128, 750 // 2 * 2 + 2)])
@pytest.mark.parametrize("bias", [False, True])
def test_gemm_matches_fp64(M, N, K, bias):
    K = (K + 3) // 4 * 4
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g) if bias else None
    ref = a.double() @ w.double().t() + (b.double() if bias else 0)
    hi, lo = ops.split_tf32(w.cuda())
    assert torch.equal((hi.cpu().view(torch.int32) & 0x1FFF), torch.zeros(N, K, dtype=torch.int32))
    out = ops.gemm_tf32x3(a.cuda(), hi, lo, b.cuda() if bias else None)
    torch.cuda.synchronize()
    e = rel_err(out, ref)
    e32 = rel_err(a @ w.t() + (b if bias else 0), ref)      # what plain fp32 achieves on the CPU
    assert e < 1e-5, (e, e32)
    assert e < 20 * max(e32, 1e-7), (e, e32)


def test_split_transpose():
    w = torch.randn(96, 200, generator=torch.Generator().manual_seed(0))
    hi, lo = ops.split_tf32(w.cuda(), transpose=True)
    assert hi.shape == (200, 96)
    assert (hi.cpu().double() + lo.cpu().double() - w.t().double()).abs().max().item() < 2.0 ** -21 * w.abs().max().item()
    h2, l2 = ops.split_tf32(w.cuda())
    assert torch.equal(h2.t().contiguous(), hi)


def test_gemm_deterministic_and_reusable():
    g = torch.Generator().manual_seed(1)
    a, w = torch.randn(4000, 256, generator=g).cuda(), torch.randn(256, 256, generator=g).cuda()
    hi, lo = ops.split_tf32(w)
    o1 = ops.gemm_tf32x3(a, hi, lo)
    o2 = ops.gemm_tf32x3(a, hi, lo)
    assert torch.equal(o1, o2)


@pytest.mark.parametrize("Nn,Kin,Nout", [(16, 128, 32), (1000, 128, 256), (5003, 256, 256), (40_000, 256, 64), (7, 128, 128),
                                          (3000, 256, 40), (999, 128, 4), (2000, 256, 100)])
def test_wgrad_matches_fp64(Nn, Kin, Nout):
    g = torch.Generator().manual_seed(Nn + Kin + Nout)
    x = torch.randn(Nn, Kin, generator=g)
    d = torch.randn(Nn, Nout, generator=g)
    ref = x.double().t() @ d.double()
    out = ops.gemm_wgrad_tf32x3(x.cuda(), d.cuda())
    torch.cuda.synchronize()
    e, e32 = rel_err(out, ref), rel_err(x.t() @ d, ref)
    assert e < 1e-5, (e, e32)
    out2 = ops.gemm_wgrad_tf32x3(x.cuda(), d.cuda())
    assert torch.equal(out, out2)


def test_wgrad_unsupported_shapes_are_reported():
    from efficient_gnns_b200 import lib
    assert not ops.wgrad_supported(64, 40) and ops.wgrad_supported(128, 256) and ops.wgrad_supported(256, 40)
    with pytest.raises(lib.B200GnnError):
        ops.gemm_wgrad_tf32x3(torch.randn(100, 64, device="cuda"), torch.randn(100, 40, device="cuda"))


# ---------------------------------------------------------------- row passes fused into the epilogue (SURVEY §8 f1)
@pytest.mark.parametrize("M,N,K", [(128, 64, 32), (1000, 256, 128), (5003, 256, 256), (40_000, 128, 128), (19_001, 256, 40)])
def test_gemm_epilogue_statistics(M, N, K):
    """C and its BatchNorm batch statistics from one launch: C bit-identical to the plain GEMM, the column sums equal to a
    fp64 reduction of C (fixed slot order: run-to-run identical)."""
    g = torch.Generator().manual_seed(M + N)
    a = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    b = torch.randn(N, generator=g).cuda()
    hi, lo = ops.split_tf32(w)
    plain = ops.gemm_tf32x3(a, hi, lo, b)
    slots = ops.gemm_stat_slots(M, N)
    part = torch.full((slots, 2, N), float("nan"), device="cuda")
    out = torch.empty(M, N, device="cuda")
    ops.gemm_tf32x3_stats(a, hi, lo, b, out, part)
    assert torch.equal(out, plain)
    s = part.double().sum(0)
    ref = torch.stack([plain.double().sum(0), (plain.double() ** 2).sum(0)])
    assert rel_err(s, ref) < 1e-6
    part2 = torch.empty_like(part)
    ops.gemm_tf32x3_stats(a, hi, lo, b, out, part2)
    assert torch.equal(part, part2)
    # ... and through the BatchNorm finalize: mean / invstd as nn.BatchNorm1d computes them
    bn = ops.bn_finalize(part, M, torch.ones(N, device="cuda"), torch.zeros(N, device="cuda"), 1e-5, 0.1, None, None)
    assert (bn[0].double() - plain.double().mean(0)).abs().max().item() < 1e-6
    assert rel_err(bn[1], (plain.double().var(0, unbiased=False) + 1e-5).rsqrt()) < 1e-6


def test_gemm_epilogue_statistics_of_an_accumulated_output():
    """SAGEConv: Y = lin_l(mean) + lin_r(x) is two GEMMs into the same buffer; the second one reduces the statistics of the SUM."""
    g = torch.Generator().manual_seed(11)
    M, N, K = 7001, 128, 96
    a1, a2 = torch.randn(M, K, generator=g).cuda(), torch.randn(M, K, generator=g).cuda()
    w1, w2 = (torch.randn(N, K, generator=g) / K ** 0.5).cuda(), (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    b = torch.randn(N, generator=g).cuda()
    ref = ops.gemm_tf32x3(a1, *ops.split_tf32(w1), b)
    ops.gemm_tf32x3(a2, *ops.split_tf32(w2), out=ref, accumulate=True)
    out = ops.gemm_tf32x3(a1, *ops.split_tf32(w1), b)
    part = torch.empty(ops.gemm_stat_slots(M, N), 2, N, device="cuda")
    ops.gemm_tf32x3_stats(a2, *ops.split_tf32(w2), None, out, part, accumulate=True)
    assert torch.equal(out, ref)
    assert rel_err(part.double().sum(0), torch.stack([ref.double().sum(0), (ref.double() ** 2).sum(0)])) < 1e-6


@pytest.mark.parametrize("M,N,K", [(1000, 256, 40), (5003, 256, 256), (33_000, 128, 64), (2500, 64, 128), (41_111, 256, 40)])
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("variant", [0, 1, 2])
def test_gemm_epilogue_bn_backward(M, N, K, accumulate, p, variant):
    """Input-gradient GEMM + pass 1 of the BatchNorm/ReLU/dropout backward == plain GEMM followed by the two-pass kernels:
    dz stored, the column sums, and after the apply pass dY / dgamma / dbeta / dbias."""
    g = torch.Generator().manual_seed(M + N + K)
    a = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    y = torch.randn(M, N, generator=g).cuda()
    mean, invstd = y.mean(0), (y.var(0, unbiased=False) + 1e-5).rsqrt()
    gamma = (torch.rand(N, generator=g) + 0.5).cuda()
    keep = (torch.rand(M, N, generator=g) >= p).cuda()
    x_out = torch.relu((y - mean) * invstd * gamma) * keep / (1.0 - p)
    seed_grad = torch.randn(M, N, generator=g).cuda()
    hi, lo = ops.split_tf32(w)
    # unfused: GEMM, then the two-pass backward
    d_out = seed_grad.clone() if accumulate else torch.empty(M, N, device="cuda")
    ops.gemm_tf32x3(a, hi, lo, out=d_out, accumulate=accumulate)
    ref = ops.bn_act_bwd(d_out, x_out, y, mean, invstd, gamma, p)
    # fused
    dz = seed_grad.clone() if accumulate else torch.empty(M, N, device="cuda")
    part = torch.full((ops.gemm_stat_slots(M, N), 2, N), float("nan"), device="cuda")
    from efficient_gnns_b200 import lib
    lib.load().b200gnn_gemm_set_bnbwd_variant(variant)       # 0 automatic, 1: TMA-staged Xout / Y, 2: register path
    try:
        ops.gemm_tf32x3_bnbwd(a, hi, lo, dz, x_out, y, mean, invstd, p, part, accumulate=accumulate)
        torch.cuda.synchronize()
    finally:
        lib.load().b200gnn_gemm_set_bnbwd_variant(0)
    inv_keep = 1.0 / (1.0 - p)
    assert torch.equal(dz, torch.where(x_out > 0, d_out * inv_keep, torch.zeros_like(d_out)))
    xhat = (y.double() - mean.double()) * invstd.double()
    sums = torch.stack([dz.double().sum(0), (dz.double() * xhat).sum(0)])
    assert rel_err(part.double().sum(0), sums) < 1e-6
    d_y = torch.empty(M, N, device="cuda")
    dg, db, dbias = (torch.empty(N, device="cuda") for _ in range(3))
    ops.bn_act_bwd_apply(dz, None, y, mean, invstd, gamma, part, M, p, d_y, dg, db, dbias,
                         torch.empty(ops.rows_slots(M), 2, N, device="cuda"), torch.empty(3, N, device="cuda"))
    torch.cuda.synchronize()
    assert rel_err(d_y, ref[0]) < 2e-6
    assert rel_err(dg, ref[1]) < 2e-6 and rel_err(db, ref[2]) < 2e-6
    # dbias = column sums of dY, which cancel to zero analytically: both results are rounding noise of that cancellation
    noise = 4e-7 * d_y.abs().sum(0).max().item()
    assert (dbias - ref[3]).abs().max().item() < max(noise, 1e-4)


def test_gemm_epilogue_statistics_unsupported_shapes():
    a = torch.randn(256, 64, device="cuda")
    for n in (40, 100, 288):
        w = torch.randn(n, 64, device="cuda")
        hi, lo = ops.split_tf32(w)
        with pytest.raises(Exception):
            ops.gemm_tf32x3_stats(a, hi, lo, None, torch.empty(256, n, device="cuda"),
                                  torch.empty(ops.gemm_stat_slots(256, n), 2, n, device="cuda"))
