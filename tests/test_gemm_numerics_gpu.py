"""Accuracy contract of the 3xTF32 GEMMs (gemm_tf32x3.cu, gemm_wgrad_tf32x3.cu), checked against float64 products of the
same fp32 operands (DESIGN.md §2):

* the tf32 split is bit-exact round-to-nearest (ties away from zero);
* every output element is within a worst-case bound beta(K) * (|A|·|B|^T)_ij derived from the algorithm below, with rows
  and columns scaled over 2^±20 so that small rows weigh as much as large ones;
* the accumulation is unbiased up to a small, K-independent mean (all-positive operands);
* the kernels read only the logical matrices and write only the logical output (NaN-poisoned views, NaN canaries);
* the call sequences of the chunked G-CRD loss and of the RGCN hold the same bound.

Every threshold is either derived in a comment or quotes the H100 measurement it was set from."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import lib, ops, rgcn

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# ----------------------------------------------------------------------------------------------------------- error model
# Per product a·b the kernels compute a_hi·b_hi + a_lo·b_hi + a_hi·b_lo with x_hi = rna_tf32(x), x_lo = rna_tf32(x - x_hi):
#   |x - x_hi| <= 2^-11 |x| and x_lo keeps 11 significant bits of it, so |x - x_hi - x_lo| <= 2^-11 |x - x_hi| <= 2^-22 |x|;
#   the two split residuals and the dropped a_lo·b_lo (<= 2^-22 |ab|) give <= 3·2^-22 |ab| (+ O(2^-32), covered by 3.01).
# The products of tf32 operands are exact in fp32.  One pipeline stage covers 32 of K in 12 wgmma k8 instructions into a
# fresh accumulator, which truncates: a k8 wgmma aligns the accumulator and its 8 products to the largest exponent and
# truncates, so it errs by at most (8 + 1 + 1)·2^-23 of the stage's sum S = sum |a||b| over its 32 K-indices (8 products and the
# accumulator aligned, the result truncated).  The 4 wgmmas of the large terms give 40·2^-23 S; the 8 of the small terms
# work on values <= 2^-10 S and give < 2^-23 S: 41·2^-23 per stage, i.e. of sum |a||b| over all K.  Then ceil(K/32)
# round-to-nearest additions of the stage results into the fp32 sum, each <= 2^-24 of sum |a||b|.
# Measured on an H100 80GB HBM3 at a 400 W power limit, the worst element of a random-sign GEMM uses 7.5% of this bound at
# K = 4, 1.4% at K = 256 and 0.15% at K = 16384.
U = 2.0 ** -24                                       # unit roundoff of fp32 round to nearest


def beta(k_stages_of_32: int, extra_adds: int = 0) -> float:
    """Worst-case relative bound of |C - C64| / (|A|·|B|^T) for a contraction of `k_stages_of_32` pipeline stages
    (+ `extra_adds` further round-to-nearest fp32 additions of partial sums, e.g. the weight gradient's split-K reduction)."""
    return 3.01 * 2.0 ** -22 + 41 * 2.0 ** -23 + (k_stages_of_32 + extra_adds) * U


def beta_k(K: int) -> float:
    return beta(-(-K // 32))


# The epilogue adds the bias and, when accumulating, the previous C with round-to-nearest: <= 2^-24 of each sum's magnitude.
# Bound them together by 2^-23 (|A|·|B|^T + |bias| + |C_in|).
EPI = 2.0 ** -23

CANARY = 0x7FC0DEAD                                   # a quiet NaN with a payload: outside a view it must survive bit for bit


def _poisoned(rows: int, cols: int) -> torch.Tensor:
    return torch.full((rows, cols), CANARY, dtype=torch.int32, device="cuda").view(torch.float32)


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def _pow2(n: int, g: torch.Generator, span: int = 20) -> torch.Tensor:
    """n powers of two 2^e, e uniform in [-span, span]: scaling by them is exact."""
    return torch.exp2(torch.randint(-span, span + 1, (n,), generator=g, device="cuda").double()).float()


def _scaled(m: int, k: int, g: torch.Generator) -> torch.Tensor:
    return torch.randn(m, k, generator=g, device="cuda") * _pow2(m, g)[:, None]


def _bound_ratio(c: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |c - ref| / bound (<= 1 passes); c fp32, ref / bound fp64, all on the GPU.  An element whose bound is 0 (every
    product of its dot product exactly zero, e.g. a dropped or ReLU-zero row of an activation) must equal ref exactly."""
    assert bool(torch.isfinite(c).all()), "non-finite output"
    err = (c.double() - ref).abs()
    return float(torch.where(bound > 0, err / bound, torch.where(err > 0, torch.inf, 0.0)).max())


def _gemm_check(a, b, c, beta_, bias=None, c_in=None):
    """c (fp32) vs fp64 a·b^T (+bias) (+c_in): ratio to the bound beta_·(|a|·|b|^T) + epilogue terms."""
    a64, b64 = a.double(), b.double()
    ref = a64 @ b64.t()
    mag = a64.abs() @ b64.abs().t()
    bound = beta_ * mag
    epi = torch.zeros_like(mag)
    if bias is not None:
        ref += bias.double()
        epi += bias.double().abs()
    if c_in is not None:
        ref += c_in.double()
        epi += c_in.double().abs()
    if bias is not None or c_in is not None:
        bound += EPI * (mag + epi)
    return _bound_ratio(c, ref, bound)


# ------------------------------------------------------------------------------------------------------ 1. the tf32 split
def _rna_bits(b: np.ndarray) -> np.ndarray:
    """Round the magnitude of fp32 bit patterns to 10 mantissa bits, ties away from zero (integer arithmetic)."""
    sign = b & np.uint32(0x80000000)
    mag = b & np.uint32(0x7FFFFFFF)
    mag = ((mag + np.uint32(0x1000)) >> np.uint32(13)) << np.uint32(13)      # a carry moves into the exponent, as it should
    return sign | mag


def _split_ref(x: np.ndarray):
    """(hi, lo) bit patterns.  x - hi is exact in fp32: hi and x are multiples of ulp(x) and |x - hi| <= 2^12 ulp(x)."""
    hi = _rna_bits(x.view(np.uint32))
    r = (x - hi.view(np.float32)).astype(np.float32)
    return hi, _rna_bits(r.view(np.uint32))


def _crafted_bits() -> np.ndarray:
    # Finite |x| >= 0x7F7FF000 rounds to inf (as cvt.rna.tf32.f32 does) and is outside the GEMM's contract: not tested.
    out = []
    for top in (0x3F800000, 0x3FAAA000, 0x4B7FE000, 0x0D3C6000, 0x72000000, 0x7F7FC000, 0x00800000, 0x00002000):
        low = np.arange(0x2000, dtype=np.uint32)                 # every pattern of the 13 dropped bits: the ties of hi and of lo
        out.append(np.uint32(top) | low)
    special = [0x00000000, 0x00000001, 0x00000FFF, 0x00001000, 0x00001001, 0x00001FFF, 0x00003000, 0x007FF000, 0x007FEFFF,
               0x007FFFFF, 0x00800FFF, 0x3FFFF000, 0x3FFFEFFF, 0x3FFFF001, 0x3F7FF000, 0x7F7FEFFF, 0x7F7FE000, 0x7F7FE001,
               0x7F7FEFFE, 0x7F7FDFFF, 0x3F801000, 0x3F803000, 0x3F800FFF, 0x3F802FFF]
    out.append(np.array(special, dtype=np.uint32))
    pos = np.concatenate(out)
    return np.concatenate([pos, pos | np.uint32(0x80000000)])   # and the negatives (-0 included)


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("shape", ["crafted", "large"])
def test_split_is_bitexact_round_to_nearest(transpose, shape):
    if shape == "crafted":
        bits = _crafted_bits()
        cols = 256
        bits = np.concatenate([bits, np.zeros((-len(bits)) % cols, dtype=np.uint32)]).reshape(-1, cols)
    else:
        # more elements than the capped grid covers in one sweep (132·8 blocks of 256): the grid-stride loop
        rng = np.random.default_rng(7)
        bits = rng.integers(0, 0x7F7FF000, size=(640, 1000), dtype=np.uint32)
        bits |= rng.integers(0, 2, size=bits.shape, dtype=np.uint32) << np.uint32(31)
    x = bits.view(np.float32)
    hi_ref, lo_ref = _split_ref(x)
    w = torch.from_numpy(x.copy()).cuda()
    hi, lo = ops.split_tf32(w, transpose=transpose)
    torch.cuda.synchronize()
    hi_b = hi.cpu().view(torch.int32).numpy().view(np.uint32)
    lo_b = lo.cpu().view(torch.int32).numpy().view(np.uint32)
    if transpose:
        hi_b, lo_b = hi_b.T, lo_b.T
    bad_hi, bad_lo = np.flatnonzero(hi_b != hi_ref), np.flatnonzero(lo_b != lo_ref)
    assert bad_hi.size == 0, [hex(int(v)) for v in bits.reshape(-1)[bad_hi[:8]]]
    assert bad_lo.size == 0, [hex(int(v)) for v in bits.reshape(-1)[bad_lo[:8]]]


# ------------------------------------------------------------------------------------- 2. elementwise error bound (GEMM)
GEMM_K = (4, 8, 28, 36, 256, 4096, 16384)
GEMM_M = (1, 4, 127, 128, 129, 3001)


@pytest.mark.parametrize("N", [1, 40, 48, 49, 128, 256, 349])
def test_gemm_elementwise_bound(N):
    """Both tile configurations (N <= 48: Cfg<48,4>), the ragged epilogue (N % 4 != 0 or a partial 32-column chunk),
    M and K tails, bias and accumulate into a random C."""
    worst = {}
    for K in GEMM_K:
        for M in GEMM_M:
            g = _gen(1000 * N + 10 * K + M)
            a, b = _scaled(M, K, g), _scaled(N, K, g)
            cs = _pow2(N, g)
            bias = torch.randn(N, generator=g, device="cuda") * cs
            c_in = torch.randn(M, N, generator=g, device="cuda") * cs * a.abs().max(1).values[:, None]
            hi, lo = ops.split_tf32(b)
            r_plain = _gemm_check(a, b, ops.gemm_tf32x3(a, hi, lo), beta_k(K))
            r_bias = _gemm_check(a, b, ops.gemm_tf32x3(a, hi, lo, bias), beta_k(K), bias=bias)
            c = c_in.clone()
            ops.gemm_tf32x3(a, hi, lo, out=c, accumulate=True)
            r_acc = _gemm_check(a, b, c, beta_k(K), c_in=c_in)
            worst[(M, K)] = max(r_plain, r_bias, r_acc)
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


WGRAD_NN = (7, 32, 33, 1000, 4099, 40_001, 169_343)
WGRAD_SHAPES = [(kin, nout) for kin in (128, 256) for nout in (4, 40, 132, 256)]


def _wgrad_beta(nn_: int) -> float:
    # node blocks of 32 are the stages; the split-K partials (at most 132 node ranges) are then added in a fixed order
    return beta(-(-nn_ // 32), extra_adds=132)


@pytest.mark.parametrize("Kin,Nout", WGRAD_SHAPES)
def test_wgrad_elementwise_bound(Kin, Nout):
    worst = {}
    for nn_ in WGRAD_NN:
        g = _gen(7 * nn_ + Kin + Nout)
        x = torch.randn(nn_, Kin, generator=g, device="cuda") * _pow2(Kin, g)[None, :]
        d = torch.randn(nn_, Nout, generator=g, device="cuda") * _pow2(Nout, g)[None, :]
        out = ops.gemm_wgrad_tf32x3(x, d)
        worst[nn_] = _gemm_check(x.t(), d.t(), out, _wgrad_beta(nn_))
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


def _ratio_rms(c: torch.Tensor, x: torch.Tensor, d: torch.Tensor) -> float:
    x64, d64 = x.double(), d.double()
    e = (c.double() - x64.t() @ d64).abs() / (x64.t().abs() @ d64.abs())
    return float(e.pow(2).mean().sqrt())


# RMS(ours) / RMS(CPU fp32) measured on an H100 80GB HBM3 at a 400 W power limit: 0.51 (Nn = 1000), 0.53 (Nn = 169,343).
WGRAD_RMS_FACTOR = 1.0


@pytest.mark.parametrize("nn_", [1000, 169_343])
def test_wgrad_error_rms_like_fp32(nn_):
    """Typical (not worst-case) error: the RMS of |C - C64| / (|X|^T·|G|) is within a small factor of what fp32 torch.mm on the
    CPU achieves on the same operands."""
    g = torch.Generator().manual_seed(nn_)
    x, d = torch.randn(nn_, 128, generator=g), torch.randn(nn_, 40, generator=g)
    ours = _ratio_rms(ops.gemm_wgrad_tf32x3(x.cuda(), d.cuda()).cpu(), x, d)
    cpu = _ratio_rms(x.t() @ d, x, d)
    assert ours < WGRAD_RMS_FACTOR * cpu, (ours, cpu)


# ------------------------------------------------------------------------------------------- 3. unbiased accumulation
def _mean_signed_rel(c: torch.Tensor, ref: torch.Tensor) -> float:
    return float(((c.double() - ref) / ref).mean())


# Mean signed relative error with all-positive operands (uniform in [0.01, 1.01)), measured on an H100 80GB HBM3 at a
# 400 W power limit:
#   GEMM  M = 4096, N = 256:  K = 32 / 256 / 1024 / 4096 / 16384  ->  -1.2016e-7 / -1.1951e-7 / -1.1985e-7 / -1.1978e-7 / -1.1960e-7
#   wgrad Kin = Nout = 256:   Nn = 2000 / 20000 / 169343           ->  -1.1939e-7 / -1.2001e-7 / -1.1922e-7
# The spread over K (resp. the node count) is below 1e-9: the mean does not grow.  For scale: cuBLAS TF32, one tensor-core
# chain over all of K, ends low by 1.4e-6 at K = 256 and 5.5e-5 at K = 65536 (BENCH.md).
BIAS_LO, BIAS_HI = -1.3e-7, -1.1e-7      # every mean lies in [BIAS_LO, BIAS_HI]
BIAS_SPREAD = 5e-9                       # max - min of the means over K (resp. the node count)


def test_gemm_accumulation_unbiased():
    means = {}
    for K in (32, 256, 1024, 4096, 16384):
        g = _gen(K)
        a = torch.rand(4096, K, generator=g, device="cuda") + 0.01
        b = torch.rand(256, K, generator=g, device="cuda") + 0.01
        c = ops.gemm_tf32x3(a, *ops.split_tf32(b))
        means[K] = _mean_signed_rel(c, a.double() @ b.double().t())
        del a, b, c
    vals = list(means.values())
    assert all(BIAS_LO <= m <= BIAS_HI for m in vals), means
    assert max(vals) - min(vals) <= BIAS_SPREAD, means


def test_wgrad_accumulation_unbiased():
    means = {}
    for nn_ in (2000, 20_000, 169_343):
        g = _gen(nn_)
        x = torch.rand(nn_, 256, generator=g, device="cuda") + 0.01
        d = torch.rand(nn_, 256, generator=g, device="cuda") + 0.01
        means[nn_] = _mean_signed_rel(ops.gemm_wgrad_tf32x3(x, d), x.double().t() @ d.double())
    vals = list(means.values())
    assert all(BIAS_LO <= m <= BIAS_HI for m in vals), means
    assert max(vals) - min(vals) <= BIAS_SPREAD, means


# --------------------------------------------------------------------------------- 4. poisoned views and output canaries
def _view(buf: torch.Tensor, r0: int, c0: int, rows: int, cols: int) -> torch.Tensor:
    return buf[r0:r0 + rows, c0:c0 + cols]


def _outside_is_canary(buf: torch.Tensor, view_mask: torch.Tensor) -> bool:
    bits = buf.view(torch.int32)
    return bool((bits[~view_mask] == CANARY).all())


def _mask_of(buf: torch.Tensor, r0: int, c0: int, rows: int, cols: int) -> torch.Tensor:
    m = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
    m[r0:r0 + rows, c0:c0 + cols] = True
    return m


def _poisoned_operand(vals: torch.Tensor, r0: int = 3, c0: int = 4, extra_rows: int = 131, extra_cols: int = 12) -> torch.Tensor:
    """vals placed at (r0, c0) of a NaN buffer with extra rows below and a wider row pitch (16-byte aligned start)."""
    rows, cols = vals.shape
    buf = _poisoned(r0 + rows + extra_rows, c0 + cols + extra_cols)
    v = _view(buf, r0, c0, rows, cols)
    v.copy_(vals)
    return v


@pytest.mark.parametrize("M,N,K", [(300, 349, 36), (129, 40, 28), (1000, 256, 100), (4, 48, 4), (257, 128, 4100), (131, 1, 8)])
@pytest.mark.parametrize("c_off", [0, 1])
@pytest.mark.parametrize("mode", ["plain", "bias", "accumulate"])
def test_gemm_poisoned_views(M, N, K, c_off, mode):
    """A, B_hi, B_lo as views with NaN around them (lda, ldb > K, rows past M / N); C a view at a row offset with ldc > N,
    c_off = 1 makes it 16-byte misaligned (the ragged epilogue for every chunk).  Outside C stays NaN bit for bit."""
    g = _gen(M + N + K + c_off)
    a, b = _scaled(M, K, g), _scaled(N, K, g)
    bias = torch.randn(N, generator=g, device="cuda") if mode == "bias" else None
    hi, lo = ops.split_tf32(b)
    av, hv, lv = _poisoned_operand(a), _poisoned_operand(hi), _poisoned_operand(lo)
    cbuf = _poisoned(M + 9, c_off + (N + 8) // 4 * 4)                # c_off = 0: ldc % 4 == 0, the vector stores
    r0 = 5
    cv = _view(cbuf, r0, c_off, M, N)
    c_in = None
    if mode == "accumulate":
        c_in = torch.randn(M, N, generator=g, device="cuda") * a.abs().max(1).values[:, None]
        cv.copy_(c_in)
    L, st = lib.load(), lib.stream_ptr()
    if mode == "accumulate":
        rc = L.b200gnn_gemm_tf32x3_acc_f32(av.data_ptr(), av.stride(0), hv.data_ptr(), lv.data_ptr(), hv.stride(0),
                                           cv.data_ptr(), cv.stride(0), M, N, K, st)
    else:
        rc = L.b200gnn_gemm_tf32x3_f32(av.data_ptr(), av.stride(0), hv.data_ptr(), lv.data_ptr(), hv.stride(0),
                                       cv.data_ptr(), cv.stride(0), M, N, K, bias.data_ptr() if bias is not None else None, st)
    lib.check(rc, "gemm")
    torch.cuda.synchronize()
    assert _gemm_check(a, b, cv, beta_k(K), bias=bias, c_in=c_in) <= 1.0
    assert _outside_is_canary(cbuf, _mask_of(cbuf, r0, c_off, M, N))


@pytest.mark.parametrize("Nn", [7, 1000, 40_001])
@pytest.mark.parametrize("Kin,Nout", [(128, 4), (256, 40), (128, 132), (256, 256)])
def test_wgrad_poisoned_views(Nn, Kin, Nout):
    """X and G as views with NaN rows past Nn and NaN columns past Kin / Nout (ldx, ldg > width); dW inside a NaN buffer;
    a NaN-filled workspace.  dW is correct and nothing outside it is written."""
    g = _gen(Nn + Kin + Nout)
    x = torch.randn(Nn, Kin, generator=g, device="cuda") * _pow2(Kin, g)[None, :]
    d = torch.randn(Nn, Nout, generator=g, device="cuda") * _pow2(Nout, g)[None, :]
    xv = _poisoned_operand(x, r0=2, c0=4, extra_rows=37, extra_cols=8)
    dv = _poisoned_operand(d, r0=2, c0=0, extra_rows=37, extra_cols=8)
    wbuf = _poisoned(1, Kin * Nout + 64).view(-1)
    dw = wbuf[32:32 + Kin * Nout].view(Kin, Nout)
    ws = _poisoned(1, ops.wgrad_workspace_floats(Kin, Nout)).view(-1)
    L = lib.load()
    lib.check(L.b200gnn_gemm_wgrad_tf32x3_f32(xv.data_ptr(), xv.stride(0), dv.data_ptr(), dv.stride(0), dw.data_ptr(), Nn,
                                              Kin, Nout, ws.data_ptr(), lib.stream_ptr()), "wgrad")
    torch.cuda.synchronize()
    assert _gemm_check(x.t(), d.t(), dw, _wgrad_beta(Nn)) <= 1.0
    inside = torch.zeros(wbuf.shape, dtype=torch.bool, device="cuda")
    inside[32:32 + Kin * Nout] = True
    assert _outside_is_canary(wbuf, inside)


@pytest.mark.parametrize("M,N,K", [(1003, 256, 40), (300, 128, 200), (129, 64, 36)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_stats_epilogue_poisoned(M, N, K, accumulate):
    """Statistics epilogue: A with NaN rows past M, C with NaN rows past M and NaN columns past N; C correct, the NaN-filled
    partial buffer fully overwritten with finite, correct column sums; the canaries intact."""
    g = _gen(M * N + K)
    a, b = _scaled(M, K, g), torch.randn(N, K, generator=g, device="cuda")
    bias = None if accumulate else torch.randn(N, generator=g, device="cuda")
    hi, lo = ops.split_tf32(b)
    av = _poisoned_operand(a)
    cbuf = _poisoned(M + 40, N + 8)
    cv = _view(cbuf, 0, 0, M, N)
    c_in = None
    if accumulate:
        c_in = torch.randn(M, N, generator=g, device="cuda") * a.abs().max(1).values[:, None]
        cv.copy_(c_in)
    slots = ops.gemm_stat_slots(M, N)
    part = _poisoned(slots, 2 * N)
    lib.check(lib.load().b200gnn_gemm_tf32x3_stats_f32(
        av.data_ptr(), av.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0), cv.data_ptr(), cv.stride(0), M, N, K,
        bias.data_ptr() if bias is not None else None, int(accumulate), part.data_ptr(), slots, lib.stream_ptr()), "stats")
    torch.cuda.synchronize()
    assert _gemm_check(a, b, cv, beta_k(K), bias=bias, c_in=c_in) <= 1.0
    assert _outside_is_canary(cbuf, _mask_of(cbuf, 0, 0, M, N))
    assert bool(torch.isfinite(part).all())
    c64 = cv.double()
    s = part.view(slots, 2, N).double().sum(0)
    assert rel_err(s, torch.stack([c64.sum(0), (c64 ** 2).sum(0)])) < 1e-6


@pytest.mark.parametrize("M,N,K", [(1003, 256, 40), (301, 128, 200)])
@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_bnbwd_epilogue_poisoned(M, N, K, variant, accumulate):
    """BatchNorm-backward epilogue through both paths (1: Xout / Y staged by TMA, 2: register loads): A, C, Xout and Y with
    NaN rows past M and NaN columns past N.  dz bit-identical to the plain GEMM followed by the mask, the partial sums finite
    and correct, rows past M of C still NaN."""
    g = _gen(M + N + K + variant)
    p = 0.5
    a, b = _scaled(M, K, g), torch.randn(N, K, generator=g, device="cuda")
    y = torch.randn(M, N, generator=g, device="cuda")
    mean, invstd = y.mean(0), (y.var(0, unbiased=False) + 1e-5).rsqrt()
    keep = torch.rand(M, N, generator=g, device="cuda") >= p
    x_out = torch.relu((y - mean) * invstd) * keep / (1.0 - p)
    seed = torch.randn(M, N, generator=g, device="cuda") * a.abs().max(1).values[:, None]
    hi, lo = ops.split_tf32(b)
    plain = seed.clone() if accumulate else torch.empty(M, N, device="cuda")
    ops.gemm_tf32x3(a, hi, lo, out=plain, accumulate=accumulate)
    assert _gemm_check(a, b, plain, beta_k(K), c_in=seed if accumulate else None) <= 1.0
    av = _poisoned_operand(a)
    bufs = [_poisoned(M + 40, N + 8) for _ in range(3)]
    cv, xv, yv = (_view(t, 0, 0, M, N) for t in bufs)
    xv.copy_(x_out)
    yv.copy_(y)
    if accumulate:
        cv.copy_(seed)
    slots = ops.gemm_stat_slots(M, N)
    part = _poisoned(slots, 2 * N)
    L = lib.load()
    L.b200gnn_gemm_set_bnbwd_variant(variant)
    try:
        lib.check(L.b200gnn_gemm_tf32x3_bnbwd_f32(
            av.data_ptr(), av.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0), cv.data_ptr(), cv.stride(0), M, N, K,
            int(accumulate), xv.data_ptr(), yv.data_ptr(), mean.data_ptr(), invstd.data_ptr(), p, part.data_ptr(), slots,
            lib.stream_ptr()), "bnbwd")
        torch.cuda.synchronize()
    finally:
        L.b200gnn_gemm_set_bnbwd_variant(0)
    dz = torch.where(x_out > 0, plain * (1.0 / (1.0 - p)), torch.zeros_like(plain))
    assert torch.equal(cv, dz)
    assert _outside_is_canary(bufs[0], _mask_of(bufs[0], 0, 0, M, N))
    assert bool(torch.isfinite(part).all())
    xhat = (y.double() - mean.double()) * invstd.double()
    sums = torch.stack([dz.double().sum(0), (dz.double() * xhat).sum(0)])
    assert rel_err(part.view(slots, 2, N).double().sum(0), sums) < 1e-6


# ---------------------------------------------------------------------------------------- 5. the callers' call sequences
def test_nce_chunk_loop_products():
    """The chunk loop of criterion._NCE at S = 16384, F = 256 with R = 1820: nine full chunks and a last chunk of 4 rows.
    Each chunk's three products — Z_c = xs_c·xt^T (K = F), d fs_c = dZ_c·xt (K = S), d ft += dZ_c^T·xs_c (K = R or 4,
    accumulating) — against fp64 of the same fp32 operands."""
    S, F, R = 16384, 256, 1820
    assert S % R == 4
    g = _gen(16384)
    xs = torch.nn.functional.normalize(torch.randn(S, F, generator=g, device="cuda"), dim=1) / 0.07
    xt = torch.nn.functional.normalize(torch.randn(S, F, generator=g, device="cuda"), dim=1)
    L, st = lib.load(), lib.stream_ptr()
    xt_hi, xt_lo = ops.split_tf32(xt)
    xtT_hi, xtT_lo = ops.split_tf32(xt, transpose=True)
    g_s = torch.empty(S, F, device="cuda")
    g_t = torch.zeros(S, F, device="cuda")
    Z, Zt = torch.empty(R, S, device="cuda"), torch.empty(S * R, device="cuda")
    part = torch.empty(S, device="cuda")
    worst = {}
    for r0 in range(0, S, R):
        r = min(R, S - r0)
        Zc = Z[:r]
        ops.gemm_tf32x3(xs[r0:r0 + r], xt_hi, xt_lo, out=Zc)
        worst[(r0, "Z")] = _gemm_check(xs[r0:r0 + r], xt, Zc, beta_k(F))
        lib.check(L.b200gnn_nce_rows_chunk_f32(Zc.data_ptr(), S, r, S, r0, part.data_ptr(), st), "nce_rows_chunk_f32")
        dZ = Zc.clone()
        ops.gemm_tf32x3(Zc, xtT_hi, xtT_lo, out=g_s[r0:r0 + r])
        worst[(r0, "dfs")] = _gemm_check(dZ, xt.t(), g_s[r0:r0 + r], beta_k(S))
        Ztc = Zt[:S * r].view(S, r)
        lib.check(L.b200gnn_transpose_f32(Zc.data_ptr(), r, S, Ztc.data_ptr(), st), "transpose_f32")
        assert torch.equal(Ztc, dZ.t())
        hi, lo = ops.split_tf32(xs[r0:r0 + r], transpose=True)
        before = g_t.clone()
        ops.gemm_tf32x3(Ztc, hi, lo, out=g_t, accumulate=True)
        worst[(r0, "dft")] = _gemm_check(Ztc, xs[r0:r0 + r].t(), g_t, beta_k(r), c_in=before)
    bad = {k: v for k, v in worst.items() if not v <= 1.0}
    assert not bad, bad


def test_rgcn_gemm_accumulates_into_349_classes():
    """rgcn.RGCNInference._gemm as the MAG model calls it: the root linear with bias into the [M, 349] output, then relation
    GEMMs accumulated into it, one with K not a multiple of 4 (zero-padded).  Every step against fp64."""
    M, N = 3001, 349
    g = _gen(349)
    out = torch.empty(M, N, device="cuda")
    x0, w0 = _scaled(M, 128, g), torch.randn(N, 128, generator=g, device="cuda")
    bias = torch.randn(N, generator=g, device="cuda")
    rgcn.RGCNInference._gemm(None, x0, w0, out, bias=bias)
    assert _gemm_check(x0, w0, out, beta_k(128), bias=bias) <= 1.0
    for k in (128, 129, 64):
        x, w = _scaled(M, k, g), torch.randn(N, k, generator=g, device="cuda")
        before = out.clone()
        rgcn.RGCNInference._gemm(None, x, w, out, accumulate=True)
        assert _gemm_check(x, w, out, beta_k(k), c_in=before) <= 1.0, k
