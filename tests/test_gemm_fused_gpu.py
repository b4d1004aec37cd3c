"""Accuracy contract of the fused-operand 3xTF32 GEMMs, through the C ABI (gemm_tf32x3.cu, gemm_wgrad_tf32x3.cu):

* b200gnn_gemm_tf32x3_act_f32 / _prelu_f32: the activation prologue (BatchNorm affine + ReLU, or PReLU, then dropout
  from packed keep bits) formed in registers from Y / Z;
* b200gnn_gemm_tf32x3_bnbwd_bits_f32: the BatchNorm-backward epilogue with its ReLU/dropout mask taken from keep bits;
* b200gnn_gemm_tf32x3_prelu_bwd_f32: the PReLU/dropout backward epilogue and its fp64 slope-gradient reduction;
* b200gnn_gemm_tf32x3_rowidx_f32: the row-indexed stores;
* b200gnn_gemm_wgrad_tf32x3_act_f32 / _prelu_f32: the weight gradients of those activations (PReLU on column blocks).

Every case has two independent oracles: bit-identity with the materialised twin (the pinned plain GEMM or weight gradient
on affine_relu_bits / prelu_bits of the same operands), and an fp64 bound against a restatement of the activation in
float64, so that a mistake shared by a kernel and its materialiser cannot hide.  The bound is beta(K) of
test_gemm_numerics_gpu.py plus the activation's own roundings (derived below).

The geometry tables reach what small shapes never do: CTAs that process two or more tiles (the keep words of the next
tile are prefetched in the last stage of the current one), both tile shapes, K off the 32-column grid with random
garbage in the keep bits past K, ragged N, misaligned C and ldc % 4 != 0 (the scalar epilogue), p = 0 with all-ones
bits (the eval forward), slopes of both signs, 0 and 1, and the weight gradient's node-range clamp.
tests/test_gemm_fused_geometry.py checks on the CPU that the tables keep reaching all of it.

Operands sit inside NaN buffers with wider pitches; outputs, workspaces and partials are NaN-filled inside canary
buffers whose canaries must survive bit for bit.  fmaxf(NaN, 0) = 0, so NaN poison in Y (or in scale / shift) cannot
show through the ReLU prologue: there a stray read is caught by the output canaries and by bit-identity with the twin,
not by a NaN in the result.  Refused calls must return their documented code and leave every output untouched."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import lib, ops
from test_gemm_numerics_gpu import (CANARY, EPI, U, _gemm_check, _gen, _mask_of, _outside_is_canary, _poisoned,
                                    _poisoned_operand, _pow2, _view, _wgrad_beta, beta_k)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

BAD_ARG, UNSUPPORTED = -1, -2

# ------------------------------------------------------------------------------------------------------- geometry
SMS = 132          # H100 SXM; the tables' multi-tile claims are made against it and checked against the device at run time


def gemm_tiles(M: int, N: int, narrow_ok: bool = True) -> int:
    """Output tiles of one launch: 128-row tiles, 48 columns wide for N <= 48 (Cfg<48, 6>) where the entry point has that
    shape (narrow_ok), else 128."""
    bn = 48 if narrow_ok and N <= 48 else 128
    return -(-M // 128) * -(-N // bn)


def wgrad_ranges(Nn: int, Kin: int, Nout: int, sms: int = SMS):
    """(node ranges before the clamp to the node-block count, node blocks) of the weight-gradient launch."""
    kpad, npad = -(-Kin // 128) * 128, -(-Nout // 32) * 32
    tiles = kpad // 128 * -(-npad // 128)
    cap = max(1, min(132, 132 * 256 * 256 // (kpad * npad)))
    return min(sms // tiles, cap), -(-Nn // 32)


# C views: "vec" 16-byte aligned with ldc % 4 == 0 (vector epilogue), "odd" ldc odd, "shift" one float off 16-byte alignment
# (both the scalar epilogue for every chunk).
# (M, N, K, p, C view, bias)
ACT_CASES = [
    (20_000, 256, 1000, 0.5, "vec", True),
    (40_001, 40, 100, 0.1, "shift", False),
    (20_000, 349, 36, 0.1, "odd", True),
    (40_001, 48, 4, 0.0, "vec", False),
    (3001, 1, 4, 0.5, "shift", True),
    (1000, 49, 2048, 0.0, "vec", True),
    (777, 100, 2048, 0.1, "odd", False),
]
# (M, N, K, p, slope, C view, bias)
PRELU_CASES = [
    (20_000, 256, 4100, 0.1, -0.5, "vec", True),
    (40_001, 40, 36, 0.5, 0.25, "shift", False),
    (20_000, 349, 100, 0.0, 1.0, "odd", True),
    (40_001, 40, 1000, 0.1, 1.0, "vec", True),
    (1001, 1, 4, 0.1, 0.0, "shift", True),
    (777, 49, 1000, 0.5, -0.5, "odd", False),
    (3001, 100, 4100, 0.0, 0.0, "vec", True),
]
# (M, N, K, p, BatchNorm-backward variant (0 automatic, 1 TMA-staged Y, 2 register loads), accumulate)
BNBWD_CASES = [
    (20_000, 256, 40, 0.5, 1, False),
    (20_000, 256, 1000, 0.1, 2, True),
    (40_001, 128, 36, 0.0, 1, True),
    (20_000, 96, 100, 0.5, 2, False),
    (1001, 64, 4, 0.1, 0, True),
    (777, 160, 2048, 0.5, 1, False),
]
# (M, N, K, p, slope, accumulate, slope_accumulate)
PRELU_BWD_CASES = [
    (20_000, 512, 1000, 0.1, -0.5, False, False),
    (40_001, 32, 36, 0.5, 0.25, True, True),
    (20_000, 256, 4, 0.0, 0.0, True, False),
    (777, 96, 100, 0.5, 1.0, False, True),
    (1001, 256, 4100, 0.1, -0.5, False, False),
]
# (M, N, K, C view)
ROWIDX_CASES = [
    (20_000, 256, 100, "vec"),
    (40_001, 40, 36, "shift"),
    (20_000, 349, 1000, "odd"),
    (40_001, 1, 4, "vec"),
    (1, 1, 4, "shift"),
    (777, 49, 4, "odd"),
    (3001, 100, 256, "vec"),
]
# (Nn, Kin, Nout, p)
WGRAD_ACT_CASES = [
    (40_001, 2048, 512, 0.1),
    (40_001, 36, 40, 0.5),
    (40_001, 132, 4, 0.0),
    (33, 520, 132, 0.0),
    (33, 2048, 40, 0.5),
    (31, 100, 4, 0.1),
    (1, 4, 512, 0.5),
    (1, 132, 132, 0.1),
]
# (Nn, Kin, Nout, p, slope, c0, spare words): Z is a column block [c0, c0 + Kin) of a wider NaN matrix whose keep bits have
# `spare` more words per row than the block needs past c0 + Kin; the kernel gets Z + c0, bits + c0 / 32 and that pitch.
WGRAD_PRELU_CASES = [
    (40_001, 2048, 512, 0.1, -0.5, 0, 0),
    (40_001, 36, 40, 0.5, 0.25, 64, 3),
    (40_001, 132, 4, 0.0, 0.25, 512, 2),
    (33, 520, 132, 0.0, 1.0, 32, 1),
    (31, 100, 4, 0.1, 0.0, 0, 0),
    (1, 4, 512, 0.5, -0.5, 2048, 0),
]
# Z wider than the kernel's 2048 columns: ops.gemm_wgrad_tf32x3_prelu runs it as 512-column blocks
WGRAD_PRELU_WIDE_KIN = [2052, 3000]


# ------------------------------------------------------------------------------------------------------ error model
# The activation prologues (and their materialisers) round twice per element: fmaf(y, sc, sh) (one rounding of the exact
# y·sc + sh; its sign is the exact sign, so the ReLU decision is exact) then the product by inv_keep; PReLU: slope·z then
# inv_keep (z > 0: one).  So the fp32 activation a satisfies |a - a64| <= ((1 + u)^2 - 1)|a64| <= (2^-23 + 2^-48)|a64|, and
# |C - C64| <= beta·(|a|·|B|^T) + |a - a64|·|B|^T <= (beta + 2^-23)(1 + 2^-22)·(|a64|·|B|^T) — the GEMM's bound taken on
# the fp64 activation.  (Subnormal activations would lose the relative bound; the operands here stay far from them.)
def act_beta(beta_: float) -> float:
    return (beta_ + 2.0 ** -23) * (1 + 2.0 ** -22)


def _inv_keep(p: float) -> float:
    """The fp32 1 / (1 - p) every kernel multiplies by (1 for p = 0)."""
    return float(torch.tensor(1.0) / (1 - torch.tensor(p))) if p > 0 else 1.0


def _keep_bits(rows: int, K: int, p: float, g: torch.Generator) -> torch.Tensor:
    """int32 [rows, ceil(K / 32)] keep bits, P(keep) = 1 - p, the bits past K random garbage; p = 0: all ones."""
    W = -(-K // 32)
    if p == 0:
        return torch.full((rows, W), -1, dtype=torch.int32, device="cuda")
    keep = torch.rand(rows, 32 * W, generator=g, device="cuda") >= p
    keep[:, K:] = torch.rand(rows, 32 * W - K, generator=g, device="cuda") < 0.5
    w = (keep.view(rows, W, 32).long() << torch.arange(32, device="cuda")).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def _affine_relu_bits(y, bits, scale, shift, p):
    """ops.affine_relu_bits (K <= 1024 per call) over 1024-column blocks: the same elementwise operations for any K."""
    K = y.shape[1]
    return torch.cat([ops.affine_relu_bits(y[:, c0:c0 + 1024].contiguous(), bits[:, c0 // 32:(c0 + 1024) // 32].contiguous(),
                                           scale[c0:c0 + 1024], shift[c0:c0 + 1024], p) for c0 in range(0, K, 1024)], 1)


def _keep(bits: torch.Tensor, K: int) -> torch.Tensor:
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    return ((bits.unsqueeze(-1) >> sh) & 1).bool().flatten(-2)[:, :K]


def _relu64(y, scale, shift, keep, k):
    a = (y.double() * scale.double() + shift.double()).clamp_min(0) * k
    return torch.where(keep, a, torch.zeros_like(a))


def _prelu64(z, slope: float, keep, k):
    z = z.double()
    a = torch.where(z > 0, z, slope * z) * k
    return torch.where(keep, a, torch.zeros_like(a))


def _bn_operands(rows: int, K: int, g: torch.Generator):
    """Y and a BatchNorm (scale, shift) with columns scaled over 2^±10 and a fifth of the scales negative."""
    y = torch.randn(rows, K, generator=g, device="cuda") * 2 + 0.3
    cs = _pow2(K, g, 10)
    sign = torch.where(torch.rand(K, generator=g, device="cuda") < 0.2, -1.0, 1.0)
    scale = (torch.rand(K, generator=g, device="cuda") + 0.5) * cs * sign
    shift = torch.randn(K, generator=g, device="cuda") * 0.5 * cs
    return y, scale, shift


def _in_canaries(vals: torch.Tensor):
    """A 1-D vector at a 16-byte aligned offset inside a canary buffer: (buffer, vector view)."""
    buf = _poisoned(1, vals.numel() + 8).view(-1)
    v = buf[4:4 + vals.numel()]
    v.copy_(vals)
    return buf, v


def _out_view(rows: int, N: int, view: str):
    """(canary buffer, [rows, N] view at row 5, its mask) with the pitch / alignment of `view`."""
    c_off = 1 if view == "shift" else 0
    ldc = N + 1 + N % 2 if view == "odd" else -(-N // 4) * 4 + 4
    buf = _poisoned(rows + 9, ldc)
    return buf, _view(buf, 5, c_off, rows, N), _mask_of(buf, 5, c_off, rows, N)


def _ptr(t):
    return None if t is None else t.data_ptr()


def _assert_multi_tile(tiles: int):
    """A table case that claims >= 2 tiles per CTA on 132 SMs has them on this device too."""
    if tiles > SMS:
        sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
        assert tiles > sms, (tiles, sms)


def _report(entry: str, case, ratio: float):
    print(f"bound ratio {entry} {case}: {ratio:.3g}")


# ------------------------------------------------------------------------------------------------ 1. ACT prologue
@pytest.mark.parametrize("M,N,K,p,view,with_bias", ACT_CASES)
def test_act_gemm(M, N, K, p, view, with_bias):
    _assert_multi_tile(gemm_tiles(M, N))
    g = _gen(M + 7 * N + 31 * K)
    y, scale, shift = _bn_operands(M, K, g)
    w = torch.randn(N, K, generator=g, device="cuda") * _pow2(N, g)[:, None]
    bias = torch.randn(N, generator=g, device="cuda") * _pow2(N, g) if with_bias else None
    bits = _keep_bits(M, K, p, g)
    hi, lo = ops.split_tf32(w)
    twin = ops.gemm_tf32x3(_affine_relu_bits(y, bits, scale, shift, p), hi, lo, bias=bias)

    yv, hv, lv = _poisoned_operand(y), _poisoned_operand(hi), _poisoned_operand(lo)
    sc, sh = _in_canaries(scale)[1], _in_canaries(shift)[1]
    bv = _in_canaries(bias)[1] if with_bias else None
    cbuf, cv, mask = _out_view(M, N, view)
    lib.check(lib.load().b200gnn_gemm_tf32x3_act_f32(
        yv.data_ptr(), yv.stride(0), hv.data_ptr(), lv.data_ptr(), hv.stride(0), cv.data_ptr(), cv.stride(0), M, N, K,
        _ptr(bv), sc.data_ptr(), sh.data_ptr(), bits.data_ptr(), p, lib.stream_ptr()), "gemm_tf32x3_act_f32")
    torch.cuda.synchronize()
    assert torch.equal(cv, twin)
    assert _outside_is_canary(cbuf, mask)
    a64 = _relu64(y, scale, shift, _keep(bits, K), _inv_keep(p))
    r = _gemm_check(a64, w, cv, act_beta(beta_k(K)), bias=bias)
    _report("act", (M, N, K, p), r)
    assert r <= 1.0


# ---------------------------------------------------------------------------------------------- 2. PReLU prologue
@pytest.mark.parametrize("M,N,K,p,slope,view,with_bias", PRELU_CASES)
def test_prelu_gemm(M, N, K, p, slope, view, with_bias):
    _assert_multi_tile(gemm_tiles(M, N))
    g = _gen(M + 7 * N + 31 * K)
    z = torch.randn(M, K, generator=g, device="cuda") * _pow2(M, g)[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") * _pow2(N, g)[:, None]
    bias = torch.randn(N, generator=g, device="cuda") * _pow2(N, g) if with_bias else None
    a = torch.tensor([slope], device="cuda")
    bits = _keep_bits(M, K, p, g)
    hi, lo = ops.split_tf32(w)
    twin = ops.gemm_tf32x3(ops.prelu_bits(z, bits, a, p), hi, lo, bias=bias)

    zv, hv, lv = _poisoned_operand(z), _poisoned_operand(hi), _poisoned_operand(lo)
    bv = _in_canaries(bias)[1] if with_bias else None
    cbuf, cv, mask = _out_view(M, N, view)
    lib.check(lib.load().b200gnn_gemm_tf32x3_prelu_f32(
        zv.data_ptr(), zv.stride(0), hv.data_ptr(), lv.data_ptr(), hv.stride(0), cv.data_ptr(), cv.stride(0), M, N, K,
        _ptr(bv), a.data_ptr(), bits.data_ptr(), p, lib.stream_ptr()), "gemm_tf32x3_prelu_f32")
    torch.cuda.synchronize()
    assert torch.equal(cv, twin)
    assert _outside_is_canary(cbuf, mask)
    a64 = _prelu64(z, slope, _keep(bits, K), _inv_keep(p))
    r = _gemm_check(a64, w, cv, act_beta(beta_k(K)), bias=bias)
    _report("prelu", (M, N, K, p, slope), r)
    assert r <= 1.0


# ------------------------------------------------------------------------------ 3. BatchNorm backward from keep bits
@pytest.mark.parametrize("M,N,K,p,variant,accumulate", BNBWD_CASES)
def test_bnbwd_bits_gemm(M, N, K, p, variant, accumulate):
    """dz = dOut·[bit && y·sc + sh > 0]·inv_keep and the partials (sum dz, sum dz·xhat): bit-identical to the bnbwd GEMM
    on the materialised Xout; dz within k·(E(1 + u) + u·(|A|·|B|^T + |C_in|)) of fp64, E the GEMM's bound on dOut (the
    mask is exact: fmaf keeps the sign of y·sc + sh)."""
    _assert_multi_tile(gemm_tiles(M, N, narrow_ok=False))
    g = _gen(M + 7 * N + 31 * K + variant)
    a = torch.randn(M, K, generator=g, device="cuda") * _pow2(M, g)[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") * _pow2(N, g)[:, None]
    y, scale, shift = _bn_operands(M, N, g)
    mean, invstd = torch.randn(N, generator=g, device="cuda"), torch.rand(N, generator=g, device="cuda") + 0.5
    c_in = torch.randn(M, N, generator=g, device="cuda") * a.abs().max(1).values[:, None] if accumulate else None
    bits = _keep_bits(M, N, p, g)
    hi, lo = ops.split_tf32(w)
    x_out = ops.affine_relu_bits(y, bits, scale, shift, p)
    slots = ops.gemm_stat_slots(M, N)

    ldc = N + 8
    av = _poisoned_operand(a)
    cbuf, ybuf = _poisoned(M + 40, ldc), _poisoned(M + 40, ldc)
    cv, yv = _view(cbuf, 0, 0, M, N), _view(ybuf, 0, 0, M, N)
    yv.copy_(y)
    if accumulate:
        cv.copy_(c_in)
    pbuf = _poisoned(1, slots * 2 * N + 64).view(-1)
    part = pbuf[32:32 + slots * 2 * N]
    sc, sh = _in_canaries(scale)[1], _in_canaries(shift)[1]
    L = lib.load()
    L.b200gnn_gemm_set_bnbwd_variant(variant)
    try:
        twin = c_in.clone() if accumulate else torch.empty(M, N, device="cuda")
        twin_part = torch.full((slots, 2, N), float("nan"), device="cuda")
        ops.gemm_tf32x3_bnbwd(a, hi, lo, twin, x_out, y, mean, invstd, p, twin_part, accumulate=accumulate)
        lib.check(L.b200gnn_gemm_tf32x3_bnbwd_bits_f32(
            av.data_ptr(), av.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0), cv.data_ptr(), ldc, M, N, K,
            int(accumulate), bits.data_ptr(), yv.data_ptr(), mean.data_ptr(), invstd.data_ptr(), sc.data_ptr(),
            sh.data_ptr(), p, part.data_ptr(), slots, lib.stream_ptr()), "gemm_tf32x3_bnbwd_bits_f32")
        torch.cuda.synchronize()
    finally:
        L.b200gnn_gemm_set_bnbwd_variant(0)
    assert torch.equal(cv, twin)
    assert bool(torch.isfinite(part).all()) and torch.equal(part.view(slots, 2, N), twin_part)
    assert _outside_is_canary(cbuf, _mask_of(cbuf, 0, 0, M, N))
    inside = torch.zeros(pbuf.shape, dtype=torch.bool, device="cuda")
    inside[32:32 + slots * 2 * N] = True
    assert _outside_is_canary(pbuf, inside)

    k = _inv_keep(p)
    a64, w64 = a.double(), w.double()
    d64, mag = a64 @ w64.t(), a64.abs() @ w64.abs().t()
    err = beta_k(K) * mag
    if accumulate:
        d64 += c_in.double()
        err += EPI * (mag + c_in.double().abs())
        mag = mag + c_in.double().abs()
    live = _keep(bits, N) & (y.double() * scale.double() + shift.double() > 0)
    assert bool((cv[~live] == 0).all())
    bound = k * (err * (1 + U) + U * mag)
    r = float(((cv.double() - d64 * k).abs() / bound)[live].max())
    _report("bnbwd_bits", (M, N, K, p, variant, accumulate), r)
    assert r <= 1.0
    dz = cv.double()
    xhat = (y.double() - mean.double()) * invstd.double()
    assert rel_err(part.view(slots, 2, N).double().sum(0), torch.stack([dz.sum(0), (dz * xhat).sum(0)])) < 1e-6


# ------------------------------------------------------------------------------------------- 4. PReLU backward epilogue
@pytest.mark.parametrize("M,N,K,p,slope,accumulate,slope_accumulate", PRELU_BWD_CASES)
def test_prelu_bwd_gemm(M, N, K, p, slope, accumulate, slope_accumulate):
    """dZ = (bit ? dA·inv_keep : 0)·(z > 0 ? 1 : slope) bit for bit against torch on the plain GEMM's dA (the same
    128-column tile shape: B padded to 64 rows for N <= 48).  The slope gradient adds t = fl(g·z) over z <= 0 in fp64:
    each product rounds once (u|g z|), the fp64 chains (per lane, the shuffle tree, the slot sum) take at most
    M·N + 4096 additions of 2^-53 each, the cast to fp32 one u of |sum| <= sum |g z|, and slope_accumulate one more fp32
    add of u·|prior + sum|.  Two calls are bit-identical."""
    _assert_multi_tile(gemm_tiles(M, N, narrow_ok=False))
    g = _gen(M + 7 * N + 31 * K)
    a = torch.randn(M, K, generator=g, device="cuda") * _pow2(M, g)[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") / K ** 0.5
    z = torch.randn(M, N, generator=g, device="cuda") * _pow2(N, g, 10)[None, :]
    c_in = torch.randn(M, N, generator=g, device="cuda") if accumulate else None
    bits = _keep_bits(M, N, p, g)
    at = torch.tensor([slope], device="cuda")
    hi, lo = ops.split_tf32(w)
    npad = max(N, 64)
    hp, lp = ops.split_tf32(torch.cat([w, torch.zeros(npad - N, K, device="cuda")]))
    d_full = torch.zeros(M, npad, device="cuda")
    if accumulate:
        d_full[:, :N] = c_in
    ops.gemm_tf32x3(a, hp, lp, out=d_full, accumulate=accumulate)
    dA = d_full[:, :N]
    k = _inv_keep(p)
    gk = torch.where(_keep(bits, N), dA * k, torch.zeros_like(dA))
    ref = torch.where(z > 0, gk, gk * at)

    ldc = N + 8
    av = _poisoned_operand(a)
    cbuf, zbuf = _poisoned(M + 40, ldc), _poisoned(M + 40, ldc)
    cv, zv = _view(cbuf, 0, 0, M, N), _view(zbuf, 0, 0, M, N)
    zv.copy_(z)
    slots = ops.gemm_stat_slots(M, N)
    pbuf = _poisoned(1, 2 * slots + 16).view(-1)
    part = pbuf[8:8 + 2 * slots].view(torch.float64)
    prior = 3.0 - slope
    outs, grads = [], []
    for _ in range(2):
        if accumulate:
            cv.copy_(c_in)
        else:
            cv.copy_(_poisoned(M, N))
        sgbuf, sg = _in_canaries(torch.tensor([prior], device="cuda"))
        lib.check(lib.load().b200gnn_gemm_tf32x3_prelu_bwd_f32(
            av.data_ptr(), av.stride(0), hi.data_ptr(), lo.data_ptr(), hi.stride(0), cv.data_ptr(), ldc, M, N, K,
            int(accumulate), zv.data_ptr(), bits.data_ptr(), at.data_ptr(), p, sg.data_ptr(), int(slope_accumulate),
            part.data_ptr(), slots, lib.stream_ptr()), "gemm_tf32x3_prelu_bwd_f32")
        torch.cuda.synchronize()
        inside = torch.zeros(sgbuf.shape, dtype=torch.bool, device="cuda")
        inside[4] = True
        assert _outside_is_canary(sgbuf, inside)
        outs.append(cv.clone())
        grads.append(sg.clone())
    assert torch.equal(outs[0], ref) and torch.equal(outs[1], ref)
    assert torch.equal(grads[0].view(torch.int32), grads[1].view(torch.int32))
    assert _outside_is_canary(cbuf, _mask_of(cbuf, 0, 0, M, N))
    inside = torch.zeros(pbuf.shape, dtype=torch.bool, device="cuda")
    inside[8:8 + 2 * slots] = True
    assert _outside_is_canary(pbuf, inside)

    t = torch.where(z <= 0, gk.double() * z.double(), torch.zeros_like(z, dtype=torch.float64))
    s, tabs = float(t.sum()), float(t.abs().sum())
    e0 = (2.0 ** -23 + (M * N + 4096) * 2.0 ** -53) * tabs * (1 + 2.0 ** -20)
    want = prior + s if slope_accumulate else s
    bound = e0 * (1 + 2.0 ** -23) + U * abs(want) if slope_accumulate else e0
    r = abs(float(grads[0]) - want) / bound if bound > 0 else float(float(grads[0]) != want)
    _report("prelu_bwd slope", (M, N, K, p, slope), r)
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ 5. row-indexed stores
@pytest.mark.parametrize("M,N,K,view", ROWIDX_CASES)
def test_rowidx_gemm(M, N, K, view):
    """C[row_idx[m]] = (A·B^T)[m] for an unsorted, distinct subset of the rows of a taller C: the named rows equal the
    plain GEMM bit for bit and hold the fp64 bound; every other element of C and its buffer keeps its canary."""
    _assert_multi_tile(gemm_tiles(M, N))
    g = _gen(M + 7 * N + 31 * K)
    rows_c = M + M // 2 + 7
    a = torch.randn(M, K, generator=g, device="cuda") * _pow2(M, g)[:, None]
    w = torch.randn(N, K, generator=g, device="cuda") * _pow2(N, g)[:, None]
    row_idx = torch.randperm(rows_c, generator=g, device="cuda")[:M]
    hi, lo = ops.split_tf32(w)
    plain = ops.gemm_tf32x3(a, hi, lo)

    av, hv, lv = _poisoned_operand(a), _poisoned_operand(hi), _poisoned_operand(lo)
    cbuf, cv, mask = _out_view(rows_c, N, view)
    lib.check(lib.load().b200gnn_gemm_tf32x3_rowidx_f32(
        av.data_ptr(), av.stride(0), hv.data_ptr(), lv.data_ptr(), hv.stride(0), cv.data_ptr(), cv.stride(0), M, N, K,
        row_idx.data_ptr(), lib.stream_ptr()), "gemm_tf32x3_rowidx_f32")
    torch.cuda.synchronize()
    got = cv[row_idx]
    assert torch.equal(got, plain)
    named = torch.zeros(rows_c, dtype=torch.bool, device="cuda")
    named[row_idx] = True
    mask[5:5 + rows_c] &= named[:, None]                 # the view's rows start at row 5 of the buffer
    assert _outside_is_canary(cbuf, mask)
    r = _gemm_check(a, w, got, beta_k(K))
    _report("rowidx", (M, N, K), r)
    assert r <= 1.0


# ------------------------------------------------------------------------------------------------ 6. weight gradients
def _wgrad_buffers(Kin: int, Nout: int):
    n_ws = ops.wgrad_workspace_floats(Kin, Nout)
    wbuf, wsbuf = _poisoned(1, Kin * Nout + 64).view(-1), _poisoned(1, n_ws + 64).view(-1)
    return wbuf, wbuf[32:32 + Kin * Nout].view(Kin, Nout), wsbuf, wsbuf[32:32 + n_ws]


def _assert_wgrad_canaries(wbuf, wsbuf, Kin: int, Nout: int):
    for buf, n in ((wbuf, Kin * Nout), (wsbuf, wsbuf.numel() - 64)):
        inside = torch.zeros(buf.shape, dtype=torch.bool, device="cuda")
        inside[32:32 + n] = True
        assert _outside_is_canary(buf, inside)


@pytest.mark.parametrize("Nn,Kin,Nout,p", WGRAD_ACT_CASES)
def test_act_wgrad(Nn, Kin, Nout, p):
    g = _gen(Nn + 7 * Kin + 31 * Nout)
    y, scale, shift = _bn_operands(Nn, Kin, g)
    d = torch.randn(Nn, Nout, generator=g, device="cuda") * _pow2(Nout, g)[None, :]
    bits = _keep_bits(Nn, Kin, p, g)
    twin = ops.gemm_wgrad_tf32x3(_affine_relu_bits(y, bits, scale, shift, p), d, wide=True)

    yv = _poisoned_operand(y, r0=2, c0=4, extra_rows=37, extra_cols=8)
    dv = _poisoned_operand(d, r0=2, c0=0, extra_rows=37, extra_cols=8)
    sc, sh = _in_canaries(scale)[1], _in_canaries(shift)[1]
    wbuf, dw, wsbuf, ws = _wgrad_buffers(Kin, Nout)
    lib.check(lib.load().b200gnn_gemm_wgrad_tf32x3_act_f32(
        yv.data_ptr(), yv.stride(0), dv.data_ptr(), dv.stride(0), dw.data_ptr(), Nn, Kin, Nout, sc.data_ptr(), sh.data_ptr(),
        bits.data_ptr(), p, ws.data_ptr(), lib.stream_ptr()), "gemm_wgrad_tf32x3_act_f32")
    torch.cuda.synchronize()
    assert torch.equal(dw, twin)
    _assert_wgrad_canaries(wbuf, wsbuf, Kin, Nout)
    a64 = _relu64(y, scale, shift, _keep(bits, Kin), _inv_keep(p))
    r = _gemm_check(a64.t(), d.t(), dw, act_beta(_wgrad_beta(Nn)))
    _report("wgrad_act", (Nn, Kin, Nout, p), r)
    assert r <= 1.0


@pytest.mark.parametrize("Nn,Kin,Nout,p,slope,c0,spare", WGRAD_PRELU_CASES)
def test_prelu_wgrad(Nn, Kin, Nout, p, slope, c0, spare):
    g = _gen(Nn + 7 * Kin + 31 * Nout + c0)
    kw = c0 + Kin
    words = -(-kw // 32) + spare
    z = torch.randn(Nn, Kin, generator=g, device="cuda") * _pow2(Kin, g)[None, :]
    zbuf = _poisoned(Nn + 37, kw + 8)
    zv = _view(zbuf, 0, c0, Nn, Kin)                       # NaN columns on both sides of the block, NaN rows past Nn
    zv.copy_(z)
    bits_all = _keep_bits(Nn, 32 * words, p, g)
    bits = bits_all[:, c0 // 32:]
    d = torch.randn(Nn, Nout, generator=g, device="cuda") * _pow2(Nout, g)[None, :]
    at = torch.tensor([slope], device="cuda")
    twin = ops.gemm_wgrad_tf32x3(ops.prelu_bits(z, bits, at, p), d, wide=True)

    dv = _poisoned_operand(d, r0=2, c0=0, extra_rows=37, extra_cols=8)
    wbuf, dw, wsbuf, ws = _wgrad_buffers(Kin, Nout)
    lib.check(lib.load().b200gnn_gemm_wgrad_tf32x3_prelu_f32(
        zv.data_ptr(), zv.stride(0), dv.data_ptr(), dv.stride(0), dw.data_ptr(), Nn, Kin, Nout, at.data_ptr(),
        bits.data_ptr(), words, p, ws.data_ptr(), lib.stream_ptr()), "gemm_wgrad_tf32x3_prelu_f32")
    torch.cuda.synchronize()
    assert torch.equal(dw, twin)
    _assert_wgrad_canaries(wbuf, wsbuf, Kin, Nout)
    a64 = _prelu64(z, slope, _keep(bits, Kin), _inv_keep(p))
    r = _gemm_check(a64.t(), d.t(), dw, act_beta(_wgrad_beta(Nn)))
    _report("wgrad_prelu", (Nn, Kin, Nout, p, slope, c0), r)
    assert r <= 1.0


@pytest.mark.parametrize("Kin", WGRAD_PRELU_WIDE_KIN)
def test_prelu_wgrad_wide_z(Kin):
    """ops.gemm_wgrad_tf32x3_prelu on a Z wider than 2048 columns (512-column blocks, the keep bits passed at word offset
    c0 / 32 with the full row pitch): each block equals the weight gradient of the materialised block, and the whole
    holds the fp64 bound."""
    Nn, Nout, p, slope = 4099, 40, 0.1, -0.25
    g = _gen(Kin)
    z = torch.randn(Nn, Kin, generator=g, device="cuda")
    d = torch.randn(Nn, Nout, generator=g, device="cuda")
    bits = _keep_bits(Nn, Kin, p, g)
    at = torch.tensor([slope], device="cuda")
    got = ops.gemm_wgrad_tf32x3_prelu(z, at, bits, p, d)
    x = ops.prelu_bits(z, bits, at, p)
    for c0 in range(0, Kin, ops.WGRAD_PRELU_BLOCK):
        blk = x[:, c0:c0 + ops.WGRAD_PRELU_BLOCK].contiguous()
        assert torch.equal(got[c0:c0 + blk.shape[1]], ops.gemm_wgrad_tf32x3(blk, d, wide=True)), c0
    a64 = _prelu64(z, slope, _keep(bits, Kin), _inv_keep(p))
    r = _gemm_check(a64.t(), d.t(), got, act_beta(_wgrad_beta(Nn)))
    _report("wgrad_prelu wide", (Nn, Kin, Nout), r)
    assert r <= 1.0


# ------------------------------------------------------------------------------------- 7. column-block wrappers (SIGN)
def test_column_block_wrappers():
    """The ops wrappers the SIGN engine calls on 16-byte aligned column blocks of wider matrices ([B, hops·hidden]): every
    result bit-identical to the same call on contiguous copies, the neighbouring columns of the output untouched."""
    M, H, hops, N, p = 3001, 256, 3, 256, 0.1
    g = _gen(3001)

    def block(col, width, vals=None):
        """(canary buffer [M, hops·H], its column block [col, col + width)) holding vals, or NaN when vals is None."""
        buf = _poisoned(M, hops * H)
        v = buf[:, col:col + width]
        if vals is not None:
            v.copy_(vals)
        return buf, v

    def untouched(buf, col, width):
        return _outside_is_canary(buf, _mask_of(buf, 0, col, M, width))

    a = torch.randn(M, H, generator=g, device="cuda")
    w = torch.randn(N, H, generator=g, device="cuda") / H ** 0.5
    bias = torch.randn(N, generator=g, device="cuda")
    hi, lo = ops.split_tf32(w)
    _, av = block(H, H, a)
    obuf, ov = block(2 * H, N)
    ops.gemm_tf32x3_rows(av, hi, lo, ov, bias)
    torch.cuda.synchronize()
    assert torch.equal(ov, ops.gemm_tf32x3(a, hi, lo, bias=bias)) and untouched(obuf, 2 * H, N)

    gr = torch.randn(M, N, generator=g, device="cuda")
    _, gv = block(H, N, gr)
    ws = torch.empty(ops.wgrad_workspace_floats(H, N), device="cuda")
    dw = ops.gemm_wgrad_tf32x3_rows(av, gv, torch.empty(H, N, device="cuda"), ws)
    assert torch.equal(dw, ops.gemm_wgrad_tf32x3(a, gr, wide=True))

    z = torch.randn(M, H, generator=g, device="cuda")
    at = torch.tensor([-0.25], device="cuda")
    bits = _keep_bits(M, H, p, g)
    _, zv = block(0, H, z)
    obuf, ov = block(H, N)
    ops.gemm_tf32x3_prelu(zv, at, bits, p, hi, lo, bias=bias, out=ov)
    torch.cuda.synchronize()
    assert torch.equal(ov, ops.gemm_tf32x3_prelu(z, at, bits, p, hi, lo, bias=bias)) and untouched(obuf, H, N)

    # prelu_bwd: A, Z and the output (dZ) all column blocks; Z and the output share the wide pitch
    w2 = torch.randn(H, N, generator=g, device="cuda") / N ** 0.5
    hi2, lo2 = ops.split_tf32(w2)
    gin = torch.randn(M, N, generator=g, device="cuda")
    zb = torch.randn(M, H, generator=g, device="cuda")
    bits2 = _keep_bits(M, H, p, g)
    part = torch.empty(ops.gemm_stat_slots(M, H), dtype=torch.float64, device="cuda")
    ref_out, ref_sg = torch.empty(M, H, device="cuda"), torch.zeros(1, device="cuda")
    ops.gemm_tf32x3_prelu_bwd(gin, hi2, lo2, ref_out, zb, bits2, at, p, ref_sg, part)
    _, gbv = block(2 * H, N, gin)
    _, zbv = block(H, H, zb)
    obuf, ov = block(H, H)
    sg = torch.zeros(1, device="cuda")
    ops.gemm_tf32x3_prelu_bwd(gbv, hi2, lo2, ov, zbv, bits2, at, p, sg, part)
    torch.cuda.synchronize()
    assert torch.equal(ov, ref_out) and torch.equal(sg, ref_sg) and untouched(obuf, H, H)


# ------------------------------------------------------------------------------------------------------- 8. refusals
def _refusals(entry: str):
    """(list of (name, expected code, thunk), output buffers that must keep their canaries) for one entry point.  Every
    buffer is large enough for the widest shape a refused call names, so a call that wrongly runs stays in bounds."""
    L, st = lib.load(), lib.stream_ptr()
    M, K, N = 300, 64, 64
    big_n, big_k = 512, 2100
    A = torch.randn(M, big_k + 8, device="cuda")
    hi, lo = (torch.randn(big_n, big_k + 8, device="cuda") for _ in range(2))
    C = _poisoned(M + 4, big_n + 8)
    vec = torch.rand(big_k + 8, device="cuda") + 0.5
    bits = torch.full((M + 4, big_k), -1, dtype=torch.int32, device="cuda")
    Y = torch.randn(M + 4, big_n + 8, device="cuda")
    slope = torch.tensor([0.25], device="cuda")
    a, h, l_, c, v, b, y = (t.data_ptr() for t in (A, hi, lo, C, vec, bits, Y))
    lda = ldb = big_k + 8
    ldc = big_n + 8
    outs = [C]
    if entry == "act":
        def call(y_=a, k=K, n=N, ldc_=ldc, sc=v, sh=v, bb=b, p=0.5, lda_=lda):
            return L.b200gnn_gemm_tf32x3_act_f32(y_, lda_, h, l_, ldb, c, ldc_, M, n, k, None, sc, sh, bb, p, st)
        cases = [("K > 2048", UNSUPPORTED, lambda: call(k=2052)), ("bits NULL", BAD_ARG, lambda: call(bb=None)),
                 ("scale NULL", BAD_ARG, lambda: call(sc=None)), ("shift NULL", BAD_ARG, lambda: call(sh=None)),
                 ("scale misaligned", BAD_ARG, lambda: call(sc=v + 4)), ("p = 1", BAD_ARG, lambda: call(p=1.0)),
                 ("p < 0", BAD_ARG, lambda: call(p=-0.1)), ("lda % 4", UNSUPPORTED, lambda: call(lda_=lda - 2)),
                 ("Y misaligned", UNSUPPORTED, lambda: call(y_=a + 4)), ("ldc < N", BAD_ARG, lambda: call(ldc_=N - 1))]
    elif entry == "prelu":
        def call(sl=slope.data_ptr(), bb=b, p=0.5, lda_=lda):
            return L.b200gnn_gemm_tf32x3_prelu_f32(a, lda_, h, l_, ldb, c, ldc, M, N, K, None, sl, bb, p, st)
        cases = [("slope NULL", BAD_ARG, lambda: call(sl=None)), ("bits NULL", BAD_ARG, lambda: call(bb=None)),
                 ("p = 1", BAD_ARG, lambda: call(p=1.0)), ("lda % 4", UNSUPPORTED, lambda: call(lda_=lda - 1))]
    elif entry == "prelu_bwd":
        slots = ops.gemm_stat_slots(M, big_n)
        part = torch.full((slots + 8,), 7.0, dtype=torch.float64, device="cuda")
        sg = torch.full((1,), 5.0, device="cuda")
        outs += [part, sg]

        def call(n=N, ldc_=ldc, c_=c, z=y, bb=b, sl=slope.data_ptr(), sgp=sg.data_ptr(), pp=part.data_ptr(), ns=slots, p=0.5):
            return L.b200gnn_gemm_tf32x3_prelu_bwd_f32(a, lda, h, l_, ldb, c_, ldc_, M, n, K, 0, z, bb, sl, p, sgp, 0, pp, ns, st)
        cases = [("N % 32", UNSUPPORTED, lambda: call(n=40)), ("ldc % 4", UNSUPPORTED, lambda: call(ldc_=ldc - 1)),
                 ("C misaligned", UNSUPPORTED, lambda: call(c_=c + 4)), ("Z misaligned", UNSUPPORTED, lambda: call(z=y + 4)),
                 ("Z NULL", BAD_ARG, lambda: call(z=None)), ("bits NULL", BAD_ARG, lambda: call(bb=None)),
                 ("slope NULL", BAD_ARG, lambda: call(sl=None)), ("slope_grad NULL", BAD_ARG, lambda: call(sgp=None)),
                 ("partial NULL", BAD_ARG, lambda: call(pp=None)),
                 ("slots short", BAD_ARG, lambda: call(ns=ops.gemm_stat_slots(M, N) - 1)), ("p = 1", BAD_ARG, lambda: call(p=1.0))]
    elif entry == "bnbwd_bits":
        slots = ops.gemm_stat_slots(M, big_n)
        part = _poisoned(slots, 2 * big_n)
        outs.append(part)
        mv = torch.randn(big_n + 8, device="cuda")

        def call(n=128, ldc_=ldc, bb=b, y_=y, sc=v, sh=v, ns=slots, p=0.5, c_=c):
            return L.b200gnn_gemm_tf32x3_bnbwd_bits_f32(a, lda, h, l_, ldb, c_, ldc_, M, n, K, 0, bb, y_, mv.data_ptr(),
                                                        mv.data_ptr(), sc, sh, p, part.data_ptr(), ns, st)
        cases = [("N % 32", UNSUPPORTED, lambda: call(n=100)), ("N > 256", UNSUPPORTED, lambda: call(n=288)),
                 ("N <= 48", UNSUPPORTED, lambda: call(n=32)), ("ldc % 4", UNSUPPORTED, lambda: call(ldc_=ldc - 1)),
                 ("C misaligned", UNSUPPORTED, lambda: call(c_=c + 4)), ("Y misaligned", UNSUPPORTED, lambda: call(y_=y + 4)),
                 ("bits NULL", BAD_ARG, lambda: call(bb=None)), ("Y NULL", BAD_ARG, lambda: call(y_=None)),
                 ("scale NULL", BAD_ARG, lambda: call(sc=None)), ("p = 1", BAD_ARG, lambda: call(p=1.0)),
                 ("slots short", BAD_ARG, lambda: call(ns=ops.gemm_stat_slots(M, 128) - 1))]
    elif entry == "rowidx":
        ri = torch.arange(M, device="cuda")

        def call(r=ri.data_ptr(), lda_=lda, ldc_=ldc):
            return L.b200gnn_gemm_tf32x3_rowidx_f32(a, lda_, h, l_, ldb, c, ldc_, M, N, K, r, st)
        cases = [("row_idx NULL", BAD_ARG, lambda: call(r=None)), ("lda % 4", UNSUPPORTED, lambda: call(lda_=lda - 1)),
                 ("ldc < N", BAD_ARG, lambda: call(ldc_=N - 1))]
    else:
        ws = _poisoned(1, max(ops.wgrad_workspace_floats(2048, 512), ops.wgrad_workspace_floats(512, 512)) + 64).view(-1)
        dW = _poisoned(1, big_k * big_n + 64).view(-1)
        G = torch.randn(M, big_n + 8, device="cuda")
        outs = [ws, dW]
        gp, wp, dp = G.data_ptr(), ws.data_ptr(), dW.data_ptr()
        if entry == "wgrad_act":
            bw = torch.full((M, big_k // 32 + 2), -1, dtype=torch.int32, device="cuda")

            def call(kin=128, nout=40, sc=v, sh=v, bb=bw.data_ptr(), p=0.5, wsp=wp):
                return L.b200gnn_gemm_wgrad_tf32x3_act_f32(a, lda, gp, big_n + 8, dp, M, kin, nout, sc, sh, bb, p, wsp, st)
            cases = [("Kin > 2048", UNSUPPORTED, lambda: call(kin=2052)), ("Kin % 4", UNSUPPORTED, lambda: call(kin=6)),
                     ("Nout > 512", UNSUPPORTED, lambda: call(nout=516)), ("Nout % 4", UNSUPPORTED, lambda: call(nout=6)),
                     ("bits NULL", BAD_ARG, lambda: call(bb=None)), ("scale NULL", BAD_ARG, lambda: call(sc=None)),
                     ("p = 1", BAD_ARG, lambda: call(p=1.0)), ("workspace NULL", BAD_ARG, lambda: call(wsp=None))]
        else:
            bw = torch.full((M, big_k // 32 + 2), -1, dtype=torch.int32, device="cuda")

            def call(kin=100, ldbits=4, sl=slope.data_ptr(), bb=bw.data_ptr(), p=0.5):
                return L.b200gnn_gemm_wgrad_tf32x3_prelu_f32(a, lda, gp, big_n + 8, dp, M, kin, 40, sl, bb, ldbits, p, wp, st)
            cases = [("ldbits < ceil(Kin/32)", BAD_ARG, lambda: call(ldbits=3)),
                     ("ldbits < ceil(2048/32)", BAD_ARG, lambda: call(kin=2048, ldbits=63)),
                     ("Kin > 2048", UNSUPPORTED, lambda: call(kin=2052, ldbits=65)), ("slope NULL", BAD_ARG, lambda: call(sl=None)),
                     ("bits NULL", BAD_ARG, lambda: call(bb=None)), ("p = 1", BAD_ARG, lambda: call(p=1.0))]
    return cases, outs


REFUSAL_ENTRIES = ["act", "prelu", "prelu_bwd", "bnbwd_bits", "rowidx", "wgrad_act", "wgrad_prelu"]


@pytest.mark.parametrize("entry", REFUSAL_ENTRIES)
def test_refusals(entry):
    cases, outs = _refusals(entry)
    before = [o.clone() for o in outs]
    got = {name: thunk() for name, _, thunk in cases}
    torch.cuda.synchronize()
    assert got == {name: code for name, code, _ in cases}
    for o, b in zip(outs, before):
        assert torch.equal(o.view(torch.uint8), b.view(torch.uint8))
    assert bool((outs[0].view(torch.int32) == CANARY).all())          # C (dW's workspace): canaries throughout
