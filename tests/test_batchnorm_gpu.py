"""Accuracy contract of training-mode BatchNorm (dense_rows.cu and the statistics epilogues that feed it), checked through
the C ABI against float64 restatements computed from the same fp32 inputs the kernels read (DESIGN.md §4.3):

* statistics -> finalize, from every producer (col_stats, the SpMM epilogue on its register / bulk / multi-slab paths, the
  3xTF32 GEMM epilogue with and without accumulate, the GAT aggregation epilogue at the padded head width).  Three stages:
    A. the producer's fp32 slots: |sum_slots P - sum_rows y| <= gamma(L) · sum_rows |y|  (and the same for y²), L the
       producer's longest fp32 addition chain (written next to each producer below);
    B. bn_finalize from those slots against an fp64 restatement of the same slots: the fp64 rounding of both plus the fp32
       output roundings.  An fp32-accumulating finalize of the same slots is restated on the CPU and must violate this bound
       in the offset-dominated cases: that is what keeps the test able to see a subtly wrong finalize;
    C. end to end, Y -> mean / invstd / scale / shift: the error of var carries
           gamma(L) · (Σy²/n + 2|mean|·Σ|y|/n),
       so the relative error of invstd grows like gamma(L)·(1 + 3 (mean/std)²) / 2 — the (mean/std)² conditioning of
       E[y²] - mean² from fp32 sums.  The invstd bound is the interval [1/sqrt(var + e + eps), 1/sqrt(max(var - e, 0) + eps)];
* all-zero columns (the GAT padding) are exact: mean 0, invstd = fp32(1/sqrt(eps)), shift = beta; constant non-dyadic
  columns exercise the var < 0 clamp (invstd never exceeds fp32(1/sqrt(eps)));
* running statistics over five steps against torch.nn.BatchNorm1d in double, momentum 0.1 and 0.3;
* the forward apply (affine_relu_dropout) against fp64 BN -> ReLU -> dropout with the mask of dropout_mask;
* the backward, three paths (bn_act_bwd; gemm_tf32x3_bnbwd + bn_act_bwd_apply; gemm_tf32x3_bnbwd_bits + apply) against
  fp64 autograd given the forward's ReLU / dropout decisions.  The bound propagates the measured error of the mean and
  invstd the kernels were given (the x̂ term, which grows with mean/std), the slot chains and every fp32 rounding;
* row-sharded (dist.py, hybrid.py R layout) and column-sharded (hybrid.py C layout) compositions on one GPU, and the
  16-byte alignment refusals of the two backward entry points.

u = 2^-24, gamma(L) = L·u / (1 - L·u) (Higham §3.1); ud = 2^-53 for the fp64 stages.  Each family prints its worst ratio
error / bound.  On an H100 80GB HBM3 at a 700 W power limit: end-to-end invstd 0.7 (GAT) and 1.00 where a column's var
clamps to 0 inside its interval, producers' slots at most 0.60, finalize against its slots 0.999, dY 0.98 (bnbwd at
mean/std 30), dgamma 0.90, row-sharded dY 0.91, column-sharded dY 0.71, running statistics 0.08; the fp32 finalize
restatement exceeds its bound by at least 20x (mean/std 10) and up to 1e6x."""
import math

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops
from efficient_gnns_b200.sparse import CsrGraph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

U = 2.0 ** -24
UD = 2.0 ** -53
EPS = 1e-5
EPS32 = float(torch.tensor(EPS, dtype=torch.float32))
INV_SQRT_EPS32 = float(torch.tensor(1.0 / math.sqrt(EPS32), dtype=torch.float32))
CANARY = 0x7FC0DEAD          # a quiet NaN with a payload: outside an output it must survive bit for bit
DEV = "cuda"
FIN_GROUPS = 64              # bn_finalize / partial_reduce: slot j goes to group j % 64, then the 64 groups in order
ROWS_THREADS = 256           # dense_rows.cu

WORST = {}


def _record(family: str, r: float) -> None:
    assert r <= 1.0, (family, r)
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst bound ratio per case: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _gamma(n, u=U):
    n = torch.as_tensor(n, dtype=torch.float64)
    return n * u / (1 - n * u)


def _gd(n):
    return _gamma(n, UD)


def _ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound; a zero bound demands an exact result."""
    assert bool(torch.isfinite(out).all()), "non-finite output"
    err = (out.double() - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=err.device).expand_as(err)
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def _interval_ratio(out: torch.Tensor, ref: torch.Tensor, lo: torch.Tensor, hi: torch.Tensor) -> float:
    """How far out - ref goes towards the edge of [lo, hi] on its side (<= 1 inside)."""
    assert bool(torch.isfinite(out).all()), "non-finite output"
    e = out.double() - ref
    up, dn = (hi - ref).clamp_min(0), (ref - lo).clamp_min(0)
    r = torch.where(e >= 0, torch.where(up > 0, e / up, torch.where(e > 0, math.inf, 0.0)),
                    torch.where(dn > 0, -e / dn, math.inf))
    return float(r.max())


def _canary(*shape) -> torch.Tensor:
    return torch.full(shape, CANARY, dtype=torch.int32, device=DEV).view(torch.float32)


def _is_canary(t: torch.Tensor) -> bool:
    return bool((t.contiguous().view(torch.int32) == CANARY).all())


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(seed)


def _ceil(a, b):
    return -(-a // b)


def _p32(p: float) -> float:
    return float(torch.tensor(p, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------ chain lengths
def L_rows(n: int, slots: int, K: int) -> int:
    """col_stats4_kernel / bn_act_bwd_reduce_kernel / bn_act_bwd_apply_kernel: a slot holds per = ceil(n / slots) rows;
    a thread adds every rows_per_iter-th of them (ceil(per / rpi) terms), then reduce_store_2xK adds the rpi row groups in
    order: ceil(per / rpi) + rpi, and never more than the per terms of the slot."""
    per = max(_ceil(n, slots), 1)
    rpi = ROWS_THREADS // (K // 4)
    return min(per, _ceil(per, rpi) + rpi)


def L_fin(slots: int) -> int:
    """bn_finalize / partial_reduce / the backward finalize: fp64, ceil(slots / 64) terms per group, then 64 groups."""
    return _ceil(slots, FIN_GROUPS) + FIN_GROUPS


def L_chunks(g: CsrGraph, warps: int, K: int) -> int:
    """SpMM and GAT epilogues: main slot c sums the rows of chunks [c·warps, (c+1)·warps) (one warp per chunk, then the warps
    in order); a hub slot holds one row.  The bound counts the rows of the fullest slot — any order of m terms is within
    gamma(m) — and, for the multi-slab SpMM (K > 512, statistics by col_stats_kernel: one sequential chain per column of
    ceil(n / slots) rows), that chain."""
    cr = g.chunk_rowptr.cpu().long()
    starts = cr[0:g.n_chunks:warps]
    ends = cr[torch.clamp(torch.arange(0, g.n_chunks, warps) + warps, max=g.n_chunks)]
    L = int((ends - starts).max()) + warps if g.n_chunks else 1
    slots = _ceil(g.n_chunks, warps) + g.n_hub
    return max(L, _ceil(g.n_rows, slots))


def L_gemm(M: int, N: int) -> int:
    """3xTF32 GEMM statistics epilogue: slot = (CTA, consumer warp); a warp owns 16 rows of each 128-row tile, and a CTA
    takes ceil(tiles / grid) tiles (persistent, grid = min(tiles, SMs)).  The bound counts the 16 · ceil(tiles / grid)
    terms of a slot (any order)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = _ceil(M, 128) * _ceil(N, 128)
    return 16 * _ceil(tiles, min(tiles, sms))


# ------------------------------------------------------------------------------------------------------ statistics model
def _fp32_finalize(partial: torch.Tensor, n: int):
    """A subtly wrong finalize, restated on the CPU: the slots added in fp32 in slot order, var = q/n - mean² in fp32."""
    P = partial.cpu()
    s, q = P[0, 0].clone(), P[0, 1].clone()
    for j in range(1, P.shape[0]):
        s += P[j, 0]
        q += P[j, 1]
    mean = s / n
    var = torch.clamp(q / n - mean * mean, min=0.0)
    return mean, 1.0 / torch.sqrt(var + EPS32)


def stage_c(Y: torch.Tensor, L: int, Lf: int, gamma, beta) -> dict:
    """Y -> (mean, invstd, scale, shift): fp64 references from the fp32 rows and their bounds.  The slots err by gamma(L) of
    Σ|y| and of Σy², the finalize's fp64 chain by gd(Lf + 4); var = q/n - mean² then errs by
        e_var = g·Σy²/n + 2|mean|·e_mean + e_mean² (+ 4 ud of Σy²/n + mean²),
    the (mean/std)² growth.  invstd lies in [lo, hi]; scale = fp32(gamma·invstd); shift = fp32(beta - mean_out·scale)."""
    n = Y.shape[0]
    Yd = Y.double()
    S, Q, A = Yd.sum(0), (Yd * Yd).sum(0), Yd.abs().sum(0)
    mean = S / n
    var = ((Yd - mean) ** 2).sum(0) / n                     # two-pass: the reference carries no cancellation of its own
    g, b = gamma.double(), beta.double()
    gl = _gamma(L) + _gd(Lf + 4)
    e_mean = gl * A / n + UD * mean.abs()
    e_var = gl * Q / n + 2 * mean.abs() * e_mean + e_mean * e_mean + 4 * UD * (Q / n + mean * mean)
    inv = 1 / torch.sqrt(var + EPS32)
    lo = (1 - U) * (1 - 4 * UD) / torch.sqrt(var + e_var + EPS32)
    hi = (1 + U) * (1 + 4 * UD) / torch.sqrt((var - e_var).clamp_min(0) + EPS32)
    e_mo = e_mean + U * (mean.abs() + e_mean)                       # mean_out: fp32 rounding
    e_inv = torch.maximum(hi - inv, inv - lo)
    sc = g * inv
    e_sc = g.abs() * e_inv + U * g.abs() * (inv + e_inv)
    e_t = e_mo * (sc.abs() + e_sc) + mean.abs() * e_sc             # mean_out·scale against mean·(gamma·invstd)
    e_sh = e_t + U * (b.abs() + (mean * sc).abs() + e_t) + U * (mean.abs() + e_mo) * (sc.abs() + e_sc)
    return dict(S=S, Q=Q, A=A, mean=mean, var=var, e_mean=e_mean, e_var=e_var, e_mo=e_mo, inv=inv, lo=lo, hi=hi,
                e_inv=e_inv, sc=sc, e_sc=e_sc, sh=b - mean * sc, e_sh=e_sh)


def running_step(Y: torch.Tensor, c: dict, momentum: float, rm0, rv0, e_rm, e_rv):
    """Bounds after one finalize call on the running statistics, given the bounds e_rm, e_rv before it:
      rm' = (1-m32) rm + m32·mean_out, rv' = (1-m32) rv + m32·fp32(var·n/(n-1)); four fp32 roundings each, the fp32
      momentum m32 against the reference's m, and the statistics' own error (stage C)."""
    n = Y.shape[0]
    dm = abs(_p32(momentum) - momentum)
    mean, var_u = c["mean"], c["var"] * n / (n - 1)
    e_rm = ((1 - momentum) * e_rm + momentum * c["e_mo"] + dm * (rm0.abs() + mean.abs())
            + 4 * U * ((1 - momentum) * rm0.abs() + momentum * mean.abs()))
    e_rv = ((1 - momentum) * e_rv + momentum * c["e_var"] * n / (n - 1) + dm * (rv0.abs() + var_u)
            + 4 * U * ((1 - momentum) * rv0.abs() + momentum * var_u) + U * var_u)
    return e_rm, e_rv


def check_stats(case: str, Y: torch.Tensor, partial: torch.Tensor, n: int, L: int, gamma, beta, bn=None, Lf=None,
                expect_fp32_fails: bool = False):
    """Stages A, B, C of the module docstring for one producer call.  Y: the fp32 rows the producer wrote (the rows the
    statistics are over); partial: its [slots, 2, K] fp32 slots (or the combined sums of a sharded run); bn: the [4, K]
    finalize output (computed here when None).  Returns bn."""
    slots, _, K = partial.shape
    Lf = L_fin(slots) if Lf is None else Lf
    if bn is None:
        bn = ops.bn_finalize(partial, n, gamma, beta, EPS32, 0.1)
    c = stage_c(Y, L, Lf, gamma, beta)
    out = bn.double()

    # A. the producer's slots (the reference sums in fp64: gd(n + slots) of the magnitudes)
    Pd = partial.double()
    gA = _gamma(L) + _gd(n + slots)
    _record(f"{case} slots", max(_ratio(Pd[:, 0].sum(0), c["S"], gA * c["A"]), _ratio(Pd[:, 1].sum(0), c["Q"], gA * c["Q"])))

    # B. finalize from the same slots.  The kernel (chain Lf) and the fp64 reference (chain <= slots) each err by
    #    e_m1 = gd·Σ|s_j|/n + ud|mean|,  e_v1 = gd·Σq_j/n + 2|mean|·e_m1 + e_m1² + 4 ud (q/n + mean²);
    #    the outputs then take their fp32 rounding (invstd: fp64 sqrt and division, 4 ud, then u).
    ps, pq = Pd[:, 0].sum(0), Pd[:, 1].sum(0)
    As, Aq = Pd[:, 0].abs().sum(0), Pd[:, 1].abs().sum(0)
    m_b = ps / n
    v_b = pq / n - m_b * m_b
    gB = _gd(max(Lf, slots + FIN_GROUPS))
    e_m1 = gB * As / n + UD * m_b.abs()
    e_m = 2 * e_m1
    e_v = 2 * (gB * Aq / n + 2 * m_b.abs() * e_m1 + e_m1 * e_m1 + 4 * UD * (pq / n + m_b * m_b))
    inv_b = 1 / torch.sqrt(v_b.clamp_min(0) + EPS32)
    lo = (1 - U) * (1 - 8 * UD) / torch.sqrt(v_b.clamp_min(0) + e_v + EPS32)
    hi = (1 + U) * (1 + 8 * UD) / torch.sqrt((v_b - e_v).clamp_min(0) + EPS32)
    _record(f"{case} finalize mean", _ratio(out[0], m_b, e_m + U * (m_b.abs() + e_m)))
    _record(f"{case} finalize invstd", _interval_ratio(out[1], inv_b, lo, hi))
    if expect_fp32_fails:
        _, i32 = _fp32_finalize(partial, n)
        r32 = _interval_ratio(i32.to(DEV).double(), inv_b, lo, hi)
        assert r32 > 1.0, f"{case}: an fp32 finalize stays within the bound (ratio {r32:.3g}): the bound cannot see it"
        key = f"{case} fp32-finalize (least ratio, must exceed 1)"
        WORST[key] = min(WORST.get(key, math.inf), r32)

    # C. end to end from Y
    _record(f"{case} mean", _ratio(out[0], c["mean"], c["e_mo"]))
    _record(f"{case} invstd", _interval_ratio(out[1], c["inv"], c["lo"], c["hi"]))
    _record(f"{case} scale", _ratio(out[2], c["sc"], c["e_sc"]))
    _record(f"{case} shift", _ratio(out[3], c["sh"], c["e_sh"]))
    # the var < 0 clamp: invstd never exceeds fp32(1/sqrt(eps)); exact zero columns give exactly that, mean 0, shift beta
    assert bool((bn[1] <= INV_SQRT_EPS32).all()), f"{case}: invstd above 1/sqrt(eps): the var < 0 clamp is missing"
    z = (Y == 0).all(0)
    if bool(z.any()):
        assert bool((bn[0][z] == 0).all()) and bool((bn[1][z] == INV_SQRT_EPS32).all()), f"{case}: zero column not exact"
        assert _bits_equal(bn[3][z], beta[z]), f"{case}: shift of a zero column is not beta"
        assert _bits_equal(bn[2][z], (gamma[z] * INV_SQRT_EPS32)), f"{case}: scale of a zero column"
    return bn


def _stats_input(n: int, K: int, ratio: float, std: float, seed: int) -> torch.Tensor:
    """mean + std·z in fp32 with mean = ratio·std; column 1 all zero, column 2 a constant 0.1, column 3 a constant -1e3/3
    (non-dyadic: q/n - mean² is not exact and may come out negative)."""
    Y = (ratio * std + std * torch.randn(n, K, generator=_gen(seed), device=DEV)).float()
    Y[:, 1] = 0.0
    if K > 2:
        Y[:, 2] = 0.1
    if K > 3:
        Y[:, 3] = -1e3 / 3
    return Y


def _affine(K: int, seed: int):
    g = _gen(seed + 1)
    return (torch.rand(K, generator=g, device=DEV) + 0.5), torch.randn(K, generator=g, device=DEV)


RATIOS = (0.0, 1.0, 10.0, 100.0, 1000.0)
STDS = (1e-3, 1.0, 1e3)


# ========================================================================== 1. statistics -> finalize, every producer
@pytest.mark.parametrize("n,K", [(2, 4), (3, 12), (255, 40), (257, 1024), (20_000, 256), (20_000, 12), (169_343, 40),
                                 (169_343, 256)])
def test_col_stats_finalize(n, K):
    """col_stats (slots = rows_slots(n): 1 .. 528, below and above the finalize's 64 groups) over mean/std x std."""
    slots = ops.rows_slots(n)
    L = L_rows(n, slots, K)
    gamma, beta = _affine(K, n + K)
    for i, ratio in enumerate(RATIOS):
        for j, std in enumerate(STDS):
            Y = _stats_input(n, K, ratio, std, 1000 * n + 10 * i + j)
            part = ops.col_stats(Y)
            check_stats(f"col_stats r{ratio:g}", Y, part, n, L, gamma, beta,
                        expect_fp32_fails=ratio >= 10 and n >= 255 and K >= 12)


def _graph(n: int, seed: int, hubs: bool = True) -> CsrGraph:
    """n rows over n sources, degrees 1..24 (every row has a neighbour, so a mean aggregation keeps the inputs' offset),
    and, with hubs, four rows of degree 600 (above the default hub threshold: their statistics take hub slots)."""
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(1, 25, (n,), generator=g)
    if hubs:
        deg[torch.tensor([0, n // 3, n // 2, n - 1])] = 600
    rowptr = torch.zeros(n + 1, dtype=torch.int64)
    rowptr[1:] = torch.cumsum(deg, 0)
    col = torch.randint(0, n, (int(rowptr[-1]),), generator=g)
    return CsrGraph(rowptr.to(DEV, torch.int32), col.to(DEV, torch.int32), None, n, n).build_plan()


@pytest.mark.parametrize("K", [40, 256, 516])
@pytest.mark.parametrize("ratio", [0.0, 10.0, 100.0])
def test_spmm_stats_finalize(K, ratio):
    """SpMM fused statistics: the register path (K = 40), a bulk / slab path (K = 256), the multi-slab col_stats_kernel
    (K = 516).  Y = mean aggregation of offset inputs, so the output columns keep mean/std ≈ ratio·sqrt(deg)."""
    n = 20_000
    G = _graph(n, 7)
    x = (ratio + torch.randn(n, K, generator=_gen(K), device=DEV)).float()
    part = torch.empty(ops.stat_slots(G), 2, K, device=DEV)
    Y = ops.spmm_csr(G, x, "mean", stat_partial=part)
    gamma, beta = _affine(K, K)
    check_stats(f"spmm K{K} r{ratio:g}", Y, part, n, L_chunks(G, 8, K), gamma, beta, expect_fp32_fails=ratio >= 10)


@pytest.mark.parametrize("M,N", [(257, 64), (20_000, 128), (169_343, 256)])
@pytest.mark.parametrize("accumulate", [False, True])
def test_gemm_stats_finalize(M, N, accumulate):
    """gemm_tf32x3_stats: C = A·B^T + bias, or C += A·B^T (SAGE's lin_l(mean) + lin_r(x)); statistics of the final C."""
    Kin = 128
    g = _gen(M + N)
    a = torch.randn(M, Kin, generator=g, device=DEV)
    w = torch.randn(N, Kin, generator=g, device=DEV) * 0.1
    hi, lo = ops.split_tf32(w)
    part = torch.empty(ops.gemm_stat_slots(M, N), 2, N, device=DEV)
    if accumulate:
        out = (30.0 + torch.randn(M, N, generator=g, device=DEV)).float()
        Y = ops.gemm_tf32x3_stats(a, hi, lo, None, out, part, accumulate=True)
    else:
        bias = torch.full((N,), 30.0, device=DEV)
        Y = ops.gemm_tf32x3_stats(a, hi, lo, bias, torch.empty(M, N, device=DEV), part)
    gamma, beta = _affine(N, M)
    check_stats(f"gemm acc{int(accumulate)}", Y, part, M, L_gemm(M, N), gamma, beta, expect_fp32_fails=M >= 20_000)


def test_gat_stats_finalize_padded_heads():
    """gat_aggregate_epi statistics at the arxiv GAT engine's padded width: 3 heads of 250 stored as 3 x 256.  The padding
    columns are all zero, so their statistics, mean, invstd, scale and shift must be exact."""
    n, H, D, Dr = 20_000, 3, 256, 250
    K = H * D
    G = _graph(n, 11)
    deg = (G.rowptr[1:] - G.rowptr[:-1]).long()
    a = (1.0 / deg.float()).repeat_interleave(deg).unsqueeze(1).expand(-1, H).contiguous()
    ft = (20.0 + torch.randn(n, H, D, generator=_gen(5), device=DEV)).float()
    ft[:, :, Dr:] = 0.0
    ft = ft.view(n, K)
    part = torch.empty(ops.gat_stat_slots(G), 2, K, device=DEV)
    Y = ops.gat_aggregate_epi(G, None, a, ft, torch.empty(n, K, device=DEV), H, stat_partial=part)
    assert bool((Y.view(n, H, D)[:, :, Dr:] == 0).all())
    gamma, beta = _affine(K, 3)
    check_stats("gat K768", Y, part, n, L_chunks(G, 8, K), gamma, beta, expect_fp32_fails=True)


# ========================================================================== 2. running statistics
@pytest.mark.parametrize("momentum", [0.1, 0.3])
@pytest.mark.parametrize("n,K,ratio", [(257, 40, 1.0), (20_000, 256, 10.0)])
def test_running_stats_five_steps(momentum, n, K, ratio):
    """Five successive finalize calls update running_mean / running_var (unbiased) like torch.nn.BatchNorm1d in double,
    within the bound running_step carries from call to call."""
    slots = ops.rows_slots(n)
    L = L_rows(n, slots, K)
    gamma, beta = _affine(K, 0)
    ref = torch.nn.BatchNorm1d(K, eps=EPS32, momentum=momentum).double().to(DEV).train()
    rm, rv = torch.zeros(K, device=DEV), torch.ones(K, device=DEV)
    e_rm = torch.zeros(K, dtype=torch.float64, device=DEV)
    e_rv = torch.zeros(K, dtype=torch.float64, device=DEV)
    for step in range(5):
        Y = (ratio * (step + 1) + torch.randn(n, K, generator=_gen(step), device=DEV) * (step + 1)).float()
        rm0, rv0 = ref.running_mean.clone(), ref.running_var.clone()
        ops.bn_finalize(ops.col_stats(Y), n, gamma, beta, EPS32, momentum, rm, rv)
        ref(Y.double())
        e_rm, e_rv = running_step(Y, stage_c(Y, L, L_fin(slots), gamma, beta), momentum, rm0, rv0, e_rm, e_rv)
        _record(f"running mean m{momentum}", _ratio(rm, ref.running_mean, e_rm))
        _record(f"running var m{momentum}", _ratio(rv, ref.running_var, e_rv))


# ========================================================================== 3. forward apply
@pytest.mark.parametrize("n,K,p,ratio", [(3001, 256, 0.5, 10.0), (500, 40, 0.3, 1.0), (257, 1024, 0.0, 0.0)])
def test_affine_relu_dropout_against_fp64_bn(n, K, p, ratio):
    """out = dropout(relu(y·scale + shift)) with finalize's scale / shift.
    Against fp64 of the same affine map: fmaf (u), relu, the product with fp32(1/(1-p)) (2u): 3u·|y·scale + shift|.
    Against fp64 BN -> ReLU -> dropout: plus |y|·e_scale + e_shift from stage C."""
    Y = (ratio + torch.randn(n, K, generator=_gen(n), device=DEV)).float()
    gamma, beta = _affine(K, n)
    slots = ops.rows_slots(n)
    bn = ops.bn_finalize(ops.col_stats(Y), n, gamma, beta, EPS32, 0.1)
    out = ops.affine_relu_dropout(Y, bn[2], bn[3], True, p, seed=3, offset=1)
    keep = (ops.dropout_mask(n, K, p, 3, 1).double() if p > 0 else torch.ones(n, K, dtype=torch.float64, device=DEV))
    ik = 1.0 / (1.0 - _p32(p))
    Yd = Y.double()
    x = Yd * bn[2].double() + bn[3].double()
    _record("apply (own scale/shift)", _ratio(out, torch.relu(x) * keep * ik, 3 * U * x.abs() * keep * ik))
    plain = ops.affine_relu_dropout(Y, bn[2], bn[3], relu=False, p=0.0)     # BN alone: one fmaf
    _record("apply (no relu, no dropout)", _ratio(plain, x, U * x.abs()))
    # fp64 BN -> ReLU -> dropout from the exact statistics: y·scale + shift - z = y·(scale - sc) + (shift - sh)
    c = stage_c(Y, L_rows(n, slots, K), L_fin(slots), gamma, beta)
    z = (Yd - c["mean"]) * c["inv"] * gamma.double() + beta.double()
    bound = (Yd.abs() * c["e_sc"] + c["e_sh"] + 3 * U * x.abs()) * keep * ik
    _record("apply vs fp64 BN", _ratio(out, torch.relu(z) * keep * ik, bound))


# ========================================================================== 4. backward
def _bwd_reference(Y, x_out, d_out, gamma, p):
    """fp64 autograd of z = BN(y) with the forward's ReLU / dropout decisions ([x_out > 0] / (1-p)) injected."""
    M = (x_out > 0).double() / (1.0 - _p32(p))
    yr = Y.double().requires_grad_(True)
    gr = gamma.double().requires_grad_(True)
    br = torch.zeros_like(gr).requires_grad_(True)
    mean, var = yr.mean(0), yr.var(0, unbiased=False)
    xhat = (yr - mean) / torch.sqrt(var + EPS32)
    ((xhat * gr + br) * M * d_out.double()).sum().backward()
    dz = d_out.double() * M
    return yr.grad, gr.grad, br.grad, dz, xhat.detach(), mean.detach(), (1 / torch.sqrt(var + EPS32)).detach()


def bwd_bounds(Y, dz, xhat, mean, inv, mean_k, inv_k, gamma, n_norm, L, Lf, L_apply, Lf_apply, exact_dz):
    """Elementwise bound of dY and per-column bounds of dgamma, dbeta and the local dbias, propagated from
      e_mu = |mean_k - mean|, e_is = |invstd_k - invstd| (the inputs the backward was given, measured),
      e_dz = 2u|dz| (the product with fp32(1/(1-p)); 0 when exact),
      x̂_k = fp32(fp32(y - mean_k)·invstd_k):  e_x = |y - mean|·e_is + e_mu·(is + e_is) + 2u(|y - mean| + e_mu)(is + e_is),
      s = Σ dz, q = Σ dz·x̂_k: fp32 slot chains L, fp64 finalize Lf,
      c1 = fp32(gamma·invstd_k), c2 = fp32(s/n), c3 = fp32(q/n),
      dY = c1·(dz - c2 - x̂_k·c3): three fp32 roundings inside (3u of the magnitudes) and one for the product."""
    Yd = Y.double()
    g = gamma.double()
    e_mu, e_is = (mean_k.double() - mean).abs(), (inv_k.double() - inv).abs()
    adz = dz.abs()
    e_dz = torch.zeros_like(dz) if exact_dz else 2 * U * adz
    D = (Yd - mean).abs()
    e_x = D * e_is + e_mu * (inv + e_is) + 2 * U * (D + e_mu) * (inv + e_is)
    xa = xhat.abs()
    gs = _gamma(L) + _gd(Lf)
    s_ref, q_ref = dz.sum(0), (dz * xhat).sum(0)
    e_s = e_dz.sum(0) + gs * (adz + e_dz).sum(0)
    e_q = (adz * e_x + e_dz * (xa + e_x)).sum(0) + gs * ((adz + e_dz) * (xa + e_x)).sum(0)
    e_dbeta = e_s + U * (s_ref.abs() + e_s)
    e_dgamma = e_q + U * (q_ref.abs() + e_q)
    c2, c3 = s_ref / n_norm, q_ref / n_norm
    e_c2 = e_s / n_norm + U * (c2.abs() + e_s / n_norm)
    e_c3 = e_q / n_norm + U * (c3.abs() + e_q / n_norm)
    c1 = g * inv
    e_c1 = g.abs() * e_is + U * g.abs() * (inv + e_is)
    T = dz - c2 - xhat * c3
    M1 = adz + e_dz + c2.abs() + e_c2
    M3 = (xa + e_x) * (c3.abs() + e_c3)
    e_T = e_dz + e_c2 + xa * e_c3 + (c3.abs() + e_c3) * e_x + 3 * U * (M1 + M3)
    e_d = (c1.abs() + e_c1) * e_T + T.abs() * e_c1 + U * (c1.abs() + e_c1) * (T.abs() + e_T)
    d_ref = c1 * T
    e_dbias = e_d.sum(0) + (_gamma(L_apply) + _gd(Lf_apply)) * (d_ref.abs() + e_d).sum(0)
    e_dbias = e_dbias + U * (d_ref.sum(0).abs() + e_dbias)
    return e_d, e_dgamma, e_dbeta, e_dbias, d_ref


def _forward(Y, gamma, beta, p, seed=1):
    n, K = Y.shape
    bn = ops.bn_finalize(ops.col_stats(Y), n, gamma, beta, EPS32, 0.1)
    x_out = ops.affine_relu_dropout(Y, bn[2], bn[3], True, p, seed=seed, offset=0)
    return bn, x_out


@pytest.mark.parametrize("n,K,p,ratio", [(2000, 64, 0.0, 0.0), (3001, 256, 0.5, 10.0), (500, 40, 0.3, 1.0),
                                         (20_000, 256, 0.5, 30.0), (257, 1024, 0.5, 3.0), (169_343, 256, 0.5, 3.0)])
def test_bn_act_bwd(n, K, p, ratio):
    g = _gen(n + K)
    Y = (ratio + torch.randn(n, K, generator=g, device=DEV) * 2).float()
    gamma, beta = _affine(K, K)
    d_out = torch.randn(n, K, generator=g, device=DEV)
    bn, x_out = _forward(Y, gamma, beta, p)
    d_y, d_gamma, d_beta, d_bias = ops.bn_act_bwd(d_out, x_out, Y, bn[0], bn[1], gamma, p)
    gy, gg, gb, dz, xhat, mean, inv = _bwd_reference(Y, x_out, d_out, gamma, p)
    slots = ops.rows_slots(n)
    L = L_rows(n, slots, K)
    e_d, e_dg, e_db, e_dbias, d_ref = bwd_bounds(Y, dz, xhat, mean, inv, bn[0], bn[1], gamma, n, L, L_fin(slots), L,
                                                 L_fin(slots), exact_dz=p in (0.0, 0.5))
    _record(f"bn_act_bwd dY r{ratio:g}", _ratio(d_y, gy, e_d))
    _record("bn_act_bwd dgamma", _ratio(d_gamma, gg, e_dg))
    _record("bn_act_bwd dbeta", _ratio(d_beta, gb, e_db))
    _record("bn_act_bwd dbias", _ratio(d_bias, gy.sum(0), e_dbias))


def _dyadic(shape, g, lo=-4, hi=4, q=3):
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float() * 2.0 ** -q


@pytest.mark.parametrize("bits", [False, True])
@pytest.mark.parametrize("n,K,p,ratio", [(3001, 256, 0.5, 10.0), (20_000, 128, 0.5, 1.0), (777, 256, 0.0, 30.0)])
def test_bnbwd_gemm_then_apply(bits, n, K, p, ratio):
    """dz from the input-gradient GEMM's epilogue (gemm_tf32x3_bnbwd, or _bits with the mask from the keep bits and
    y·scale + shift), then bn_act_bwd_apply(Xout = None).  The GEMM operands are multiples of 1/8 in [-1/2, 1/2] over 64
    terms: exact in tf32 and every partial sum exact in fp32, so dOut is exact and only BatchNorm is under test.
    dY written over dOut in place (allowed by the C ABI) must be bit-identical to the separate output."""
    Kin = 64
    g = _gen(n + K + int(bits))
    Y = (ratio + torch.randn(n, K, generator=g, device=DEV) * 2).float()
    gamma, beta = _affine(K, K + 1)
    a, w = _dyadic((n, Kin), g), _dyadic((K, Kin), g)
    hi, lo = ops.split_tf32(w)
    assert bool((lo == 0).all())
    d_out = (a.double() @ w.double().t()).float()       # exact: multiples of 2^-6 below 2^5
    bn = ops.bn_finalize(ops.col_stats(Y), n, gamma, beta, EPS32, 0.1)
    slots_g = ops.gemm_stat_slots(n, K)
    part = torch.empty(slots_g, 2, K, device=DEV)
    dz_k = torch.empty(n, K, device=DEV)
    if bits:
        kb = ops.dropout_bits(torch.empty(1, n, _ceil(K, 32), dtype=torch.int32, device=DEV), p, 5, 0, K=K)[0]
        x_out = ops.affine_relu_bits(Y, kb, bn[2], bn[3], p)
        ops.gemm_tf32x3_bnbwd_bits(a, hi, lo, dz_k, kb, Y, bn[0], bn[1], bn[2], bn[3], p, part)
    else:
        x_out = ops.affine_relu_dropout(Y, bn[2], bn[3], True, p, seed=5, offset=0)
        ops.gemm_tf32x3_bnbwd(a, hi, lo, dz_k, x_out, Y, bn[0], bn[1], p, part)
    gy, gg, gb, dz, xhat, mean, inv = _bwd_reference(Y, x_out, d_out, gamma, p)
    assert torch.equal(dz_k.double(), dz)               # p in {0, 0.5}: the masked, scaled dz is exact too
    slots = ops.rows_slots(n)
    d_y, d_g, d_b, d_bias = (torch.empty(n, K, device=DEV), torch.empty(K, device=DEV), torch.empty(K, device=DEV),
                             torch.empty(K, device=DEV))
    coef, apart = torch.empty(3, K, device=DEV), torch.empty(slots, 2, K, device=DEV)
    ops.bn_act_bwd_apply(dz_k, None, Y, bn[0], bn[1], gamma, part, n, p, d_y, d_g, d_b, d_bias, apart, coef)
    e_d, e_dg, e_db, e_dbias, _ = bwd_bounds(Y, dz, xhat, mean, inv, bn[0], bn[1], gamma, n, L_gemm(n, K), L_fin(slots_g),
                                             L_rows(n, slots, K), L_fin(slots), exact_dz=True)
    tag = "bnbwd_bits" if bits else "bnbwd"
    _record(f"{tag}+apply dY r{ratio:g}", _ratio(d_y, gy, e_d))
    _record(f"{tag}+apply dgamma", _ratio(d_g, gg, e_dg))
    _record(f"{tag}+apply dbeta", _ratio(d_b, gb, e_db))
    _record(f"{tag}+apply dbias", _ratio(d_bias, gy.sum(0), e_dbias))
    # in place: dY over dOut
    inplace = dz_k.clone()
    d_g2, d_b2, d_bias2 = torch.empty_like(d_g), torch.empty_like(d_b), torch.empty_like(d_bias)
    ops.bn_act_bwd_apply(inplace, None, Y, bn[0], bn[1], gamma, part, n, p, inplace, d_g2, d_b2, d_bias2, apart, coef)
    assert _bits_equal(inplace, d_y) and _bits_equal(d_bias2, d_bias)
    assert _bits_equal(d_g2, d_g) and _bits_equal(d_b2, d_b)


# ========================================================================== 5. row-sharded composition (dist.py, hybrid.py R)
def _blocks(N: int, P: int):
    """Row offsets of P uneven blocks: block 1 holds 3 rows, fewer than the slot count every rank uses; the others share the
    rest in proportion 1 : 2 : ... : P-1."""
    rest = N - 3
    w = torch.arange(1, P, dtype=torch.float64)
    share = (w / w.sum() * rest).floor().long().tolist()
    share[-1] += rest - sum(share)
    sizes = [share[0], 3] + share[1:]
    off = [0]
    for s in sizes:
        off.append(off[-1] + s)
    return off


def _col_stats_slots(y: torch.Tensor, slots: int) -> torch.Tensor:
    n, K = y.shape
    part = torch.empty(slots, 2, K, device=DEV)
    lib.check(lib.load().b200gnn_col_stats_f32(y.data_ptr(), n, K, part.data_ptr(), slots, lib.stream_ptr()), "col_stats")
    return part


@pytest.mark.parametrize("combine", ["allreduce", "gather"])
@pytest.mark.parametrize("P", [2, 3, 8])
def test_row_sharded(P, combine):
    """Each rank: local slots (col_stats, or bn_act_bwd_reduce) -> partial_reduce (fp64 sum rounded to fp32: one more u) ->
    combined over ranks: an fp32 all-reduce in rank order (P - 1 more additions, 1 slot) or a [P, 2, K] gather (summed by
    the fp64 finalize) -> bn_finalize / bn_act_bwd_apply with n_norm = N.  dgamma / dbeta from rank 0, dbias summed over
    the ranks in fp32.  Every rank's mapped activation pass equals the rows of the unsharded pass bit for bit."""
    N, K, p, ratio = 20_000, 256, 0.5, 10.0
    g = _gen(P)
    Y = (ratio + torch.randn(N, K, generator=g, device=DEV) * 2).float()
    gamma, beta = _affine(K, P)
    off = _blocks(N, P)
    S = max(ops.rows_slots(off[r + 1] - off[r]) for r in range(P))
    assert S > 3
    extra = 1 + (P - 1 if combine == "allreduce" else 0)
    L = max(L_rows(off[r + 1] - off[r], S, K) for r in range(P)) + extra
    Lf = L_fin(S) + L_fin(1 if combine == "allreduce" else P)

    def combine_sums(parts):
        s = [ops.partial_reduce(pt) for pt in parts]
        if combine == "allreduce":
            tot = s[0].clone()
            for t in s[1:]:
                tot += t
            return tot.view(1, 2, K)
        return torch.stack(s)

    blocks = [Y[off[r]:off[r + 1]] for r in range(P)]
    sums = combine_sums([_col_stats_slots(b, S) for b in blocks])
    bn = check_stats(f"row-sharded {combine}", Y, sums, N, L, gamma, beta, Lf=Lf)
    # forward activation: per-rank mapped pass (row_offset, and rowmap over a permuted partition) == the unsharded rows
    full = ops.affine_relu_dropout(Y, bn[2], bn[3], True, p, seed=9, offset=2)
    for r, b in enumerate(blocks):
        loc = ops.affine_relu_dropout_mapped(b, bn[2], bn[3], True, p, seed=9, offset=2, row_offset=off[r])
        assert _bits_equal(loc, full[off[r]:off[r + 1]]), f"rank {r}: row_offset pass differs"
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(P)).to(DEV, torch.int32)
    for r in range(P):
        rows = perm[off[r]:off[r + 1]].contiguous()
        loc = ops.affine_relu_dropout_mapped(Y[rows.long()], bn[2], bn[3], True, p, seed=9, offset=2, rowmap=rows)
        assert _bits_equal(loc, full[rows.long()]), f"rank {r}: rowmap pass differs"
    # backward
    d_out = torch.randn(N, K, generator=g, device=DEV)
    parts = []
    for r in range(P):
        pt = torch.empty(S, 2, K, device=DEV)
        ops.bn_act_bwd_reduce(d_out[off[r]:off[r + 1]], full[off[r]:off[r + 1]], blocks[r], bn[0], bn[1], p, pt)
        parts.append(pt)
    bsums = combine_sums(parts)
    d_y = torch.empty(N, K, device=DEV)
    dgs, dbs, dbias = [], [], []
    for r in range(P):
        dg, db, dbi = torch.empty(K, device=DEV), torch.empty(K, device=DEV), torch.empty(K, device=DEV)
        ops.bn_act_bwd_apply(d_out[off[r]:off[r + 1]], full[off[r]:off[r + 1]], blocks[r], bn[0], bn[1], gamma, bsums, N, p,
                             d_y[off[r]:off[r + 1]], dg, db, dbi, parts[r], torch.empty(3, K, device=DEV))
        dgs.append(dg); dbs.append(db); dbias.append(dbi)
    for r in range(1, P):            # every rank forms dgamma / dbeta from the same global sums
        assert _bits_equal(dgs[r], dgs[0]) and _bits_equal(dbs[r], dbs[0])
    dbias_sum = dbias[0].clone()
    for t in dbias[1:]:
        dbias_sum += t
    gy, gg, gb, dz, xhat, mean, inv = _bwd_reference(Y, full, d_out, gamma, p)
    e_d, e_dg, e_db, _, d_ref = bwd_bounds(Y, dz, xhat, mean, inv, bn[0], bn[1], gamma, N, L, Lf, 0, 0, exact_dz=True)
    _record(f"row-sharded {combine} dY", _ratio(d_y, gy, e_d))
    _record(f"row-sharded {combine} dgamma", _ratio(dgs[0], gg, e_dg))
    _record(f"row-sharded {combine} dbeta", _ratio(dbs[0], gb, e_db))
    # dbias: each rank's local column sum (its slot chain + fp64 finalize + fp32 rounding), then P - 1 fp32 additions
    e_bias = torch.zeros(K, dtype=torch.float64, device=DEV)
    mag = torch.zeros(K, dtype=torch.float64, device=DEV)
    for r in range(P):
        sl = slice(off[r], off[r + 1])
        Lr = L_rows(off[r + 1] - off[r], S, K)
        loc = e_d[sl].sum(0) + (_gamma(Lr) + _gd(L_fin(S))) * (d_ref[sl].abs() + e_d[sl]).sum(0)
        loc = loc + U * (d_ref[sl].sum(0).abs() + loc)
        e_bias += loc
        mag += d_ref[sl].sum(0).abs() + loc
    e_bias += _gamma(P - 1) * mag
    _record(f"row-sharded {combine} dbias", _ratio(dbias_sum, gy.sum(0), e_bias))


# ========================================================================== 6. column-sharded composition (hybrid.py C)
@pytest.mark.parametrize("P", [2, 4])
def test_column_sharded(P):
    """Rank q owns columns [q·kc, (q+1)·kc): col_stats and bn_finalize on its slice with gamma, beta and the running
    statistics passed as views into the full vectors; the mapped activation pass with k_global / col_offset; bn_act_bwd
    writing dgamma / dbeta / dbias into views of full gradient vectors.  Every value outside the slice is a NaN canary
    that must survive bit for bit."""
    N, K, p, ratio = 20_000, 256, 0.5, 10.0
    kc = K // P
    g = _gen(100 + P)
    Y = (ratio + torch.randn(N, K, generator=g, device=DEV) * 2).float()
    gamma, beta = _affine(K, P)
    d_out = torch.randn(N, K, generator=g, device=DEV)
    sc_all, sh_all, bns = torch.empty(K, device=DEV), torch.empty(K, device=DEV), []
    for q in range(P):
        cols = slice(q * kc, (q + 1) * kc)
        gam, bet = _canary(K), _canary(K)
        gam[cols], bet[cols] = gamma[cols], beta[cols]
        rm, rv = _canary(K), _canary(K)
        rm[cols], rv[cols] = 0.0, 1.0
        Yc = Y[:, cols].contiguous()
        part = ops.col_stats(Yc)
        bn = ops.bn_finalize(part, N, gam[cols], bet[cols], EPS32, 0.1, rm[cols], rv[cols])
        outside = torch.ones(K, dtype=torch.bool, device=DEV)
        outside[cols] = False
        for t in (gam, bet, rm, rv):
            assert _is_canary(t[outside]), f"rank {q}: a value outside the slice changed"
        slots = ops.rows_slots(N)
        check_stats(f"col-sharded P{P}", Yc, part, N, L_rows(N, slots, kc), gamma[cols], beta[cols], bn=bn)
        ref = torch.nn.BatchNorm1d(kc, eps=EPS32, momentum=0.1).double().to(DEV).train()
        rm0, rv0 = ref.running_mean.clone(), ref.running_var.clone()
        ref(Yc.double())
        zero = torch.zeros(kc, dtype=torch.float64, device=DEV)
        e_rm, e_rv = running_step(Yc, stage_c(Yc, L_rows(N, slots, kc), L_fin(slots), gamma[cols], beta[cols]), 0.1,
                                  rm0, rv0, zero, zero)
        _record(f"col-sharded P{P} running mean", _ratio(rm[cols], ref.running_mean, e_rm))
        _record(f"col-sharded P{P} running var", _ratio(rv[cols], ref.running_var, e_rv))
        sc_all[cols], sh_all[cols] = bn[2], bn[3]
        bns.append((bn, Yc, part))
    full = ops.affine_relu_dropout(Y, sc_all, sh_all, True, p, seed=4, offset=1)
    for q, (bn, Yc, _) in enumerate(bns):
        cols = slice(q * kc, (q + 1) * kc)
        Ac = ops.affine_relu_dropout_mapped(Yc, bn[2], bn[3], True, p, seed=4, offset=1, k_global=K, col_offset=q * kc)
        assert _bits_equal(Ac, full[:, cols]), f"rank {q}: column-block activation differs from the full pass"
        gg, gb, gbias = _canary(K), _canary(K), _canary(K)
        gam = _canary(K)
        gam[cols] = gamma[cols]
        d_y, _, _, _ = ops.bn_act_bwd(d_out[:, cols].contiguous(), Ac, Yc, bn[0], bn[1], gam[cols], p,
                                      d_gamma=gg[cols], d_beta=gb[cols], d_bias=gbias[cols])
        outside = torch.ones(K, dtype=torch.bool, device=DEV)
        outside[cols] = False
        for t in (gg, gb, gbias, gam):
            assert _is_canary(t[outside]), f"rank {q}: a gradient outside the slice changed"
        ry, rg, rb, dz, xhat, mean, inv = _bwd_reference(Yc, Ac, d_out[:, cols], gamma[cols], p)
        slots = ops.rows_slots(N)
        L = L_rows(N, slots, kc)
        e_d, e_dg, e_db, e_dbias, _ = bwd_bounds(Yc, dz, xhat, mean, inv, bn[0], bn[1], gamma[cols], N, L, L_fin(slots), L,
                                                 L_fin(slots), exact_dz=True)
        _record(f"col-sharded P{P} dY", _ratio(d_y, ry, e_d))
        _record(f"col-sharded P{P} dgamma", _ratio(gg[cols], rg, e_dg))
        _record(f"col-sharded P{P} dbeta", _ratio(gb[cols], rb, e_db))
        _record(f"col-sharded P{P} dbias", _ratio(gbias[cols], ry.sum(0), e_dbias))


# ========================================================================== 7. alignment refusals
def _misaligned(t: torch.Tensor) -> torch.Tensor:
    """A contiguous copy of t that starts 4 bytes past a 16-byte boundary."""
    buf = torch.empty(t.numel() + 4, dtype=t.dtype, device=t.device)
    v = buf[1:1 + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 4
    return v


def test_backward_entry_points_refuse_misaligned_operands():
    """bn_act_bwd_reduce and bn_act_bwd_apply read their operands as float4: a view one float into its storage is refused
    with an error before anything is launched."""
    n, K, p = 64, 16, 0.5
    Y = torch.randn(n, K, generator=_gen(0), device=DEV)
    gamma, beta = _affine(K, 0)
    bn, x_out = _forward(Y, gamma, beta, p)
    d_out = torch.randn(n, K, generator=_gen(1), device=DEV)
    mean, inv = bn[0].contiguous(), bn[1].contiguous()
    slots = ops.rows_slots(n)
    part = torch.empty(slots, 2, K, device=DEV)
    ok = dict(d_out=d_out, x_out=x_out, y=Y, mean=mean, invstd=inv)
    ops.bn_act_bwd_reduce(**ok, p=p, partial=part)           # the aligned call runs
    torch.cuda.synchronize()

    def outs():
        return dict(d_y=torch.empty(n, K, device=DEV), d_gamma=torch.empty(K, device=DEV), d_beta=torch.empty(K, device=DEV),
                    d_bias=torch.empty(K, device=DEV), partial=torch.empty(slots, 2, K, device=DEV),
                    coef=torch.empty(3, K, device=DEV))

    ops.bn_act_bwd_apply(**ok, gamma=gamma, sums=part, n_norm=n, p=p, **outs())
    torch.cuda.synchronize()
    for name in ok:
        args = dict(ok)
        args[name] = _misaligned(ok[name])
        before = lib.launch_count()
        with pytest.raises(lib.B200GnnError):
            ops.bn_act_bwd_reduce(**args, p=p, partial=part)
        with pytest.raises(lib.B200GnnError):
            ops.bn_act_bwd_apply(**args, gamma=gamma, sums=part, n_norm=n, p=p, **outs())
        with pytest.raises(lib.B200GnnError):
            ops.bn_act_bwd(args["d_out"], args["x_out"], args["y"], args["mean"], args["invstd"], gamma, p)
        assert lib.launch_count() == before, f"{name}: a kernel was launched"
    for name in ("d_y", "coef"):
        o = outs()
        o[name] = _misaligned(o[name])
        before = lib.launch_count()
        with pytest.raises(lib.B200GnnError):
            ops.bn_act_bwd_apply(**ok, gamma=gamma, sums=part, n_norm=n, p=p, **o)
        assert lib.launch_count() == before, f"{name}: a kernel was launched"
    # the dz form (Xout = NULL) checks the same operands
    o = outs()
    before = lib.launch_count()
    with pytest.raises(lib.B200GnnError):
        ops.bn_act_bwd_apply(_misaligned(d_out), None, Y, mean, inv, gamma, part, n, p, **o)
    assert lib.launch_count() == before
