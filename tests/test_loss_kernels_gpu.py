"""Accuracy contract of the loss kernels (loss_rows.cu, loss_pair.cu, loss_edge.cu), checked through the C ABI against plain
float64 restatements of each pass, computed from the same fp32 inputs the kernel reads (DESIGN.md §2):

* every output element obeys |out - out64| <= (model) · magnitude, the model derived below from fp32 rounding
  (u = 2^-24), the libdevice ulp limits of expf (2 ulp), logf and log1pf (1 ulp), correctly rounded sqrtf and division,
  and the length of the summation chains.  For softmax-type outputs the dominant term is the absolute error of the
  exponent argument, u·(|z_j - zmax| + |lse|)·inv_T, so the bound grows with the logit range, not only with C;
* for a well-conditioned random input every relative bound is below 1e-5 (asserted where the inputs are random);
* the kernels write nothing outside their outputs: dlogits rows outside train_idx and columns [C, ldd), the pitch padding
  of a G-CRD chunk, the tails of the partial buffers of the advertised sizes, all NaN canaries that survive bit for bit;
* repeated calls are bit-identical, and the chunked G-CRD row pass is bit-identical to the single call;
* the transpose is exact, past the 65,535 row-tile limit of gridDim.y.

Worst observed ratio (error / bound) of each family on an H100 80GB HBM3 at a 400 W power limit:
  kd 0.41, bce 0.65, mse 0.44, normalize 0.999, sqnorm/axpy 1.00 (single correctly rounded operations reach their
  half-ulp bound), nce 0.70, gsp 0.90, edge_sim 0.38, lsp_segment 0.50, lsp_values 0.99, edge_sim_bwd 0.98;
  the callers' shapes: ARXIV KD 0.34, MAG 0.30, PPI BCE 0.51, G-CRD 0.36.
Every threshold is either derived in a comment or quotes the H100 measurement it was set from."""
import math

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion, lib, ops

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# ----------------------------------------------------------------------------------------------------------- error model
U = 2.0 ** -24          # unit roundoff of fp32 round to nearest; one ulp of a result is at most 2U relative
EXP = 4 * U             # expf: 2 ulp
LOG = 2 * U             # logf, log1pf: 1 ulp
TINY = 2.0 ** -126      # absolute floor for results that leave the normal range (subnormal, or underflowed to 0)
COS_EPS = float(torch.tensor(1e-8, dtype=torch.float32))
TIGHT = 1e-5            # a well-conditioned random input must get a relative bound below this

CANARY = 0x7FC0DEAD     # a quiet NaN with a payload: outside an output it must survive bit for bit
OK, ERR_UNSUPPORTED = 0, -2

WORST = {}


def _record(family: str, r: float) -> None:
    assert r <= 1.0, (family, r)
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst bound ratio per family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def _pow2(n: int, g: torch.Generator, span: int) -> torch.Tensor:
    """n powers of two 2^e, e uniform in [-span, span]: scaling by them is exact."""
    return torch.exp2(torch.randint(-span, span + 1, (n,), generator=g, device="cuda").double()).float()


def _canary(*shape) -> torch.Tensor:
    return torch.full(shape, CANARY, dtype=torch.int32, device="cuda").view(torch.float32)


def _is_canary(t: torch.Tensor) -> bool:
    return bool((t.contiguous().view(torch.int32) == CANARY).all())


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _bound_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound (<= 1 passes); a zero bound demands an exact result."""
    assert bool(torch.isfinite(out).all()), "non-finite output"
    err = (out.double() - ref).abs()
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def _tight(bound: torch.Tensor, mag: torch.Tensor) -> None:
    m = mag > 0
    assert float((bound[m] / mag[m]).max()) < TIGHT


def _ceil(a, b):
    return -(-a // b)


L = None


def _L():
    global L
    if L is None:
        L = lib.load()
    return L


def _st():
    return lib.stream_ptr()


def _p(t):
    return None if t is None else t.data_ptr()


# ======================================================================================== 1. CE / logit KD (loss_rows.cu)
# kd_rows_kernel, one warp per row, NJ = ceil(C/32) values per lane (NJ in {2, 8, 16, 32}):
#   d_j = z_j - zmax (u|d_j|), se = sum expf(d_j) (positive terms: expf 4u, argument u·H with H = sum_j sm_j|d_j|, an
#   NJ-long lane chain and a 5-level xor tree), lse = logf(se): delta_lse <= u(4 + H + NJ + 5) + 2u|lse|.
#   sm_j = expf(d_j - lse): argument error u|d_j| + u|d_j - lse| + delta_lse, plus expf's 4u, so
#     eps_sm_j <= u (4|d_j| + 3|lse| + 3H + NJ + 13).
#   The tempered softmaxes q (of z/T) and p (of t/T) are the same with d -> d·inv_T (inv_T's rounding folded into the 4).
#   g_j = w_cls (sm_j - [j=y]) + w_kd inv_T (q_j - p_j): w_cls, w_kd, inv_T and the products and differences add 5u of
#   the cross-entropy term and 10u of the KD term.
#   CE_i = (zmax + lse) - z_y: delta_lse + 2u(|zmax| + |lse|) + u|z_y|.
#   KL_i = sum_j p_j (logp_j - logq_j): sum_j p_j [(eps_p + eps_q)(1 + |logp - logq|) + (NJ + 8) u |logp - logq|].
#   The loss sums rows per warp (m = ceil(n_train / (8 grid)) adds), then 8 warps, then fp64: (m + 8) u of sum |term|;
#   the scaling and the final combination add 2u and 5u of the result.
def _kd_nj(C: int) -> int:
    return 2 if C <= 64 else 8 if C <= 256 else 16 if C <= 512 else 32


def _softmax64(d: torch.Tensor, nj: int):
    lse = torch.logsumexp(d, 1, keepdim=True)
    p = torch.exp(d - lse)
    H = (p * d.abs()).sum(1, keepdim=True)
    eps = U * (4 * d.abs() + 3 * lse.abs() + 3 * H + nj + 13)
    return lse, p, H, eps


def _kd_ref(z, t, y, C, alpha, T, n_norm, n_train, grid):
    """fp64 dlogits, losses and their bounds for the train rows z [n, C] (fp32), teacher rows t or None, labels y."""
    nj = _kd_nj(C)
    z = z.double()
    zmax = z.max(1, keepdim=True).values
    d = z - zmax
    lse, sm, H, eps_sm = _softmax64(d, nj)
    oh = torch.zeros_like(z)
    oh.scatter_(1, y[:, None], 1.0)
    zy = z.gather(1, y[:, None])
    nn = float(n_norm if n_norm > 0 else n_train)
    ce = (lse - d.gather(1, y[:, None]))[:, 0]
    ce_b = (U * (4 + H + nj + 5) + 2 * U * lse.abs() + 2 * U * (zmax.abs() + lse.abs()) + U * zy.abs())[:, 0]
    m = _ceil(max(n_train, 1), 8 * grid)
    out = {}
    if t is None:
        w_cls = 1.0 / nn
        out["g"] = w_cls * (sm - oh)
        out["gb"] = w_cls * (sm * eps_sm + 5 * U * (sm - oh).abs() + TINY) + 2.0 ** -147
        mag = w_cls * (sm + oh)
        kl = torch.zeros_like(ce)
        kl_b = torch.zeros_like(ce)
        kl_mag = kl
    else:
        alpha = float(torch.tensor(alpha, dtype=torch.float32))
        T = float(torch.tensor(T, dtype=torch.float32))
        w_cls = (1.0 - alpha) / nn
        w_kd = alpha * T * T / (nn * C) / T
        dT = d / T
        lseT, q, _, eps_q = _softmax64(dT, nj)
        t = t.double()
        tT = (t - t.max(1, keepdim=True).values) / T
        lsteT, p, _, eps_p = _softmax64(tT, nj)
        logq, logp = dT - lseT, tT - lsteT
        out["g"] = w_cls * (sm - oh) + w_kd * (q - p)
        out["gb"] = (w_cls * (sm * eps_sm + 5 * U * (sm - oh).abs()) + w_kd * (q * eps_q + p * eps_p + 10 * U * (q - p).abs())
                     + TINY * (w_cls + w_kd) + 2.0 ** -147)
        mag = w_cls * (sm + oh) + w_kd * (q + p)
        dl = (logp - logq)
        kl = (p * dl).sum(1)
        kl_b = (p * ((eps_p + eps_q) * (1 + dl.abs()) + (nj + 8) * U * dl.abs())).sum(1) + C * TINY
        kl_mag = (p * (1 + logp.abs() + logq.abs())).sum(1)      # KL cancels: its bound is relative to this
    loss_cls = float(ce.sum()) / nn
    b_cls = (float(ce_b.sum()) + (m + 8) * U * float(ce.abs().sum())) / nn + 2 * U * abs(loss_cls)
    loss_kd = float(kl.sum()) / (nn * C)
    b_kd = (float(kl_b.sum()) + (m + 8) * U * float(kl.abs().sum())) / (nn * C) + 3 * U * abs(loss_kd)
    m_cls = float((zmax.abs() + lse.abs() + zy.abs()).sum()) / nn
    m_kd = float(kl_mag.sum()) / (nn * C)
    if t is None:
        loss, b_loss, m_loss = loss_cls, b_cls, m_cls
    else:
        a, b = alpha * T * T, 1.0 - alpha
        loss = a * loss_kd + b * loss_cls
        b_loss = a * b_kd + b * b_cls + 5 * U * (a * abs(loss_kd) + b * abs(loss_cls))
        m_loss = a * m_kd + b * m_cls
    out["loss"] = torch.tensor([loss, loss_cls, loss_kd], dtype=torch.float64, device="cuda")
    out["lb"] = torch.tensor([b_loss, b_cls, b_kd], dtype=torch.float64, device="cuda")
    out["mag"] = mag
    out["lmag"] = torch.tensor([m_loss, m_cls, m_kd], dtype=torch.float64, device="cuda")
    return out


def _kd_inputs(C: int, n_rows: int, g: torch.Generator, extreme: bool = True):
    """Logits at 2^[-6, 3] row scales, saturated rows (|z| up to 1e3); teacher rows with ties; labels in the first and the
    last lane group and at column C - 1."""
    z = torch.randn(n_rows, C, generator=g, device="cuda")
    t = torch.randn(n_rows, C, generator=g, device="cuda") * 2
    if extreme:
        z *= torch.exp2(torch.randint(-6, 4, (n_rows,), generator=g, device="cuda").float())[:, None]
        sat = torch.arange(0, n_rows, 7, device="cuda")
        z[sat] = (torch.randn(len(sat), C, generator=g, device="cuda") * 400).clamp(-1e3, 1e3)
        ties = torch.arange(3, n_rows, 5, device="cuda")
        t[ties] = torch.randint(-2, 3, (len(ties), C), generator=g, device="cuda").float()
        t[5 % n_rows] = 1.5                                     # a teacher row that is all one tie
    y = torch.randint(0, C, (n_rows,), generator=g, device="cuda")
    special = torch.tensor([0, min(31, C - 1), (C - 1) // 32 * 32, max(C - 32, 0), C - 1], device="cuda")
    k = min(n_rows, 40)
    y[:k] = special[torch.arange(k, device="cuda") % len(special)]
    return z, t, y


def _kd_run(z, t, y, train_idx, n_train, C, alpha, T, n_norm, pads=(3, 5, 7), dl_rows=None):
    """One ABI call with z, t placed in canary buffers of pitch C + pad; returns (dlogits buffer, loss buffer, partials,
    grid, rc)."""
    n_rows = z.shape[0]
    lbuf = _canary(n_rows, C + pads[0])
    lbuf[:, :C] = z
    tbuf = None
    if t is not None:
        tbuf = _canary(n_rows, C + pads[1])
        tbuf[:, :C] = t
    ldd = C + pads[2]
    dbuf = _canary(n_rows if dl_rows is None else dl_rows, ldd)
    grid = int(_L().b200gnn_kd_partials(n_train))
    part = _canary(2 * grid + 32)
    loss = _canary(8)
    rc = _L().b200gnn_kd_loss_fwd_bwd_f32(lbuf.data_ptr(), lbuf.stride(0), _p(train_idx), n_train, y.data_ptr(), _p(tbuf),
                                        tbuf.stride(0) if tbuf is not None else 0, C, alpha, T, n_norm, dbuf.data_ptr(), ldd,
                                        loss.data_ptr(), part.data_ptr(), _st())
    torch.cuda.synchronize()
    return dbuf, loss, part, grid, rc


def _kd_check(z, t, y, train_idx, C, alpha, T, n_norm, tight=False, repeat=True):
    n_rows = z.shape[0]
    n_train = n_rows if train_idx is None else train_idx.numel()
    dbuf, loss, part, grid, rc = _kd_run(z, t, y, train_idx, n_train, C, alpha, T, n_norm)
    assert rc == OK
    rows = torch.arange(n_rows, device="cuda") if train_idx is None else train_idx
    ref = _kd_ref(z[rows], None if t is None else t[rows], y[rows], C, alpha, T, n_norm, n_train, grid)
    r = max(_bound_ratio(dbuf[rows, :C], ref["g"], ref["gb"]), _bound_ratio(loss[:3], ref["loss"], ref["lb"]))
    if tight and C > 1:                                  # C = 1: every output is exactly 0
        _tight(ref["gb"], ref["mag"])
        _tight(ref["lb"], ref["lmag"])
    inside = torch.zeros(dbuf.shape, dtype=torch.bool, device="cuda")
    inside[rows, :C] = True
    assert _is_canary(dbuf[~inside]), "dlogits written outside the train rows x [0, C)"
    assert _is_canary(part[2 * grid:]) and bool(torch.isfinite(part[:2 * grid]).all())
    assert _is_canary(loss[3:])
    if repeat:
        dbuf2, loss2, _, _, _ = _kd_run(z, t, y, train_idx, n_train, C, alpha, T, n_norm)
        assert _bits_equal(dbuf2, dbuf) and _bits_equal(loss2, loss)
    return r


KD_C = [1, 2, 31, 32, 33, 40, 64, 65, 121, 255, 256, 257, 349, 511, 512, 513, 1000, 1024]


@pytest.mark.parametrize("C", KD_C)
def test_kd_rows_elementwise(C):
    """Every tiling and its edges; train_idx unsorted / NULL / sorted / one row; T in {0.5, 1, 4}, alpha in {0, 0.9, 1};
    n_norm != n_train; padded pitches with canaries in the logits, the teacher and dlogits."""
    g = _gen(C)
    n_rows = 333
    z, t, y = _kd_inputs(C, n_rows, g)
    unsorted = torch.randperm(n_rows, generator=g, device="cuda")[:200]
    r = _kd_check(z, t, y, unsorted, C, 0.9, 4.0, 0)
    r = max(r, _kd_check(z, None, y, None, C, 0.0, 1.0, 0))                                # CE, train_idx NULL
    r = max(r, _kd_check(z, t, y, unsorted.sort().values[:150], C, 1.0, 0.5, 1000))       # sharded normalisation
    r = max(r, _kd_check(z, t, y, torch.tensor([n_rows - 1], device="cuda"), C, 0.0, 1.0, 0))
    zr, tr, yr = _kd_inputs(C, 64, g, extreme=False)
    r = max(r, _kd_check(zr, tr, yr, None, C, 0.9, 4.0, 0, tight=True))
    _record("kd", r)


@pytest.mark.parametrize("n_rows,n_train,C", [(169_343, 90_941, 40), (20_000, 17_003, 513)])
def test_kd_rows_grid_stride(n_rows, n_train, C):
    """More rows than the 2,112-CTA grid covers in one sweep (ARXIV: 90,941 training rows of 169,343)."""
    g = _gen(n_train)
    z, t, y = _kd_inputs(C, n_rows, g)
    idx = torch.randperm(n_rows, generator=g, device="cuda")[:n_train]
    assert n_train > 8 * int(_L().b200gnn_kd_partials(n_train))
    _record("kd", _kd_check(z, t, y, idx, C, 0.9, 4.0, 0, repeat=False))


def test_kd_rows_no_train_rows_and_unsupported_width():
    """n_train = 0 with a global n_norm (a shard without training rows): the loss is exactly 0 and nothing is written.
    C = 1025 is past the widest tiling and is refused."""
    g = _gen(0)
    z, t, y = _kd_inputs(40, 50, g)
    empty = torch.empty(0, dtype=torch.long, device="cuda")
    dbuf, loss, part, grid, rc = _kd_run(z, t, y, empty, 0, 40, 0.9, 4.0, 1000)
    assert rc == OK
    assert loss[:3].tolist() == [0.0, 0.0, 0.0] and _is_canary(loss[3:])
    assert _is_canary(dbuf) and _is_canary(part[2 * grid:])
    z, t, y = _kd_inputs(1025, 4, g)
    assert _kd_run(z, t, y, None, 4, 1025, 0.9, 4.0, 0)[4] == ERR_UNSUPPORTED


# ============================================================================================ 2. BCE with logits, MSE
# bce_logits_kernel, per element: t = 1/(1 + expf(-target)) for logit targets: 6u t (expf 4u, the add u, the division u)
# plus TINY where the true sigmoid is subnormal.  l = max(z,0) - z t + log1pf(expf(-|z|)): |z| dt + 2u(|z| + |z t|)
# + 8u log1p(.) (log1pf's 2u and the 4u of expf times v/((1+v) log1p v) <= 1.45) + u l.  dz = (sigmoid(z) - t) w:
# w (6u s + dt + 3u |s - t|) + w TINY.  The loss sums k = ceil(n / (256 grid)) elements per thread, a 5-level warp tree
# and 8 warps ((k + 13) u of sum l), then fp64; the cast adds 2u.
# mse_fwd_bwd_kernel: d = a - b (u), d^2 by fma chains: (k + 13 + 2) u of sum d^2; d_a = (2 w / n) d: 3u.
BCE_N = 2 * 1056 * 1024 + 77      # ragged, and more than the capped grid (132 x 8 CTAs) x 256 threads x 4


def _ew_grid_k(n: int):
    """(grid, elements per thread) of the elementwise reductions."""
    grid = int(_L().b200gnn_reduce_slots(n))
    return grid, _ceil(n, 256 * grid)


def _bce_ref(z, target, is_logits, gw, n, k):
    z, tg = z.double(), target.double()
    if is_logits:
        t = torch.sigmoid(tg)
        dt = 6 * U * t + TINY
    else:
        t, dt = tg, torch.zeros_like(tg)
    v = torch.exp(-z.abs())
    lp = torch.log1p(v)
    l = z.clamp_min(0) - z * t + lp
    dl = z.abs() * dt + 2 * U * (z.abs() + (z * t).abs()) + 8 * U * lp + U * l.abs() + TINY
    s = torch.sigmoid(z)
    w = gw / n
    dz = (s - t) * w
    dzb = w * (6 * U * s + dt + 3 * U * (s - t).abs() + TINY) + 2.0 ** -147
    loss = float(l.sum()) / n
    lb = (float(dl.sum()) + (k + 13) * U * float(l.abs().sum())) / n + 2 * U * abs(loss)
    return dz, dzb, loss, lb, w * (s + t)


def _bce_inputs(g, n):
    z = torch.randn(n, generator=g, device="cuda") * 3
    special = torch.tensor([0.0, 1e-30, -1e-30, 20.0, -20.0, 100.0, -100.0], device="cuda")
    z[: 7 * 1000] = special.repeat(1000)
    hard = (torch.rand(n, generator=g, device="cuda") < 0.5).float()
    soft = torch.rand(n, generator=g, device="cuda")
    logit_t = torch.randn(n, generator=g, device="cuda") * 4
    logit_t[:7 * 1000:3] = 100.0
    logit_t[1:7 * 1000:3] = -100.0
    return z, hard, soft, logit_t


def test_bce_logits_elementwise():
    g = _gen(11)
    n = BCE_N
    z, hard, soft, logit_t = _bce_inputs(g, n)
    grid, k = _ew_grid_k(n)
    worst = 0.0
    for target, is_logits in ((hard, 0), (soft, 0), (logit_t, 1)):
        for with_dz in (True, False):
            dz = _canary(n + 16)
            part = _canary(grid + 16)
            loss = _canary(4)
            lib.check(_L().b200gnn_bce_logits_fwd_bwd_f32(z.data_ptr(), target.data_ptr(), is_logits, n, 0.75,
                                                        dz.data_ptr() if with_dz else None, loss.data_ptr(),
                                                        part.data_ptr(), _st()), "bce")
            torch.cuda.synchronize()
            dzr, dzb, lr, lb, mag = _bce_ref(z, target, is_logits, 0.75, n, k)
            worst = max(worst, _bound_ratio(loss[:1], torch.tensor([lr], device="cuda", dtype=torch.float64),
                                            torch.tensor([lb], device="cuda", dtype=torch.float64)))
            if with_dz:
                worst = max(worst, _bound_ratio(dz[:n], dzr, dzb))
                assert _is_canary(dz[n:])
                if not is_logits:
                    _tight(dzb[7000:], mag[7000:])
            else:
                assert _is_canary(dz)
            assert _is_canary(part[grid:]) and _is_canary(loss[1:])
            assert lb / abs(lr) < TIGHT
    _record("bce", worst)


def test_mse_elementwise():
    g = _gen(12)
    worst = 0.0
    for n in (1, 257, BCE_N):
        grid, k = _ew_grid_k(n)
        a = torch.randn(n, generator=g, device="cuda") * _pow2(n, g, 10)
        b = a + torch.randn(n, generator=g, device="cuda") * a.abs() * 0.1
        for with_grad in (True, False):
            da = _canary(n + 16)
            part = _canary(grid + 16)
            loss = _canary(4)
            lib.check(_L().b200gnn_mse_fwd_bwd_f32(a.data_ptr(), b.data_ptr(), n, 1.5, da.data_ptr() if with_grad else None,
                                                 loss.data_ptr(), part.data_ptr(), _st()), "mse")
            torch.cuda.synchronize()
            d = a.double() - b.double()
            lr = float((d * d).sum()) / n
            lb = (k + 15) * U * lr + 2 * U * lr
            assert lb / lr < TIGHT
            worst = max(worst, _bound_ratio(loss[:1], torch.tensor([lr], device="cuda", dtype=torch.float64),
                                            torch.tensor([lb], device="cuda", dtype=torch.float64)))
            if with_grad:
                ref = 3.0 / n * d
                worst = max(worst, _bound_ratio(da[:n], ref, 3 * U * ref.abs()))
                assert _is_canary(da[n:])
            else:
                assert _is_canary(da)
            assert _is_canary(part[grid:]) and _is_canary(loss[1:])
    _record("mse", worst)


# ================================================================================ 3. row normalisation, squared norms
# row_normalize_fwd_kernel: ss = sum x^2 by an m = ceil(F/32) fma chain and a 5-level tree: (m + 5) u relative (positive
# terms); sqrtf: half of that + u; inv = scale / max(nrm, eps): u; out = x inv: u.  max() is continuous, so rows on
# either side of eps obey the same bound.
# row_normalize_bwd_kernel, from the fp32 (out, norm, d_out) it reads: u_k = out_k (1/scale) (2u), dot = sum u g by fma
# chains ((m + 7) u of sum |u g|), and per element inv (g - u dot): inv [|u| dot_err + 3u |u dot| + 3u |g - u dot|] + u.
# Rows with norm < eps take the clamped branch d_out scale/eps (2u): the gradient of clamp_min, which passes none to
# the norm.  accumulate adds u of |d_x_prev + v|.
# row_sqnorm: (m + 5) u relative; its backward 2 x d_out is one rounding; row_axpy fma(alpha coef, x, y): u |alpha coef x|
# + u |y_out|.
NORM_F = [1, 31, 32, 33, 64, 750, 3072]
EPS = float(torch.tensor(1e-12, dtype=torch.float32))    # the fp32 eps the kernels compare with


def _norm_inputs(n: int, F: int, g: torch.Generator) -> torch.Tensor:
    x = torch.randn(n, F, generator=g, device="cuda") * _pow2(n, g, 20)[:, None]
    x[0] = 0                                                    # all-zero row
    if n > 4:
        x[1] *= 1e-14 / float(x[1].norm().clamp_min(1e-30))    # norm in (0, 1e-12)
        x[2] = x[1]
        x[2, 0] = 0.9e-12                                       # just under eps
        x[3, 0] = 0                                             # some exact zeros in a row
    if n > 6:
        x[4] = 0
        x[4, 0] = 1.1e-12                                       # just over eps
        x[5] = 0
        x[5, : min(F, 7)] = 1e-12 / math.sqrt(min(F, 7))          # on eps, within rounding
    return x


def _norm_fwd_ref(x, scale, m):
    x64 = x.double()
    nrm = x64.norm(dim=1, keepdim=True)
    out = x64 * scale / nrm.clamp_min(EPS)
    ob = (0.5 * (m + 5) + 3) * U * out.abs()
    nb = (0.5 * (m + 5) + 1) * U * nrm
    return out, ob, nrm[:, 0], nb[:, 0]


def _norm_bwd_ref(out, norm, d_out, scale, m):
    o, nr, gd = out.double(), norm.double()[:, None], d_out.double()
    uu = o / scale
    dot = (uu * gd).sum(1, keepdim=True)
    dot_err = (m + 7) * U * (uu * gd).abs().sum(1, keepdim=True)
    inv = scale / nr.clamp_min(EPS)
    clamped = nr < EPS
    v = torch.where(clamped, gd * inv, inv * (gd - uu * dot))
    vb = torch.where(clamped, 2 * U * v.abs(),
                     inv * (uu.abs() * dot_err + 3 * U * (uu * dot).abs() + 3 * U * (gd - uu * dot).abs()) + U * v.abs())
    mag = torch.where(clamped, v.abs(), inv * (gd.abs() + uu.abs() * (uu * gd).abs().sum(1, keepdim=True)))
    return v, vb, mag


@pytest.mark.parametrize("n,F", [(257, F) for F in NORM_F] + [(1, 169_343)])
@pytest.mark.parametrize("scale", [1.0, 1.0 / 0.075])
def test_row_normalize_elementwise(n, F, scale):
    """Zero rows, norms in (0, 1e-12) and on either side of eps, the G-CRD scale, accumulate onto a pre-filled d_x, and the
    attention-transfer shape: one row of 169,343 elements normalised by a single warp."""
    g = _gen(n * F + int(scale))
    scale32 = float(torch.tensor(scale, dtype=torch.float32))
    m = _ceil(F, 32)
    x = _norm_inputs(n, F, g)
    out, nrm = _canary(n + 1, F), _canary(n + 1)
    lib.check(_L().b200gnn_row_normalize_fwd_f32(x.data_ptr(), n, F, EPS, scale32, out.data_ptr(), nrm.data_ptr(), _st()), "fwd")
    torch.cuda.synchronize()
    o_ref, ob, n_ref, nb = _norm_fwd_ref(x, scale32, m)
    r = max(_bound_ratio(out[:n], o_ref, ob), _bound_ratio(nrm[:n], n_ref, nb))
    assert _is_canary(out[n:]) and _is_canary(nrm[n:])
    d_out = torch.randn(n, F, generator=g, device="cuda") * _pow2(n, g, 10)[:, None]
    prev = torch.randn(n, F, generator=g, device="cuda")
    for acc in (0, 1):
        dx = _canary(n + 1, F)
        dx[:n] = prev
        lib.check(_L().b200gnn_row_normalize_bwd_f32(out.data_ptr(), nrm.data_ptr(), d_out.data_ptr(), n, F, EPS, scale32,
                                                   dx.data_ptr(), acc, _st()), "bwd")
        torch.cuda.synchronize()
        v, vb, mag = _norm_bwd_ref(out[:n], nrm[:n], d_out, scale32, m)
        if acc:
            v = v + prev.double()
            vb = vb + U * v.abs()
        r = max(r, _bound_ratio(dx[:n], v, vb))
        assert _is_canary(dx[n:])
        if n > 6 and not acc:
            _tight(vb[6:], mag[6:])
    if n > 6:   # the clamped rows really are clamped, with the clamp_min gradient d_out * scale / eps
        small = nrm[:n] < EPS
        assert bool(small[:3].all()) and not bool(small[4]) and bool(small[2])
    _record("normalize", r)


def test_row_normalize_zero_rows_ok():
    x = torch.zeros(1, 4, device="cuda")
    assert _L().b200gnn_row_normalize_fwd_f32(x.data_ptr(), 0, 4, EPS, 1.0, x.data_ptr(), None, _st()) == OK
    assert _L().b200gnn_row_normalize_bwd_f32(x.data_ptr(), x.data_ptr(), x.data_ptr(), 0, 4, EPS, 1.0, x.data_ptr(), 0,
                                              _st()) == OK


@pytest.mark.parametrize("n,F", [(257, F) for F in NORM_F] + [(1, 169_343)])
def test_row_sqnorm_and_axpy(n, F):
    g = _gen(7 * n + F)
    m = _ceil(F, 32)
    x = _norm_inputs(n, F, g)
    out = _canary(n + 1)
    lib.check(_L().b200gnn_row_sqnorm_f32(x.data_ptr(), n, F, out.data_ptr(), _st()), "sqnorm")
    torch.cuda.synchronize()
    ref = (x.double() ** 2).sum(1)
    r = _bound_ratio(out[:n], ref, (m + 5) * U * ref + 2.0 ** -149)
    assert _is_canary(out[n:])
    d_out = torch.randn(n, generator=g, device="cuda") * _pow2(n, g, 10)
    dx = _canary(n * F + 8)
    lib.check(_L().b200gnn_row_sqnorm_bwd_f32(x.data_ptr(), d_out.data_ptr(), n, F, dx.data_ptr(), _st()), "sqnorm_bwd")
    torch.cuda.synchronize()
    ref = 2 * x.double() * d_out.double()[:, None]
    r = max(r, _bound_ratio(dx[:n * F].view(n, F), ref, U * ref.abs() + 2.0 ** -149))
    assert _is_canary(dx[n * F:])
    coef = torch.randn(n, generator=g, device="cuda")
    y0 = torch.randn(n, F, generator=g, device="cuda") * x.abs().max(1).values[:, None]
    y = _canary(n * F + 8)
    y[:n * F] = y0.view(-1)
    lib.check(_L().b200gnn_row_axpy_f32(x.data_ptr(), coef.data_ptr(), n, F, 4.0, y.data_ptr(), _st()), "axpy")
    torch.cuda.synchronize()
    t = 4.0 * coef.double()[:, None] * x.double()
    ref = t + y0.double()
    r = max(r, _bound_ratio(y[:n * F].view(n, F), ref, U * t.abs() + U * ref.abs() + 2.0 ** -149))
    assert _is_canary(y[n * F:])
    _record("sqnorm_axpy", r)


# ========================================================================================== 4. G-CRD rows (InfoNCE)
# nce_rows_kernel, one CTA per row: se = sum expf(Z_j - m) over k = ceil(S/256) terms per thread, a 5-level warp tree and
# 8 warps through another (k + 10 adds), lse = m + logf(se):
#   delta_lse <= u(4 + H + k + 10) + 2u |log se| + u |lse|,   H = sum_j p_j |Z_j - m|;
# dZ_j = (expf(Z_j - lse) - [j = i]) w: w [p_j (u |Z_j - lse| + delta_lse + 4u) + 3u |p_j - [j=i]|] (w = 1/S: u).
# The loss term lse - Z_ii: delta_lse + u |lse - Z_ii|; the fp64 mean of the fp32 terms, cast: 2u.
NCE_S = [1, 2, 255, 256, 257, 901]


def _nce_inputs(rows: int, S: int, g: torch.Generator) -> torch.Tensor:
    z = (torch.rand(rows, S, generator=g, device="cuda") * 2 - 1) / 0.075          # the G-CRD range |Z| <= 1/tau
    z[1::5] *= 8                                                                     # and beyond
    d = torch.arange(min(rows, S), device="cuda")
    z[3::7, :] = -13.0
    z[d[3::7], d[3::7]] = 13.0                                                       # a dominant positive: p_ii ~ 1
    return z


def _nce_ref(z: torch.Tensor, S: int, row_offset: int = 0):
    z = z.double()
    rows = z.shape[0]
    m = z.max(1, keepdim=True).values
    ls = torch.log(torch.exp(z - m).sum(1, keepdim=True))
    lse = m + ls
    p = torch.exp(z - lse)
    H = (p * (z - m).abs()).sum(1, keepdim=True)
    k = _ceil(S, 256)
    dl = U * (4 + H + k + 10) + 2 * U * ls.abs() + U * lse.abs()
    eye = torch.zeros_like(z)
    diag = torch.arange(rows, device="cuda")
    eye[diag, diag + row_offset] = 1.0
    w = 1.0 / S
    dz = (p - eye) * w
    dzb = w * (p * (U * (z - lse).abs() + dl + EXP) + 3 * U * (p - eye).abs() + TINY) + 2.0 ** -147
    zii = z[diag, diag + row_offset][:, None]
    part = (lse - zii)[:, 0]
    pb = (dl + U * (lse - zii).abs())[:, 0]
    return dz, dzb, part, pb, w * (p + eye)


@pytest.mark.parametrize("S", NCE_S)
def test_nce_rows_single_and_chunked(S):
    """Single call against fp64; then the chunked sequence (ragged last chunk, padded pitch with canary columns) must be
    bit-identical to it, partials and loss included."""
    g = _gen(S)
    z = _nce_inputs(S, S, g)
    Z = z.clone()
    part, loss = _canary(S + 8), _canary(4)
    lib.check(_L().b200gnn_nce_rows_f32(Z.data_ptr(), S, loss.data_ptr(), part.data_ptr(), _st()), "nce_rows")
    torch.cuda.synchronize()
    dz, dzb, pr, pb, mag = _nce_ref(z, S)
    lr = float(pr.mean())
    lb = float(pb.mean()) + 2 * U * abs(lr)
    r = max(_bound_ratio(Z, dz, dzb), _bound_ratio(part[:S], pr, pb),
            _bound_ratio(loss[:1], torch.tensor([lr], device="cuda", dtype=torch.float64),
                         torch.tensor([lb], device="cuda", dtype=torch.float64)))
    assert _is_canary(part[S:]) and _is_canary(loss[1:])
    if S >= 255:   # the random rows of the G-CRD range
        plain = torch.ones(S, dtype=torch.bool, device="cuda")
        plain[1::5] = False
        plain[3::7] = False
        _tight(dzb[plain], mag[plain])
    ldz = S + 5
    R = max(1, (S * 2) // 5)
    part2, loss2 = _canary(S + 8), _canary(4)
    Zc = _canary(R, ldz)
    for r0 in range(0, S, R):
        rr = min(R, S - r0)
        Zc[:rr, :S] = z[r0:r0 + rr]
        lib.check(_L().b200gnn_nce_rows_chunk_f32(Zc.data_ptr(), ldz, rr, S, r0, part2.data_ptr(), _st()), "nce_chunk")
        torch.cuda.synchronize()
        assert _bits_equal(Zc[:rr, :S], Z[r0:r0 + rr]), r0
        assert _is_canary(Zc[:, S:]), "pitch padding written"
    lib.check(_L().b200gnn_nce_finish_f32(part2.data_ptr(), S, loss2.data_ptr(), _st()), "nce_finish")
    torch.cuda.synchronize()
    assert _bits_equal(part2, part) and _bits_equal(loss2[:1], loss[:1]) and _is_canary(loss2[1:])
    _record("nce", r)


# ============================================================================================== 5. GSP pair pass
# gsp_pair_kernel on the fp32 Gram matrices and squared norms it is given (the test rounds fp64 Grams, so the GEMM is
# not part of the check).  Per (i, j):
#   cosine  sim = a exactly;  poly sim = a^2 (u);
#   l2/rbf  d2 = max(n_i + n_j - 2a, 0) (2a exact): delta_d2 <= u (n_i + n_j) + u d2 (0 on the forced diagonal).  Relative
#           to d2 this is u (n_i + n_j) / d2, the Gram form's conditioning on near-duplicate rows (u |x|^2 / d^2); the
#           difference form has none.  It is the kernel's design, and the bound below carries it.
#   l2      sim = sqrtf(d2): min(sqrt(delta_d2), delta_d2 / sqrt(d2)) + u sim; its derivative 0.5/sim: relative r/(1-r) + u
#           with r = delta_sim / sim; the sub-gradient is 0 where d2 is exactly 0 (duplicate rows);
#   rbf     sim = expf(-d2/2): sim (4u + delta_d2 / 2) + TINY.
# diff = sim_s - sim_t: both errors + u |diff|; dG = (w diff) dsim/dG with w = 2/S^2 rounded: 3u of the result plus the
# propagated terms; rowcoef sums S/256 + 10 terms; the loss (fp32 fma chains of diff^2, then fp64) likewise.
GSP_S = [1, 7, 257, 600]


def _gsp_ref(Gs, Gt, ns, nt, S, kernel):
    a, b = Gs.double(), Gt.double()
    w = 2.0 / (S * S)
    zero = torch.zeros_like(a)
    eye = torch.eye(S, dtype=torch.bool, device="cuda")

    def side(G, n):
        if kernel == 0:
            return G, zero, torch.ones_like(G), zero, zero, zero
        if kernel == 1:
            return G * G, U * G * G, 2 * G, zero, zero, zero
        n = n.double()
        nsum = n[:, None] + n[None, :]
        d2 = (nsum - 2 * G).clamp_min(0).masked_fill(eye, 0.0)
        dd2 = (U * nsum + U * d2).masked_fill(eye, 0.0)
        if kernel == 2:
            s = d2.sqrt()
            ds = torch.where(d2 > 0, torch.minimum(dd2.sqrt(), dd2 / s.clamp_min(1e-300)), dd2.sqrt()) + U * s
            inv = torch.where(s > 0, 0.5 / s.clamp_min(1e-300), zero)
            rr = ds / s.clamp_min(1e-300)
            dinv = torch.where(s > 0, inv * (rr / (1 - rr).clamp_min(0) + U), zero)
            dinv = torch.where(rr < 1, dinv, torch.full_like(dinv, math.inf)).masked_fill(d2 == 0, 0.0)
            return s, ds, -2 * inv, 2 * dinv, inv, dinv
        s = torch.exp(-0.5 * d2)
        ds = s * (EXP + 0.5 * dd2) + TINY
        return s, ds, s, ds, -0.5 * s, 0.5 * ds

    ss, dss, dg, ddg, dn, ddn = side(a, ns)
    st, dst_, _, _, _, _ = side(b, nt)
    diff = ss - st
    ddiff = dss + dst_ + U * diff.abs()
    gs = w * diff * dg
    gsb = w * (ddiff * dg.abs() + diff.abs() * ddg) + 3 * U * gs.abs() + 2.0 ** -147
    k = _ceil(S, 256)
    rc = (w * diff * dn).sum(1)
    rcb = (w * (ddiff * dn.abs() + diff.abs() * ddn)).sum(1) + (k + 13) * U * (w * diff * dn).abs().sum(1) + 2.0 ** -147
    loss = float((diff * diff).sum()) / (S * S)
    lb = float((2 * diff.abs() * ddiff + (k + 12) * U * diff * diff).sum()) / (S * S) + 2 * U * loss + 2.0 ** -147
    return gs, gsb, rc, rcb, loss, lb, w * (ss.abs() + st.abs()) * dg.abs()


def _gsp_features(S: int, F: int, g: torch.Generator, kernel: int, dup: bool):
    x = torch.randn(S, F, generator=g, device="cuda")
    if kernel == 3:
        x *= 0.15                                      # distances where exp(-d2/2) is not all 0
    if S >= 7:
        x[4] = x[3] * (1 + 2.0 ** -6 * torch.randn(F, generator=g, device="cuda"))   # near-duplicates
    if dup and S >= 7:                                 # exact duplicates: Gram, norms and d2 = 0 exact
        x[1] = torch.randint(-3, 4, (F,), generator=g, device="cuda").float()
        x[2] = x[1]
    if dup and S > 100:
        x[50:60] = torch.randint(-2, 3, (10, F), generator=g, device="cuda").float()
        x[60:70] = x[50:60]
    return x


@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
@pytest.mark.parametrize("S", GSP_S)
def test_gsp_pair_elementwise(S, kernel):
    g = _gen(10 * S + kernel)
    F = 48
    # the duplicates are in the student only, so that the sub-gradient at d2 = 0 meets a non-zero difference
    xs, xt = _gsp_features(S, F, g, kernel, True), _gsp_features(S, F, g, kernel, False)
    if kernel <= 1:
        xs = torch.nn.functional.normalize(xs.double(), dim=1)
        xt = torch.nn.functional.normalize(xt.double(), dim=1)
    xs64, xt64 = xs.double(), xt.double()
    Gs, Gt = (xs64 @ xs64.t()).float(), (xt64 @ xt64.t()).float()
    ns = (xs64 ** 2).sum(1).float() if kernel >= 2 else None
    nt = (xt64 ** 2).sum(1).float() if kernel >= 2 else None
    if kernel >= 2:   # the caller's Gram diagonal (GEMM) and norms (row_sqnorm) differ in the last bits: the diagonal
        Gs.diagonal().mul_(1 - 2.0 ** -20)       # distance must still be exactly 0
        Gt.diagonal().mul_(1 + 2.0 ** -20)
    dG = Gs.clone()
    rc = _canary(S + 8) if kernel >= 2 else None
    part, loss = _canary(S + 8), _canary(4)
    lib.check(_L().b200gnn_gsp_pair_f32(dG.data_ptr(), Gt.data_ptr(), _p(ns), _p(nt), S, kernel, _p(rc), loss.data_ptr(),
                                      part.data_ptr(), _st()), "gsp_pair")
    torch.cuda.synchronize()
    gs, gsb, rcr, rcb, lr, lb, mag = _gsp_ref(Gs, Gt, ns, nt, S, kernel)
    r = max(_bound_ratio(dG, gs, gsb), _bound_ratio(loss[:1], torch.tensor([lr], device="cuda", dtype=torch.float64),
                                                    torch.tensor([lb], device="cuda", dtype=torch.float64)))
    if kernel >= 2:
        r = max(r, _bound_ratio(rc[:S], rcr, rcb))
        assert _is_canary(rc[S:])
        assert bool((dG.diagonal() == 0).all()), "the diagonal distance is forced to 0"
        if S >= 7 and kernel == 2:
            assert float(dG[1, 2]) == 0.0 and float(dG[2, 1]) == 0.0, "duplicate rows: sub-gradient 0"
    assert _is_canary(part[S:]) and _is_canary(loss[1:])
    if S > 100:
        ok = torch.ones(S, S, dtype=torch.bool, device="cuda")
        ok[:5] = False
        ok[:, :5] = False
        ok[50:70] = False
        ok[:, 50:70] = False
        ok.fill_diagonal_(False)
        _tight(gsb[ok], mag[ok])
    _record("gsp", r)


# ============================================================================================ 6. LSP edge passes
# edge_sim_kernel, one warp per edge, m = ceil(F/32):
#   cosine  dot by fma chains: (m + 5) u sum |x y|; the norms (m + 5)/2 u + u each (sqrtf), clamped at COS_EPS
#           (continuous); the product and the division 2u: delta_c <= (m+5) u sum|xy| / (na nb) + |c| (m + 9) u;
#   poly    2 |c| delta_c + u c^2;
#   l2      d = a - b (u), d^2 by fma chains: (m + 7) u d2; sqrtf: ((m + 7)/2 + 1) u sim;
#   rbf     sim (4u + delta_d2 / 2) + TINY (rbf similarities underflow to exactly 0).
# lsp_segment_kernel, one warp per destination segment of length len (k = ceil(len/32)), PyG softmax with + 1e-16:
#   delta_lz <= u (5 + H + k + 5) + 2u |lz|, eps_p = u |s - m| + u |lp| + delta_lz + 4u;
#   kld g = (ps T - pt) / E: (ps (eps_ps + 3u) + pt (eps_pt + 3u)) / E + 2u |g|;
#   mse g = 2/E ps (d - q), d = ps - pt, q = sum d ps: the propagated errors of ps, d and q, + 3u |g|.
#   The loss adds each lane's terms over all its segments (c terms), a 5-level tree and 8 warps: (c + 13) u sum |term|.
# lsp_edge_coef_kernel: w = g' / (na nb), sa = g' c / na^2 (0 when the norm is clamped) with g' = g (cosine) or 2 c g
# (poly), from the same dot and norms: the propagated errors + 2-4u; l2 coef = g / sim (0 at sim = 0), rbf -g sim: u.
# lsp_diag_kernel: -(sum of the row's off-diagonal selfc) by a k-long chain and a 5-level tree: (k + 5) u sum |selfc|.
# edge_sim_bwd_kernel adds every edge's two row updates with atomics: in any order, a row updated cnt times is within
# cnt u of sum |terms| (initial value included), plus the propagated errors of w, sa, sb or coef (+2u per term).
def _lsp_graph(n: int, g: torch.Generator):
    """dst-sorted edges: empty segments (leading, trailing, runs), lengths 1, 31, 32, 33, a 3,000-edge hub, self-loops
    and duplicate edges, random small segments."""
    lens = torch.zeros(n, dtype=torch.long)
    design = {1: 1, 5: 31, 6: 32, 7: 33, 8: 3000, 9: 6, 10: 2, 11: 1, 13: 33, 14: 64, 15: 65}
    for i, v in design.items():
        lens[i] = v
    rnd = torch.randint(0, 5, (n - 20,), generator=torch.Generator().manual_seed(n))
    lens[20:n] = rnd
    lens[40:47] = 0                                         # a run of empty segments in the middle
    lens[n - 6:] = 0                                        # trailing empty segments
    dst = torch.repeat_interleave(torch.arange(n), lens)
    src = torch.randint(0, n, (int(lens.sum()),), generator=torch.Generator().manual_seed(n + 1))
    b9 = int(lens[:9].sum())
    src[b9:b9 + 6] = torch.tensor([9, 9, 1, 3, 3, 9])     # self-loops, an identical row (x[1] = x[9]), duplicate edges
    src[b9 + 6] = 10                                        # node 10: a self-loop
    rowptr = torch.zeros(n + 1, dtype=torch.long)
    rowptr[1:] = torch.cumsum(lens, 0)
    return src.int().cuda(), dst.int().cuda(), rowptr.int().cuda()


def _lsp_features(n: int, F: int, g: torch.Generator, kernel: int) -> torch.Tensor:
    x = torch.randn(n, F, generator=g, device="cuda") * _pow2(n, g, 2 if kernel == 3 else 10)[:, None]
    if kernel == 3:
        x *= 0.3
    x[3] = 0                                                # zero rows: COS_EPS
    x[100] = 0
    x[8] *= 2.0 ** -40 / float(x[8].abs().max())            # norm far below COS_EPS
    x[9] = x[1]                                             # identical rows: l2 = 0
    x[5] = x[100]
    return x


def _edge_sim_ref(x, src, dst, kernel):
    F = x.shape[1]
    m = _ceil(F, 32)
    a, b = x.double()[src.long()], x.double()[dst.long()]
    if kernel <= 1:
        dot = (a * b).sum(1)
        ra, rb = a.norm(dim=1), b.norm(dim=1)
        NA, NB = ra.clamp_min(COS_EPS), rb.clamp_min(COS_EPS)
        c = dot / (NA * NB)
        dc = (m + 5) * U * (a * b).abs().sum(1) / (NA * NB) + c.abs() * (m + 9) * U
        if kernel == 0:
            return c, dc
        return c * c, 2 * c.abs() * dc + U * c * c
    d2 = ((a - b) ** 2).sum(1)
    dd2 = (m + 7) * U * d2
    if kernel == 2:
        s = d2.sqrt()
        return s, ((m + 7) / 2 + 1) * U * s
    s = torch.exp(-0.5 * d2)
    return s, s * (EXP + 0.5 * dd2) + TINY


def _seg_ids(rowptr):
    lens = (rowptr[1:] - rowptr[:-1]).long()
    return torch.repeat_interleave(torch.arange(len(lens), device="cuda"), lens), lens


def _segsum(v, seg, n):
    return torch.zeros(n, dtype=v.dtype, device="cuda").index_add_(0, seg, v)


def _pyg_softmax(s, seg, n, lens):
    mx = torch.full((n,), -math.inf, dtype=torch.float64, device="cuda").scatter_reduce(0, seg, s, "amax")
    d = s - mx[seg]
    z = _segsum(torch.exp(d), seg, n) + 1e-16
    lz = torch.log(z)
    lp = d - lz[seg]
    p = torch.exp(lp)
    H = _segsum(p * d.abs(), seg, n)
    k = (lens + 31) // 32
    dlz = U * (5 + H + k + 5) + 2 * U * lz.abs()
    eps = U * d.abs() + U * lp.abs() + dlz[seg] + EXP
    return p, lp, eps, z, k


def _lsp_segment_ref(sim_s, sim_t, rowptr, E, criterion_, grid):
    seg, lens = _seg_ids(rowptr)
    n = len(lens)
    ps, lps, eps_s, _, k = _pyg_softmax(sim_s.double(), seg, n, lens)
    pt, lpt, eps_t, zt, _ = _pyg_softmax(sim_t.double(), seg, n, lens)
    warp = torch.arange(n, device="cuda") % (grid * 8)
    c = int(_segsum(k.double(), warp, grid * 8).max()) + 13
    if criterion_ == 0:
        T = ((zt - 1e-16) / zt)[seg]
        gr = (ps * T - pt) / E
        gb = (ps * (eps_s + 3 * U) + pt * (eps_t + 3 * U)) / E + 2 * U * gr.abs() + TINY / E
        dl = lpt - lps
        term = torch.where(pt > 0, pt * dl, torch.zeros_like(pt))
        tb = pt * (eps_t * dl.abs() + eps_t + eps_s + 2 * U * dl.abs()) + TINY
        mag = (ps + pt) / E
    else:
        d = ps - pt
        dd = ps * eps_s + pt * eps_t + U * d.abs()
        q = _segsum(d * ps, seg, n)
        dq = _segsum(dd * ps + d.abs() * ps * eps_s + 2 * U * (d * ps).abs(), seg, n) + (k + 5) * U * _segsum((d * ps).abs(), seg, n)
        dmq = d - q[seg]
        gr = 2.0 / E * ps * dmq
        gb = 2.0 / E * (ps * eps_s * dmq.abs() + ps * (dd + dq[seg] + U * dmq.abs())) + 3 * U * gr.abs() + TINY / E
        term = d * d
        tb = 2 * d.abs() * dd
        mag = 2.0 / E * ps * (d.abs() + _segsum((d * ps).abs(), seg, n)[seg])
    loss = float(term.sum()) / E
    lb = (float(tb.sum()) + c * U * float(term.abs().sum())) / E + 2 * U * abs(loss)
    return gr, gb, loss, lb, mag


def _coef_ref(x, src, dst, kernel, sim, gin):
    """fp64 (w, sa, sb) of every edge and their bounds, from the fp32 features, similarities and g the kernel reads."""
    F = x.shape[1]
    m = _ceil(F, 32)
    ge = gin.double()
    if kernel <= 1:
        a, b = x.double()[src.long()], x.double()[dst.long()]
        dot = (a * b).sum(1)
        ra, rb = a.norm(dim=1), b.norm(dim=1)
        NA, NB = ra.clamp_min(COS_EPS), rb.clamp_min(COS_EPS)
        c = dot / (NA * NB)
        dc = (m + 5) * U * (a * b).abs().sum(1) / (NA * NB) + c.abs() * (m + 9) * U
        rn = (0.5 * (m + 5) + 1) * U
        dge = torch.zeros_like(ge)
        if kernel == 1:
            ge = ge * 2 * c
            dge = 2 * gin.double().abs() * dc + U * ge.abs()
        w = ge / (NA * NB)
        dw = dge / (NA * NB) + w.abs() * (2 * rn + 2 * U)
        sa = torch.where(ra > COS_EPS, ge * c / (NA * NA), torch.zeros_like(ge))
        sb = torch.where(rb > COS_EPS, ge * c / (NB * NB), torch.zeros_like(ge))
        dsa = torch.where(ra > COS_EPS, (dge * c.abs() + ge.abs() * dc) / (NA * NA) + sa.abs() * (2 * rn + 3 * U), torch.zeros_like(ge))
        dsb = torch.where(rb > COS_EPS, (dge * c.abs() + ge.abs() * dc) / (NB * NB) + sb.abs() * (2 * rn + 3 * U), torch.zeros_like(ge))
        return w, dw, sa, dsa, sb, dsb
    s = sim.double()
    coef = torch.where(s > 0, ge / s.clamp_min(1e-300), torch.zeros_like(ge)) if kernel == 2 else -ge * s
    dcoef = U * coef.abs()
    return -coef, dcoef, -coef, dcoef, -coef, dcoef


LSP_N, LSP_F = 4000, 48


@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
def test_lsp_passes_elementwise(kernel):
    """edge_sim, lsp_segment (kld and mse), the values of the backward matrix and the atomic edge_sim_bwd on a designed
    dst-sorted edge list."""
    g = _gen(100 + kernel)
    src, dst, rowptr = _lsp_graph(LSP_N, g)
    E = src.numel()
    xs, xt = _lsp_features(LSP_N, LSP_F, g, kernel), _lsp_features(LSP_N, LSP_F, g, kernel)
    sims = []
    r_sim = 0.0
    for x in (xs, xt):
        sim = _canary(E + 8)
        lib.check(_L().b200gnn_edge_sim_f32(x.data_ptr(), LSP_F, src.data_ptr(), dst.data_ptr(), E, kernel, sim.data_ptr(),
                                          _st()), "edge_sim")
        torch.cuda.synchronize()
        ref, b = _edge_sim_ref(x, src, dst, kernel)
        r_sim = max(r_sim, _bound_ratio(sim[:E], ref, b + 2.0 ** -149))
        assert _is_canary(sim[E:])
        sims.append(sim[:E].clone())
    if kernel == 2:
        assert bool((sims[0][rowptr[9]:rowptr[9] + 6][torch.tensor([0, 1, 2, 5], device="cuda")] == 0).all())   # identical rows
    if kernel == 3:
        assert bool((sims[0] == 0).any()), "some rbf similarities underflow to exactly 0"
    _record("edge_sim", r_sim)
    n_seg = LSP_N
    grid = int(_L().b200gnn_lsp_partials(n_seg))
    r_seg = 0.0
    plan = criterion.LspPlan(torch.stack([src.long(), dst.long()]))
    G, pos_dst, pos_src, diag_pos, _ = plan.backward_matrix(LSP_N)
    nnz = G.val.numel()
    for crit in (0, 1):
        gbuf, part, loss = _canary(E + 8), _canary(grid + 8), _canary(4)
        lib.check(_L().b200gnn_lsp_segment_f32(sims[0].data_ptr(), sims[1].data_ptr(), rowptr.data_ptr(), n_seg, E, crit,
                                             gbuf.data_ptr(), loss.data_ptr(), part.data_ptr(), _st()), "lsp_segment")
        torch.cuda.synchronize()
        gr, gb, lr, lb, mag = _lsp_segment_ref(sims[0], sims[1], rowptr, E, crit, grid)
        r_seg = max(r_seg, _bound_ratio(gbuf[:E], gr, gb),
                    _bound_ratio(loss[:1], torch.tensor([lr], device="cuda", dtype=torch.float64),
                                 torch.tensor([lb], device="cuda", dtype=torch.float64)))
        assert _is_canary(gbuf[E:]) and _is_canary(part[grid:]) and _is_canary(loss[1:])
        if kernel == 0 and crit == 0:
            _tight(gb[mag > 1e-3 * float(mag.max())], mag[mag > 1e-3 * float(mag.max())])
        gvals = gbuf[:E].clone()
        # values of the backward matrix: w_e at (dst, src) and (src, dst), the diagonal -sum of the row's selfc
        val, selfc = _canary(nnz + 8), _canary(nnz + 8)
        lib.check(_L().b200gnn_lsp_bwd_values_f32(xs.data_ptr(), LSP_F, src.data_ptr(), dst.data_ptr(), E, kernel,
                                                sims[0].data_ptr(), gvals.data_ptr(), pos_dst.data_ptr(), pos_src.data_ptr(),
                                                G.rowptr.data_ptr(), diag_pos.data_ptr(), LSP_N, val.data_ptr(),
                                                selfc.data_ptr(), _st()), "lsp_bwd_values")
        torch.cuda.synchronize()
        w, dw, sa, dsa, sb, dsb = _coef_ref(xs, src, dst, kernel, sims[0], gvals)
        pd, ps_ = pos_dst.long(), pos_src.long()
        assert bool((G.col.long()[pd] == src.long()).all()) and bool((G.col.long()[ps_] == dst.long()).all())
        vr = torch.zeros(nnz, dtype=torch.float64, device="cuda")
        vb = torch.zeros_like(vr)
        vr[pd], vb[pd] = w, dw
        vr[ps_], vb[ps_] = w, dw
        sc = torch.zeros_like(vr)
        scb = torch.zeros_like(vr)
        sc[pd], scb[pd] = sb, dsb
        sc[ps_], scb[ps_] = sa, dsa
        rseg, rlen = _seg_ids(G.rowptr)
        k = (rlen + 31) // 32
        dg = diag_pos.long()
        vr[dg] = -_segsum(sc, rseg, LSP_N)
        vb[dg] = _segsum(scb, rseg, LSP_N) + (k + 5) * U * _segsum(sc.abs(), rseg, LSP_N)
        r_val = _bound_ratio(val[:nnz], vr, vb + 2.0 ** -149)
        assert _is_canary(val[nnz:]) and _is_canary(selfc[dg]), "selfc written on the diagonal"
        r_val = max(r_val, _bound_ratio(selfc[pd], sb, dsb + 2.0 ** -149), _bound_ratio(selfc[ps_], sa, dsa + 2.0 ** -149))
        lonely = rlen == 1                                              # nodes without edges: a diagonal of exactly 0
        assert bool(lonely.any()) and bool((val[dg[lonely]] == 0).all())
        _record("lsp_values", r_val)
        # the atomic backward, in any order of its additions
        d0 = torch.randn(LSP_N, LSP_F, generator=g, device="cuda")
        dfeat = _canary(LSP_N + 2, LSP_F)
        dfeat[:LSP_N] = d0
        lib.check(_L().b200gnn_edge_sim_bwd_f32(xs.data_ptr(), LSP_F, src.data_ptr(), dst.data_ptr(), E, kernel,
                                              sims[0].data_ptr(), gvals.data_ptr(), dfeat.data_ptr(), _st()), "edge_sim_bwd")
        torch.cuda.synchronize()
        a, b = xs.double()[src.long()], xs.double()[dst.long()]
        if kernel <= 1:
            ca, cb = w[:, None] * b - sa[:, None] * a, w[:, None] * a - sb[:, None] * b
            cab = dw[:, None] * b.abs() + dsa[:, None] * a.abs() + 2 * U * ((w[:, None] * b).abs() + (sa[:, None] * a).abs())
            cbb = dw[:, None] * a.abs() + dsb[:, None] * b.abs() + 2 * U * ((w[:, None] * a).abs() + (sb[:, None] * b).abs())
        else:
            coef = -w
            ca = coef[:, None] * (a - b)
            cb = -ca
            cab = dw[:, None] * (a - b).abs() + 2 * U * ca.abs()
            cbb = cab
        z64 = torch.zeros(LSP_N, LSP_F, dtype=torch.float64, device="cuda")
        ref = d0.double() + z64.clone().index_add_(0, src.long(), ca).index_add_(0, dst.long(), cb)
        absum = d0.double().abs() + z64.clone().index_add_(0, src.long(), ca.abs()).index_add_(0, dst.long(), cb.abs())
        prop = z64.clone().index_add_(0, src.long(), cab).index_add_(0, dst.long(), cbb)
        cnt = (torch.bincount(src.long(), minlength=LSP_N) + torch.bincount(dst.long(), minlength=LSP_N)).double()[:, None]
        bound = prop + cnt * U * absum + 2.0 ** -149
        _record("edge_sim_bwd", _bound_ratio(dfeat[:LSP_N], ref, bound))
        assert _is_canary(dfeat[LSP_N:])
    _record("lsp_segment", r_seg)


# ============================================================================================ 7. transpose (exact)
@pytest.mark.parametrize("rows,cols", [(1, 1), (31, 33), (33, 31), (1000, 3), (2_097_153, 3)])
def test_transpose_exact(rows, cols):
    """The last shape has more row tiles (65,537) than gridDim.y can hold (65,535)."""
    g = _gen(rows + cols)
    x = torch.randn(rows, cols, generator=g, device="cuda")
    out = _canary(rows * cols + 8)
    lib.check(_L().b200gnn_transpose_f32(x.data_ptr(), rows, cols, out.data_ptr(), _st()), "transpose")
    torch.cuda.synchronize()
    assert torch.equal(out[:rows * cols].view(cols, rows), x.t())
    assert _is_canary(out[rows * cols:])


# ========================================================================= 8. the callers' shapes, through criterion.py
def test_caller_arxiv_kd():
    """ARXIV logit KD as the engines call it: 169,343 x 40 logits, 90,941 training rows, dlogits zero elsewhere."""
    g = _gen(40)
    n, C, n_train = 169_343, 40, 90_941
    z, t, y = _kd_inputs(C, n, g, extreme=False)
    idx = torch.randperm(n, generator=g, device="cuda")[:n_train].sort().values
    out, dl = ops.kd_loss_fwd_bwd(z, y, idx, t, 0.9, 4.0)
    torch.cuda.synchronize()
    ref = _kd_ref(z[idx], t[idx], y[idx], C, 0.9, 4.0, 0, n_train, int(_L().b200gnn_kd_partials(n_train)))
    r = max(_bound_ratio(dl[idx], ref["g"], ref["gb"]), _bound_ratio(out, ref["loss"], ref["lb"]))
    _tight(ref["gb"], ref["mag"])
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    mask[idx] = False
    assert bool((dl[mask] == 0).all())
    _record("caller_arxiv_kd", r)


@pytest.mark.parametrize("teacher", [False, True])
def test_caller_mag_349_in_352(teacher):
    """The MAG student's loss as the R-GCN calls it: 349 classes read from 352-wide logits (and teacher) rows and written
    into 352-wide dlogits rows; the 3 pad columns are never written."""
    g = _gen(349 + teacher)
    n, C, W, n_train = 20_000, 349, 352, 6_000
    z, t, y = _kd_inputs(C, n, g, extreme=False)
    zbuf, tbuf, dbuf = _canary(n, W), _canary(n, W), _canary(n, W)
    zbuf[:, :C], tbuf[:, :C] = z, t
    dbuf[:, :C] = 0
    idx = torch.randperm(n, generator=g, device="cuda")[:n_train]
    grid = int(_L().b200gnn_kd_partials(n_train))
    part, out = torch.empty(2 * grid, device="cuda"), torch.empty(3, device="cuda")
    lib.check(_L().b200gnn_kd_loss_fwd_bwd_f32(zbuf.data_ptr(), W, idx.data_ptr(), n_train, y.data_ptr(),
                                             tbuf.data_ptr() if teacher else None, W if teacher else 0, C, 0.9, 4.0, 0,
                                             dbuf.data_ptr(), W, out.data_ptr(), part.data_ptr(), _st()), "kd")
    torch.cuda.synchronize()
    ref = _kd_ref(z[idx], t[idx] if teacher else None, y[idx], C, 0.9, 4.0, 0, n_train, grid)
    r = max(_bound_ratio(dbuf[idx, :C], ref["g"], ref["gb"]), _bound_ratio(out, ref["loss"], ref["lb"]))
    _tight(ref["gb"], ref["mag"])
    assert _is_canary(dbuf[:, C:])
    _record("caller_mag", r)


def test_caller_ppi_bce():
    """PPI: 121 labels per node, the gradient through autograd (upstream gradient 1: the kernel's d_z)."""
    g = _gen(121)
    n, C = 9_716, 121
    z = (torch.randn(n, C, generator=g, device="cuda") * 4).requires_grad_(True)
    y = (torch.rand(n, C, generator=g, device="cuda") < 0.3).float()
    loss = criterion.bce_with_logits(z, y)
    loss.backward()
    torch.cuda.synchronize()
    grid, k = _ew_grid_k(n * C)
    dzr, dzb, lr, lb, mag = _bce_ref(z.detach().view(-1), y.view(-1), 0, 1.0, n * C, k)
    r = max(_bound_ratio(z.grad.view(-1), dzr, dzb),
            _bound_ratio(loss.detach().view(1), torch.tensor([lr], device="cuda", dtype=torch.float64),
                         torch.tensor([lb], device="cuda", dtype=torch.float64)))
    _tight(dzb, mag)
    _record("caller_ppi_bce", r)


# G-CRD end to end (criterion._NCE: normalisation, the 3xTF32 logits GEMM, the row pass, two gradient GEMMs, the
# normalisation backward) against fp64 autograd.  The elementwise magnitude is the absolute-value chain of the
# backward, M = scale/||f_i|| ((|dZ| |x_o|)_ik + |u_ik| sum_l |u_il| (|dZ| |x_o|)_il) with |dZ| = (P + I)/S; the bound is
# GCRD_REL · M.  GCRD_REL quotes a measurement: on an H100 80GB HBM3 at 400 W the worst element used 1.44e-6 of M (student
# and teacher side, S = 8,192, F = 256).  The 3xTF32 GEMMs' worst-case bound composed through the softmax would allow
# about 2e-4; 4e-6 keeps a margin over the measurement and stays below 1e-5.
GCRD_REL = 4e-6


def test_caller_gcrd_8192x256():
    S, F, tau = 8_192, 256, 0.075
    g = _gen(8192)
    fs = torch.randn(S, F, generator=g, device="cuda").requires_grad_(True)
    ft = torch.randn(S, F, generator=g, device="cuda").requires_grad_(True)
    loss = criterion._NCE.apply(fs, ft, tau)
    loss.backward()
    torch.cuda.synchronize()
    fs64 = fs.detach().double().requires_grad_(True)
    ft64 = ft.detach().double().requires_grad_(True)
    xs, xt = torch.nn.functional.normalize(fs64, dim=1), torch.nn.functional.normalize(ft64, dim=1)
    z = xs @ xt.t() / tau
    ref = -torch.log_softmax(z, 1).diagonal().mean()
    ref.backward()
    with torch.no_grad():
        P = torch.softmax(z, 1)
        A = (P + torch.eye(S, dtype=torch.float64, device="cuda")) / S
        worst = 0.0
        for f, x, other, grad, ref_grad, scale, AA in ((fs64, xs, xt, fs.grad, fs64.grad, 1 / tau, A),
                                                       (ft64, xt, xs, ft.grad, ft64.grad, 1 / tau, A.t())):
            v = AA @ other.abs()
            M = scale / f.norm(dim=1, keepdim=True) * (v + x.abs() * (x.abs() * v).sum(1, keepdim=True))
            worst = max(worst, float(((grad.double() - ref_grad).abs() / M).max()))
        lr = float(ref)
        # the loss: the logits' GEMM error through the log-sum-exp, measured at 3.1e-8 relative (same H100); 1e-6 holds it
        lratio = abs(float(loss) - lr) / (1e-6 * abs(lr))
    print(f"\nG-CRD worst |err|/M = {worst:.3g}, loss ratio {lratio:.3g}")
    _record("caller_gcrd", max(worst / GCRD_REL, lratio))
