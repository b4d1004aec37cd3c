"""Bit-exact contract of the row-segmented sparse kernels (spmm.cu, gat.cu) over every dispatch path and plan geometry.

Exact arithmetic.  If every term of a sum is a multiple of 2^-q, every partial sum, in any order and any summation tree, is
a multiple of 2^-q no larger than sum |terms|; so it is exact in fp32 when 2^q * sum |terms| < 2^24.  The data here is built
for that: small-integer features, edge values in 2^-2 Z ∩ (0, 2], attention coefficients in 2^-3 Z ∩ [0, 1], leaky-ReLU slope
1/4, attn_scale in {0, 2}.  Every test checks the claim in fp64 for every output and every intermediate sum (`_assert_exact`),
so the fp64 scatter sum of the same values IS the result, and each kernel must equal it bit for bit (`torch.equal`) whatever
order it sums in.  A row that is dropped, duplicated, written to the wrong place or loses one edge fails whatever its
magnitude — which the global max-norm metric of test_spmm_gpu.py / test_gat_gpu.py cannot promise.  The epilogue is
reproduced in fp32 in the kernels' order: S / max(deg, 1) rounded, then + bias rounded.  The division is IEEE (the library is
built without fast-math), and rounding S64 / d to fp64 and then to fp32 is correctly rounded (53 >= 2·24 + 2), so
(S64 / d).float() is exact too.

The graphs are designed, not only random: empty-row runs of 1 / 31 / 32 / 33 / 100 (leading and trailing), the degrees at the
kernels' internal boundaries, hub_threshold ± 1 and k·seg_len ± 1 of the plan in use, a 20,000-edge hub, hubs as first, last
and adjacent rows, duplicate columns and self-loops, and n_src != n_rows with NaN rows past n_src.  Each graph runs under five
plans (`PLANS`).  The kernels are called through the C ABI with poisoned views: operands inside NaN buffers with a wider pitch,
outputs NaN-filled inside buffers of NaN canaries that must survive bit for bit, NaN-filled workspaces and partial buffers.

Non-dyadic data gets an elementwise bound instead: the SpMM on scaled random data and the edge softmax, each derived below."""
import functools
import zlib

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib
from efficient_gnns_b200.sparse import CsrGraph

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

U = 2.0 ** -24                                        # unit roundoff of fp32 round to nearest
CANARY = 0x7FC0DEAD                                   # a quiet NaN with a payload: outside an output it must survive bit for bit
NAN_BITS = 0x7FC00000                                 # the NaN an output is filled with before a call (distinct from CANARY)
DEV = "cuda"
SUM, MEAN = lib.REDUCE_SUM, lib.REDUCE_MEAN
ERR_UNSUPPORTED = -2                                  # B200GNN_ERR_UNSUPPORTED (include/b200gnn.h)

# (hub_threshold, seg_len, chunk_nnz, row_cost) of CsrGraph.build_plan
PLANS = [
    (256, 256, 128, 4),          # the defaults (sparse.py)
    (0, 1, 1, 1),                # every non-empty row is a hub, 1-edge segments, one-row chunks
    (31, 7, 5, 1),
    (255, 257, 33, 2),
    (2 ** 30, 256, 4096, 64),    # no hubs; huge chunks full of empty rows
]
PLAN_IDS = ["default", "all-hubs", "31-7-5-1", "255-257-33-2", "no-hubs"]
GRAPH_KINDS = ("edges", "empties")


# ----------------------------------------------------------------------------------------------------- exactness helpers
def _gamma(n):
    """gamma(n) = n·u / (1 - n·u): any summation tree of n terms (products fused or exact) errs by at most gamma(n) of the
    sum of their magnitudes (Higham, Accuracy and Stability of Numerical Algorithms, §3.1)."""
    n = torch.as_tensor(n, dtype=torch.float64)
    return n * U / (1 - n * U)


def _assert_on_grid(x: torch.Tensor, q: int, what: str):
    s = x.double() * 2.0 ** q
    assert bool((s == s.round()).all()), f"{what}: not a multiple of 2^-{q}"


def _assert_exact(abs_sum: torch.Tensor, q: int, what: str):
    """Every sum whose terms are multiples of 2^-q and whose magnitudes add up to abs_sum is exact in fp32."""
    worst = float(abs_sum.max()) if abs_sum.numel() else 0.0
    assert worst * 2.0 ** q < 2.0 ** 24, f"{what}: 2^{q} · sum|terms| = {worst * 2.0 ** q:.3g} >= 2^24, not exact in fp32"


def _scatter(index: torch.Tensor, vals: torch.Tensor, n: int) -> torch.Tensor:
    out = torch.zeros((n,) + tuple(vals.shape[1:]), dtype=vals.dtype, device=vals.device)
    return out.index_add_(0, index, vals)


# ------------------------------------------------------------------------------------------------------ designed graphs
EMPTY_RUNS = (1, 31, 32, 33, 100)
# 1-9, 15-17, 31-33, 63-65: the G = 2/4/8 barrier groups, ring depths 8/16, 32-edge windows; 512/513: GAT_CTA_DEG
BOUNDARY_DEGS = list(range(1, 10)) + [15, 16, 17, 31, 32, 33, 63, 64, 65, 512, 513]
BIG_HUB = 20_000                                      # the ARXIV-scale hub


def _plan_degrees(plan) -> list:
    thr, seg = plan[0], plan[1]
    d = [thr - 1, thr, thr + 1] if thr < 50_000 else []
    d += [k * seg + o for k in (1, 2, 3) for o in (-1, 0, 1)]
    return [x for x in d if 0 <= x <= 5000]


def _degrees(plan, kind: str, rng) -> np.ndarray:
    body = []
    for i, d in enumerate(BOUNDARY_DEGS + _plan_degrees(plan)):
        body += rng.integers(0, 24, size=6).tolist() + [d]
        if i % 3 == 0:
            body += [0] * EMPTY_RUNS[(i // 3) % len(EMPTY_RUNS)]
    filler = rng.integers(0, 30, size=1500)
    filler[rng.random(1500) < 0.15] = 0
    body += filler.tolist()
    if kind == "edges":                 # hubs as the first and the last row, and two adjacent hubs in the middle
        degs = [3000] + body[: len(body) // 2] + [BIG_HUB, 1000] + body[len(body) // 2:] + [2500]
    else:                               # leading and trailing empty runs, a 5000-edge hub next to a 700-edge row
        degs = [0] * 33 + body[: len(body) // 3] + [700, 5000] + body[len(body) // 3:] + [0] * 100
    return np.asarray(degs, dtype=np.int64)


def _seed(*key) -> int:
    return zlib.crc32(repr(key).encode())


@functools.lru_cache(maxsize=None)
def designed(plan, kind: str):
    """(rowptr, col, n_rows, n_src) as int64 numpy.  Columns are uniform over the sources; every row of degree >= 2 holds a
    duplicated column (counted twice, as the reference's scatter counts it), every row of degree >= 3 with a matching source
    a self-loop, and the largest row reaches the last source.  "edges" has more sources than rows (so that the 20,000-edge
    hub reaches about as many distinct sources), "empties" fewer."""
    rng = np.random.default_rng(_seed(plan, kind))
    degs = _degrees(plan, kind, rng)
    n_rows = degs.size
    n_src = 24_000 if kind == "edges" else n_rows - 301
    rowptr = np.concatenate([[0], np.cumsum(degs)])
    col = rng.integers(0, n_src, size=int(rowptr[-1]))
    for i in np.flatnonzero(degs >= 2):
        b = rowptr[i]
        col[b + 1] = col[b]
        if degs[i] >= 3 and i < n_src:
            col[b + 2] = i
    col[rowptr[int(np.argmax(degs)) + 1] - 1] = n_src - 1
    return rowptr, col, n_rows, n_src


@functools.lru_cache(maxsize=None)
def device_graph(plan, kind: str) -> CsrGraph:
    rowptr, col, n_rows, n_src = designed(plan, kind)
    g = CsrGraph(torch.from_numpy(rowptr).to(DEV, torch.int32), torch.from_numpy(col).to(DEV, torch.int32), None,
                 n_rows, n_src)
    return g.build_plan(*plan)


def _row_index(rowptr: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.repeat(np.arange(rowptr.size - 1), np.diff(rowptr))).to(DEV)


def _deg(rowptr: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.diff(rowptr)).to(DEV)


def _gen(*key) -> torch.Generator:
    return torch.Generator(device=DEV).manual_seed(_seed(*key))


def _dyadic(shape, lo: int, hi: int, q: int, g) -> torch.Tensor:
    """Uniform multiples of 2^-q in [lo·2^-q, hi·2^-q]."""
    return torch.randint(lo, hi + 1, shape, generator=g, device=DEV).float() * 2.0 ** -q


# ------------------------------------------------------------------------------------------------------ poisoned buffers
class Boxed:
    """A [rows, cols] view at row r0 of a flat buffer with pitch ld, starting c0 floats into it; the rest of the buffer
    holds `fill` bits (CANARY by default)."""

    def __init__(self, rows: int, cols: int, ld: int, c0: int = 0, r0: int = 0, extra_rows: int = 3, fill: int = CANARY):
        total = c0 + (r0 + rows + extra_rows) * ld
        self.flat = torch.full((total,), fill, dtype=torch.int32, device=DEV).view(torch.float32)
        self.view = self.flat[c0:].view(-1, ld)[r0:r0 + rows, :cols]
        self.mask = torch.zeros(total, dtype=torch.bool, device=DEV)
        self.mask[c0:].view(-1, ld)[r0:r0 + rows, :cols] = True
        self.fill = fill

    def reset(self, inside: torch.Tensor | None = None):
        """Canaries everywhere, then `inside` (or NaN) in the view."""
        self.flat.view(torch.int32).fill_(self.fill)
        if inside is None:
            self.view.view(torch.int32).fill_(NAN_BITS)
        else:
            self.view.copy_(inside)

    def outside_intact(self) -> bool:
        return bool((self.flat.view(torch.int32)[~self.mask] == self.fill).all())


def _nan_flat(n: int) -> torch.Tensor:
    return torch.full((max(n, 1),), NAN_BITS, dtype=torch.int32, device=DEV).view(torch.float32)


def _slot_of_row(G: CsrGraph, n_rows: int) -> torch.Tensor:
    """Fused statistics (SpMM and GAT epilogues): slot s holds the rows of chunks 8s .. 8s+7 minus the hub rows; slot
    main_grid + h hub row h."""
    rows = torch.arange(n_rows, device=DEV, dtype=torch.int32)
    chunk = torch.searchsorted(G.chunk_rowptr, rows, right=True) - 1
    slot = chunk // 8
    if G.n_hub:
        main_grid = (G.n_chunks + 7) // 8
        slot[G.hub_rows[:G.n_hub].long()] = main_grid + torch.arange(G.n_hub, device=DEV)
    return slot.long()


# ================================================================================================================ plans
@pytest.mark.parametrize("plan", PLANS, ids=PLAN_IDS)
@pytest.mark.parametrize("kind", GRAPH_KINDS)
def test_plan_matches_numpy(plan, kind):
    """chunk_rowptr: monotone from 0 to n_rows, chunk c starting at the first row r with rowptr[r] + r·row_cost >= c·chunk_nnz;
    hub_rows / hub_segptr: the rows of degree > hub_threshold in order, ceil(deg / seg_len) segments each."""
    thr, seg, cnnz, cost = plan
    rowptr, _, n_rows, _ = designed(plan, kind)
    G = device_graph(plan, kind)
    deg = np.diff(rowptr)
    total = int(rowptr[-1]) + n_rows * cost
    assert G.n_chunks == -(-total // cnnz)
    cr = G.chunk_rowptr.cpu().numpy().astype(np.int64)
    assert cr[0] == 0 and cr[-1] == n_rows and bool((np.diff(cr) >= 0).all())
    key = rowptr + np.arange(n_rows + 1) * cost
    expect = np.searchsorted(key, np.arange(G.n_chunks) * cnnz, side="left")
    assert np.array_equal(cr[:-1], expect)
    hubs = np.flatnonzero(deg > thr)
    segs = -(-deg[hubs] // seg)
    assert G.n_hub == hubs.size and G.n_seg == int(segs.sum())
    assert np.array_equal(G.hub_rows[:G.n_hub].cpu().numpy(), hubs)
    assert np.array_equal(G.hub_segptr.cpu().numpy(), np.concatenate([[0], np.cumsum(segs)]))
    if kind == "edges" and thr < 50_000:
        assert hubs[0] == 0 and hubs[-1] == n_rows - 1     # hubs as the first and the last row


# ================================================================================================= SpMM: exact, every path
# (id, K, X pitch pad, X offset in floats, Y pitch pad, Y offset, fused statistics).  The dispatch is in
# b200gnn_spmm_csr_f32 (spmm.cu): W (the vector width) from K, the pitches and the base alignment; then the bulk-copy block
# (`if (W == 4 && K % 128 == 0 && K <= 4096)`, bulk_auto_slab picks 256-float slabs when K % 256 == 0, else 128); then
# `narrow_ok` (W == 4, nvec <= 16, no statistics); else dispatch_ch<float4 / float2 / float> with CH = 1 / 2 / 4 for
# nvec <= 32 / 64 / more, one slab when nvec <= 32·CH (statistics fused) and otherwise several slabs with the separate
# col_stats pass.  Hub rows end in spmm_hub_finalize_kernel: its float4 path when K % 4 == 0, K <= 1024 and Y, ldy and the
# workspace are 16-byte aligned, its scalar path otherwise.
SPMM_PATHS = [
    # bulk-copy ring, 256-float slabs (launch_spmm_bulk<2, 4>); K = 2048: scalar hub finalize (K > 1024)
    ("bulk256-K256", 256, 4, 0, 8, 0, True),
    ("bulk256-K512", 512, 4, 0, 4, 0, True),
    ("bulk256-K2048", 2048, 4, 0, 4, 0, True),
    # bulk-copy ring, 128-float slabs (launch_spmm_bulk<1, 4>)
    ("bulk128-K128", 128, 4, 0, 4, 0, True),
    ("bulk128-K384", 384, 8, 0, 4, 0, True),
    # narrow multi-row kernel (spmm_rows_narrow_kernel<.., 4>); with statistics these take dispatch_ch<float4> CH = 1
    ("narrow-K4", 4, 4, 0, 4, 0, True),
    ("narrow-K16", 16, 4, 0, 4, 0, True),
    ("narrow-K40", 40, 4, 0, 8, 0, True),
    ("narrow-K64", 64, 4, 0, 4, 0, True),
    # register float4, one slab: CH = 1 (K = 100), 2 (K = 200), 4 (K = 500)
    ("reg4-K100", 100, 4, 0, 4, 0, True),
    ("reg4-K200", 200, 4, 0, 4, 0, True),
    ("reg4-K500", 500, 4, 0, 4, 0, True),
    # register float4, several slabs + col_stats; K = 4224 is past the bulk kernels' 4096 and takes the scalar finalize
    ("reg4multi-K516", 516, 4, 0, 4, 0, False),
    ("reg4multi-K1000", 1000, 4, 0, 4, 0, False),
    ("reg4multi-K4224", 4224, 4, 0, 4, 0, False),
    # register float2: K % 4 == 2 (K = 6: CH 1, scalar finalize; K = 130: CH 4), or ldx / ldy = 2 (mod 4)
    ("reg2-K6", 6, 2, 0, 2, 0, True),
    ("reg2-K130", 130, 2, 0, 6, 0, True),
    ("reg2-ldx-K128", 128, 2, 0, 4, 0, True),
    ("reg2-ldy-K256", 256, 4, 0, 2, 0, True),
    # register float: K odd (K = 1025: several slabs), or a base misaligned by 4 bytes (a contiguous view one float into
    # its buffer: K = 128 would take the bulk kernel if it were aligned)
    ("reg1-K7", 7, 1, 0, 3, 0, True),
    ("reg1-K33", 33, 3, 0, 3, 0, True),
    ("reg1-K1025", 1025, 3, 0, 3, 0, False),
    ("reg1-xmis-K128", 128, 0, 1, 4, 0, True),
    ("reg1-ymis-K128", 128, 4, 0, 0, 1, True),
]


def _spmm_c(G: CsrGraph, val, xv, yv, K, reduce, bias, part, ws) -> int:
    return lib.load().b200gnn_spmm_csr_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), None if val is None else val.data_ptr(), xv.data_ptr(), xv.stride(0),
        yv.data_ptr(), yv.stride(0), G.n_rows, G.n_cols, K, reduce, None if bias is None else bias.data_ptr(),
        None if part is None else part.data_ptr(), G.chunk_rowptr.data_ptr(), G.n_chunks, G.hub_threshold, G.seg_len,
        G.hub_rows.data_ptr() if G.n_hub else None, G.hub_segptr.data_ptr() if G.n_hub else None, G.n_hub, G.n_seg,
        None if ws is None else ws.data_ptr(), lib.stream_ptr())


class SpmmCase:
    """Dyadic operands and the exact references of one (plan, graph, K): X in {-1, 0, 1} (+-1 with probability 1/9 each, so
    that the statistics' sums of squares stay exact on the hubs), values in 2^-2 Z ∩ (0, 2], bias in 2^-2 Z ∩ [-2, 2]."""

    def __init__(self, plan, kind, K, x_pad, x_c0, y_pad, y_c0):
        rowptr, col, n_rows, n_src = designed(plan, kind)
        self.G, self.K, self.n_rows = device_graph(plan, kind), K, n_rows
        g = _gen(plan, kind, K)
        nnz = int(rowptr[-1])
        self.val = _dyadic((nnz,), 1, 8, 2, g)
        x = torch.randint(-4, 5, (n_src, K), generator=g, device=DEV).div(4, rounding_mode="trunc").float()
        self.bias = _dyadic((K,), -8, 8, 2, g)
        self.X = Boxed(n_src, K, K + x_pad, c0=x_c0, extra_rows=5)    # NaN rows past n_src, NaN columns past K
        self.X.reset(x)
        self.Y = Boxed(n_rows, K, K + y_pad, c0=y_c0, r0=3)
        self.deg = _deg(rowptr)
        rows, cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
        x64 = x.double()
        self.ref, self.refb = {}, {}
        for reduce, val in ((SUM, self.val), (MEAN, None)):
            w = val.double()[:, None] if val is not None else 1.0
            terms = x64[cols] * w
            S = _scatter(rows, terms, n_rows)
            _assert_exact(_scatter(rows, terms.abs(), n_rows), 2, f"S (K={K})")
            del terms
            y = S.float() if reduce == SUM else (S / self.deg.clamp(min=1)[:, None].double()).float()
            self.ref[reduce] = y
            self.refb[reduce] = y + self.bias             # one fp32 rounding, as the kernels' epilogue
        self.ws = _nan_flat(self.G.n_seg * K)
        self.slots = int(lib.load().b200gnn_spmm_stat_slots(self.G.n_chunks, self.G.n_hub))
        self.part = _nan_flat(self.slots * 2 * K).view(self.slots, 2, K)

    def run(self, reduce, use_bias: bool, stats: bool) -> torch.Tensor:
        self.Y.reset()
        self.ws.view(torch.int32).fill_(NAN_BITS)
        self.part.view(torch.int32).fill_(NAN_BITS)
        val = self.val if reduce == SUM else None
        lib.check(_spmm_c(self.G, val, self.X.view, self.Y.view, self.K, reduce, self.bias if use_bias else None,
                          self.part if stats else None, self.ws), "spmm_csr_f32")
        return self.Y.view

    def slot_of_row(self) -> torch.Tensor:
        return _slot_of_row(self.G, self.n_rows)

    def check(self, reduce, use_bias, stats, fused, what):
        y = self.run(reduce, use_bias, stats)
        ref = (self.refb if use_bias else self.ref)[reduce]
        torch.cuda.synchronize()
        bad = (y != ref).any(1)
        assert not bool(bad.any()), f"{what}: rows {torch.nonzero(bad).flatten()[:8].tolist()} differ from the exact sum"
        assert self.Y.outside_intact(), f"{what}: a store outside Y"
        if not stats:
            return
        part = self.part.double()
        assert bool(torch.isfinite(part).all()), f"{what}: a statistics slot left unwritten"
        y64 = ref.double()
        if reduce == SUM:              # dyadic y (2^-2 Z): each slot's sum y and sum y^2 (2^-4 Z) are exact, so is their fp64 sum
            if fused:
                slot = self.slot_of_row()
            else:                      # col_stats_kernel: slot s holds rows [s·per, (s+1)·per), per = ceil(n_rows / slots)
                slot = torch.arange(self.n_rows, device=DEV) // -(-self.n_rows // self.slots)
            _assert_exact(_scatter(slot, y64.abs(), self.slots), 2, "sum y")
            _assert_exact(_scatter(slot, y64 * y64, self.slots), 4, "sum y^2")
            want = torch.stack([y64.sum(0), (y64 * y64).sum(0)])
            assert torch.equal(part.sum(0), want), f"{what}: column statistics differ from the exact sums"
            per = _scatter(slot, torch.stack([y64, y64 * y64], 1), self.slots)
            bad = (per != part).flatten(1).any(1)
            assert not bool(bad.any()), f"{what}: statistics slots {torch.nonzero(bad).flatten()[:8].tolist()} wrong"
        else:                                              # y = S / deg is not dyadic: any summation tree of n fp32 values
            n = self.n_rows + self.slots                   # (the squares fused) errs by at most gamma(n) of sum |terms|
            tol = _gamma(n) * torch.stack([y64.abs().sum(0), (y64 * y64).sum(0)]) * 1.01
            want = torch.stack([y64.sum(0), (y64 * y64).sum(0)])
            assert bool(((part.sum(0) - want).abs() <= tol).all()), f"{what}: column statistics outside gamma(n)"


@pytest.mark.parametrize("path", SPMM_PATHS, ids=[p[0] for p in SPMM_PATHS])
def test_spmm_exact_every_path_and_plan(path):
    """Sum with values and mean without, each with and without bias and with and without statistics, on both designed
    graphs under every plan: bit-exact Y, canaries outside Y intact, every statistics slot written and exact."""
    name, K, x_pad, x_c0, y_pad, y_c0, fused = path
    for plan, pid in zip(PLANS, PLAN_IDS):
        for kind in GRAPH_KINDS:
            case = SpmmCase(plan, kind, K, x_pad, x_c0, y_pad, y_c0)
            for reduce in (SUM, MEAN):
                for use_bias in (False, True):
                    for stats in (False, True):
                        case.check(reduce, use_bias, stats, fused,
                                   f"{name} {pid} {kind} {'sum' if reduce == SUM else 'mean'} bias={use_bias} stats={stats}")
            del case
            torch.cuda.empty_cache()


# ======================================================================================== SpMM: elementwise bound, real data
# Y_i = epilogue(sum_e val_e·X[col_e]).  The kernels form S_i with fused multiply-adds and additions of partial sums (lanes,
# groups, warps, hub segments, the finalize): one summation tree over deg_i exact products, so |S^ - S| <= gamma(deg_i)·M_i
# with M_i = (|A|·|X|)_i.  The epilogue: S^ / d rounded adds u·|S^ / d|, + bias rounded adds u·|S^ / d + b|; with
# |S^ / d| <= (1 + gamma)·M_i / d both are within 1.01·u·(2·M_i / d + |b|).  So, with d = max(deg, 1) for the mean, 1 for
# the sum:   |Y - Y64| <= gamma(deg_i)·M_i / d + 1.01·u·(2·M_i / d + |b|).
BOUND_PATHS = [p for p in SPMM_PATHS if p[0] in ("bulk256-K256", "bulk128-K384", "narrow-K40", "reg4-K200", "reg4multi-K516",
                                                 "reg2-K130", "reg1-K7", "reg1-K1025")]


@pytest.mark.parametrize("path", BOUND_PATHS, ids=[p[0] for p in BOUND_PATHS])
def test_spmm_elementwise_bound(path):
    """Random-normal X with source rows scaled by 2^e, e in [-20, 20], values in (0, 1]: every element within the bound
    above, on every plan; the worst ratio to the bound is printed."""
    name, K, x_pad, x_c0, y_pad, y_c0, _ = path
    worst = 0.0
    for plan in PLANS:
        for kind in GRAPH_KINDS:
            case = SpmmCase(plan, kind, K, x_pad, x_c0, y_pad, y_c0)
            rowptr, col, n_rows, n_src = designed(plan, kind)
            g = _gen("bound", plan, kind, K)
            x = torch.randn(n_src, K, generator=g, device=DEV) * torch.exp2(
                torch.randint(-20, 21, (n_src, 1), generator=g, device=DEV).float())
            case.X.reset(x)
            case.val = torch.rand(int(rowptr[-1]), generator=g, device=DEV).clamp_(min=2.0 ** -24)
            bias = torch.randn(K, generator=g, device=DEV)
            case.bias = bias
            rows, cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
            deg = case.deg.double()[:, None]
            for reduce in (SUM, MEAN):
                w = case.val.double()[:, None] if reduce == SUM else 1.0
                t = x.double()[cols] * w
                S, M = _scatter(rows, t, n_rows), _scatter(rows, t.abs(), n_rows)
                del t
                d = deg.clamp(min=1) if reduce == MEAN else torch.ones_like(deg)
                for use_bias in (False, True):
                    y = case.run(reduce, use_bias, stats=False).double()
                    b = bias.double() if use_bias else torch.zeros_like(bias.double())
                    ref = S / d + b
                    bound = _gamma(deg) * M / d + 1.01 * U * (2 * M / d + b.abs())
                    err = (y - ref).abs()
                    assert bool(torch.isfinite(y).all())
                    exact0 = bound == 0                        # empty rows without bias: exactly 0
                    assert bool((err[exact0] == 0).all())
                    worst = max(worst, float((err[~exact0] / bound[~exact0]).max()))
                    assert case.Y.outside_intact()
            del case
    print(f"\n{name}: worst |Y - Y64| / bound = {worst:.3g}")
    assert worst <= 1.0


# ============================================================================================================== GAT
def _transpose(rowptr: np.ndarray, col: np.ndarray, n_src: int):
    """CSR of the transposed graph (rows = sources, stable in edge order) and eidx (position of each edge in CSR order)."""
    perm = np.argsort(col, kind="stable")
    rowptr_t = np.concatenate([[0], np.cumsum(np.bincount(col, minlength=n_src))])
    row = np.repeat(np.arange(rowptr.size - 1), np.diff(rowptr))
    return rowptr_t, row[perm], perm


@functools.lru_cache(maxsize=None)
def device_graph_t(plan, kind: str):
    rowptr, col, n_rows, n_src = designed(plan, kind)
    rowptr_t, col_t, perm = _transpose(rowptr, col, n_src)
    g = CsrGraph(torch.from_numpy(rowptr_t).to(DEV, torch.int32), torch.from_numpy(col_t).to(DEV, torch.int32), None,
                 n_src, n_rows)
    return g.build_plan(*plan), torch.from_numpy(perm).to(DEV, torch.int32), rowptr_t, col_t, perm


def _hub_args(G: CsrGraph, ws: torch.Tensor | None):
    if not G.n_hub:
        return G.hub_threshold, G.seg_len, None, None, 0, 0, None
    return G.hub_threshold, G.seg_len, G.hub_rows.data_ptr(), G.hub_segptr.data_ptr(), G.n_hub, G.n_seg, ws.data_ptr()


def _pad_for(D: int) -> int:
    return 4 if D % 4 == 0 else (2 if D % 2 == 0 else 3)


# (H, D): float4 (D % 4 == 0, K <= 1536) with NJ = 1 / 1 / 2 / 4 / 8 / 12 vectors per lane; float2 (D % 4 == 2, K <= 768);
# float (D odd, K <= 384).  b200gnn_gat_aggregate_f32 picks the type, launch_agg the (NJ, U) shape.
AGG_SHAPES = [(4, 16), (1, 128), (8, 32), (3, 128), (16, 48), (12, 128), (3, 250), (5, 6), (3, 7), (16, 23)]


def _agg_ref(rows, cols, a64, ft64, n_out, H, D, what):
    """out[i, h·D + d] = sum_e a[e, h]·ft[col_e, h·D + d]; a in 2^-3 Z, ft integers: exact when 2^3·sum|terms| < 2^24."""
    terms = a64.repeat_interleave(D, dim=1) * ft64[cols]
    _assert_exact(_scatter(rows, terms.abs(), n_out), 3, what)
    return _scatter(rows, terms, n_out).float()


def _agg_c(G, eidx, a, ftv, outv, H, D, ws) -> int:
    return lib.load().b200gnn_gat_aggregate_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), None if eidx is None else eidx.data_ptr(), a.data_ptr(), ftv.data_ptr(),
        ftv.stride(0), outv.data_ptr(), outv.stride(0), G.n_rows, H, D, G.chunk_rowptr.data_ptr(), G.n_chunks,
        *_hub_args(G, ws), lib.stream_ptr())


@pytest.mark.parametrize("H,D", AGG_SHAPES)
def test_gat_aggregate_exact(H, D):
    """Forward CSR and transposed CSR with eidx (the d ft product), hub segments and finalize included, every plan."""
    K = H * D
    for plan in PLANS:
        for kind in GRAPH_KINDS:
            rowptr, col, n_rows, n_src = designed(plan, kind)
            G = device_graph(plan, kind)
            Gt, perm, rowptr_t, col_t, perm_np = device_graph_t(plan, kind)
            g = _gen("agg", plan, kind, H, D)
            a = _dyadic((int(rowptr[-1]), H), 0, 8, 3, g)
            ft = torch.randint(-2, 3, (n_src, K), generator=g, device=DEV).float()
            dout = torch.randint(-2, 3, (n_rows, K), generator=g, device=DEV).float()
            rows, cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
            ref = _agg_ref(rows, cols, a.double(), ft.double(), n_rows, H, D, "gat out")
            ref_t = _agg_ref(_row_index(rowptr_t), torch.from_numpy(col_t).to(DEV), a.double()[perm.long()], dout.double(),
                             n_src, H, D, "gat d ft")
            for graph, eidx, src, want, n_out in ((G, None, ft, ref, n_rows), (Gt, perm, dout, ref_t, n_src)):
                fv = Boxed(src.shape[0], K, K + _pad_for(D), extra_rows=4)
                fv.reset(src)
                out = Boxed(n_out, K, K + _pad_for(D), r0=2)
                out.reset()
                ws = _nan_flat(graph.n_seg * K)
                lib.check(_agg_c(graph, eidx, a, fv.view, out.view, H, D, ws), "gat_aggregate_f32")
                torch.cuda.synchronize()
                bad = (out.view != want).any(1)
                assert not bool(bad.any()), (plan, kind, eidx is not None, torch.nonzero(bad).flatten()[:8].tolist())
                assert out.outside_intact(), (plan, kind, eidx is not None)


def test_gat_aggregate_rejects_k1540():
    """K = 1540 with D % 4 == 0 is past every vector type's limit (float4: 1536): B200GNN_ERR_UNSUPPORTED, nothing written."""
    plan, kind = PLANS[0], "edges"
    rowptr, _, n_rows, n_src = designed(plan, kind)
    G = device_graph(plan, kind)
    H, D = 1, 1540
    a = torch.full((int(rowptr[-1]), H), 0.5, device=DEV)
    ft = torch.ones(n_src, D, device=DEV)
    out = Boxed(n_rows, D, D + 4)
    out.reset()
    rc = _agg_c(G, None, a, ft, out.view, H, D, _nan_flat(G.n_seg * D))
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED
    assert out.outside_intact() and bool(torch.isnan(out.view).all())


# (H, D) of the backward: SEG reduction (W == 4, D/4 a power of two <= 32, NJ·log2(D/4) < 5·H in launch_bwd_nj) for
# (8, 32), (16, 4), (16, 32); whole-warp sums for (1, 128), (4, 256), (12, 128) (float4), (3, 250) (float2), (2, 7) (float).
BWD_SHAPES = [(8, 32), (16, 4), (16, 32), (1, 128), (4, 256), (12, 128), (3, 250), (2, 7)]
SLOPE = 0.25


def _bwd_c(G, a, ftv, doutv, el, er, H, D, dpre, der, ws, scale) -> int:
    return lib.load().b200gnn_gat_bwd_rows_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), a.data_ptr(), ftv.data_ptr(), ftv.stride(0), doutv.data_ptr(), doutv.stride(0),
        el.data_ptr(), None if er is None else er.data_ptr(), G.n_rows, H, D, SLOPE, dpre.data_ptr(),
        None if der is None else der.data_ptr(), G.chunk_rowptr.data_ptr(), G.n_chunks, *_hub_args(G, ws),
        None if scale is None else scale.data_ptr(), lib.stream_ptr())


def _bwd_data(plan, kind, H, D, with_scale: bool):
    """ft, dout in {-1, 0, 1}; el, er in 2^-3 Z ∩ [-2, 2]; a in 2^-3 Z ∩ [0, 1] with about 64 non-zero entries per row on
    rows longer than that (so that S, d er stay exact on the hubs), attn_scale in {0, 2}."""
    rowptr, col, n_rows, n_src = designed(plan, kind)
    nnz = int(rowptr[-1])
    g = _gen("bwd", plan, kind, H, D, with_scale)
    deg = _deg(rowptr)
    rows = _row_index(rowptr)
    keep_p = (64.0 / deg.double().clamp(min=1)).clamp(max=1.0)[rows]
    a = _dyadic((nnz, H), 0, 8, 3, g) * (torch.rand(nnz, H, generator=g, device=DEV, dtype=torch.float64)
                                          < keep_p[:, None]).float()
    ft = torch.randint(-1, 2, (n_src, H * D), generator=g, device=DEV).float()
    dout = torch.randint(-1, 2, (n_rows, H * D), generator=g, device=DEV).float()
    el, er = _dyadic((n_src, H), -16, 16, 3, g), _dyadic((n_rows, H), -16, 16, 3, g)
    scale = (torch.randint(0, 2, (nnz, H), generator=g, device=DEV) * 2).float() if with_scale else None
    return a, ft, dout, el, er, scale


def _bwd_ref(rowptr, col, a, ft, dout, el, er, scale, H, D):
    """d a = <ft[src, h], dout[dst, h]> (·scale); S = sum_e a·d a; d pre = a (d a - S)·leaky'(el + er); d er = sum_e d pre.
    Grids: d a integer, S in 2^-3 Z, a (d a - S) in 2^-6 Z, d pre in 2^-8 Z."""
    n_rows = rowptr.size - 1
    rows, cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
    prod = (ft.double()[cols] * dout.double()[rows]).view(-1, H, D)
    da = prod.sum(2)
    _assert_exact(prod.abs().sum(2), 0, "d a")
    if scale is not None:
        da = da * scale.double()
    a64 = a.double()
    S = _scatter(rows, a64 * da, n_rows)
    _assert_exact(_scatter(rows, (a64 * da).abs(), n_rows), 3, "S")
    diff = da - S[rows]
    _assert_exact(da.abs() + S[rows].abs(), 3, "d a - S")
    de = a64 * diff
    _assert_exact(de.abs(), 6, "a (d a - S)")
    pre = el.double()[cols] + (er.double()[rows] if er is not None else 0.0)
    dp = torch.where(pre > 0, de, de * SLOPE)
    _assert_on_grid(dp, 8, "d pre")
    der = _scatter(rows, dp, n_rows)
    _assert_exact(_scatter(rows, dp.abs(), n_rows), 8, "d er")
    return dp.float(), der.float()


@pytest.mark.parametrize("H,D", BWD_SHAPES)
def test_gat_bwd_rows_exact(H, D):
    """d pre and d er bit-exact, attn_scale absent and in {0, 2}, hub rows (S assembled from the segment partials in
    gat_bwd_hub_finalize_kernel) included, every plan; one shape without er (d er not requested)."""
    K = H * D
    for plan in PLANS:
        for kind in GRAPH_KINDS:
            rowptr, col, n_rows, n_src = designed(plan, kind)
            G = device_graph(plan, kind)
            nnz = int(rowptr[-1])
            for with_scale in (False, True):
                a, ft, dout, el, er, scale = _bwd_data(plan, kind, H, D, with_scale)
                if (H, D) == (2, 7):
                    er = None
                dp_ref, der_ref = _bwd_ref(rowptr, col, a, ft, dout, el, er, scale, H, D)
                fv = Boxed(n_src, K, K + _pad_for(D), extra_rows=4)
                fv.reset(ft)
                dv = Boxed(n_rows, K, K + _pad_for(D), extra_rows=4)
                dv.reset(dout)
                dpre = Boxed(nnz, H, H, r0=1)
                dpre.reset()
                der = Boxed(n_rows, H, H, r0=1)
                der.reset()
                ws = _nan_flat(G.n_seg * H)
                lib.check(_bwd_c(G, a, fv.view, dv.view, el, er, H, D, dpre.view, der.view if er is not None else None, ws,
                                 scale), "gat_bwd_rows_f32")
                torch.cuda.synchronize()
                what = (plan, kind, with_scale)
                bad = (dpre.view != dp_ref).any(1)
                assert not bool(bad.any()), (what, "d pre", torch.nonzero(bad).flatten()[:8].tolist())
                assert dpre.outside_intact(), what
                if er is not None:
                    bad = (der.view != der_ref).any(1)
                    assert not bool(bad.any()), (what, "d er", torch.nonzero(bad).flatten()[:8].tolist())
                assert der.outside_intact(), what
                if er is None:
                    assert bool(torch.isnan(der.view).all()), what


@pytest.mark.parametrize("H", [1, 3, 16])
def test_segment_sum_heads_exact(H):
    """out[j, h] = sum_k vals[eidx[k], h] over the transposed rows (d el), and over the forward rows without eidx: rows of
    degree 512 (the last one a warp takes) and 513 (the CTA's), the hub, empty rows."""
    plan = PLANS[0]
    for kind in GRAPH_KINDS:
        rowptr, col, n_rows, n_src = designed(plan, kind)
        Gt, perm, rowptr_t, _, _ = device_graph_t(plan, kind)
        G = device_graph(plan, kind)
        nnz = int(rowptr[-1])
        assert {512, 513} <= set(np.diff(rowptr).tolist())
        vals = _dyadic((nnz, H), -8, 8, 3, _gen("segsum", kind, H))
        for graph, eidx, rp, n in ((G, None, rowptr, n_rows), (Gt, perm, rowptr_t, n_src)):
            v = vals.double() if eidx is None else vals.double()[eidx.long()]
            rows = _row_index(rp)
            _assert_exact(_scatter(rows, v.abs(), n), 3, "segment sum")
            want = _scatter(rows, v, n).float()
            out = Boxed(n, H, H, r0=2)
            out.reset()
            lib.check(lib.load().b200gnn_segment_sum_heads_f32(graph.rowptr.data_ptr(),
                                                                None if eidx is None else eidx.data_ptr(), vals.data_ptr(),
                                                                n, H, out.view.data_ptr(), lib.stream_ptr()),
                      "segment_sum_heads_f32")
            torch.cuda.synchronize()
            bad = (out.view != want).any(1)
            assert not bool(bad.any()), (kind, eidx is not None, torch.nonzero(bad).flatten()[:8].tolist())
            assert out.outside_intact()


# ------------------------------------------------------------------------------------------------- edge softmax: bound
# a_k = exp(x_k - m) / (sum_j exp(x_j - m) + eps), x = leaky_relu(el[src] + er[dst]), m = max_j x_j over the kept edges.
# The kernel's errors, with u = 2^-24:
#   pre^ = fl(el + er) = pre (1 + d1):                      |pre^ - pre| <= u |pre|;
#   x^ = pre^ or fl(slope · pre^) (slope <= 1):             |x^ - x| <= u |pre| + u (1 + u) |pre| <= 2.01 u |pre|;
#   m^ = max x^ (exact);  t^ = fl(x^ - m^):                 |t^ - (x^ - m^)| <= u |x^ - m^| <= 1.01 u (|pre| + |m|);
#   so t^_k = x_k - m^ + phi_k with |phi_k| <= Phi_k = 1.01 u (3 |pre_k| + |m|)   (m^ cancels in the ratio);
#   e^ = expf(t^) = exp(t^)(1 + eps_e), |eps_e| <= 2 ulp <= 4u: the CUDA C++ Programming Guide's maximum error of expf
#        (2 ulp over the full range, without -use_fast_math, which build.py does not pass);
#   s^ = the kept e^ summed in any tree:                    s^ = sum_j e^_j (1 + eta_j), |eta_j| <= gamma(deg);
#   eps in {0, 1e-16} vanishes in fl(s^ + eps) (s^ >= 1: the arg-max edge gives expf(0) = 1, and 1e-16 < u/2);
#   one division:                                           (1 + d3), |d3| <= u.
# With w_j = exp(x_j - m^), a^_k / a_k = e^{phi_k} (1 + eps_e)(1 + d3) / sum_j w~_j e^{phi_j} (1 + eps_j)(1 + eta_j) (w~ the
# normalised weights), which lies in [1/c', c'] with c' = e^{Phi_k + Phi_max} (1 + 4u)(1 + u) / ((1 - 4u)(1 - gamma(deg))).
# The fp64 reference keeps eps: a64 = a_k (1 - eps / (s + eps)).  Hence |a - a64| <= (c' - 1 + 2 eps / s) · a64 =: c · a64.
EXPF_ULP = 2


def _softmax_ref_and_bound(rowptr, col, el, er, keep, slope, eps, H):
    n_rows = rowptr.size - 1
    rows, cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
    kept = keep.bool()[:, None].expand(-1, H)
    pre = el.double()[cols] + er.double()[rows]
    x = torch.where(pre > 0, pre, pre * slope)
    m = torch.full((n_rows, H), -np.inf, dtype=torch.float64, device=DEV)
    m = m.scatter_reduce(0, rows[:, None].expand(-1, H), torch.where(kept, x, -np.inf), "amax")
    e = torch.where(kept, torch.exp(x - m[rows]), 0.0)
    s = _scatter(rows, e, n_rows)
    a64 = torch.where(kept, e / (s[rows] + eps), 0.0)
    nkept = _scatter(rows, kept.double(), n_rows)
    mrow = torch.where(torch.isfinite(m), m.abs(), 0.0)
    phi = 1.01 * U * (3 * pre.abs() + mrow[rows])
    phi_max = torch.zeros(n_rows, H, dtype=torch.float64, device=DEV).scatter_reduce(
        0, rows[:, None].expand(-1, H), torch.where(kept, phi, 0.0), "amax")
    ulp4 = 2 * EXPF_ULP * U
    cp = torch.exp(phi + phi_max[rows]) * (1 + ulp4) * (1 + U) / ((1 - ulp4) * (1 - _gamma(nkept[rows])))
    c = cp - 1 + 2 * eps / s[rows].clamp(min=1.0)
    return a64, c, kept


@pytest.mark.parametrize("H", [1, 3, 16])
@pytest.mark.parametrize("eps", [0.0, 1e-16])
def test_gat_edge_softmax_bound(H, eps):
    """Slope 0.2, edge_keep with about 20% of the edges dropped and one row (of degree 513) dropped entirely: every kept
    coefficient within c·a64 (the bound above), every dropped one exactly 0; the worst ratio is printed."""
    slope = 0.2
    worst = 0.0
    plan = PLANS[0]
    for kind in GRAPH_KINDS:
        rowptr, col, n_rows, n_src = designed(plan, kind)
        G = device_graph(plan, kind)
        nnz = int(rowptr[-1])
        g = _gen("softmax", kind, H, eps)
        el = torch.randn(n_src, H, generator=g, device=DEV) * 2
        er = torch.randn(n_rows, H, generator=g, device=DEV) * 2
        keep = (torch.rand(nnz, generator=g, device=DEV) >= 0.2).to(torch.uint8)
        r513 = int(np.flatnonzero(np.diff(rowptr) == 513)[0])
        keep[int(rowptr[r513]):int(rowptr[r513 + 1])] = 0
        for kp in (None, keep):
            k = torch.ones(nnz, dtype=torch.uint8, device=DEV) if kp is None else kp
            a64, c, kept = _softmax_ref_and_bound(rowptr, col, el, er, k, slope, eps, H)
            out = Boxed(nnz, H, H, r0=1)
            out.reset()
            lib.check(lib.load().b200gnn_gat_edge_softmax_f32(
                G.rowptr.data_ptr(), G.col.data_ptr(), el.data_ptr(), er.data_ptr(), n_rows, H, slope, eps,
                out.view.data_ptr(), None if kp is None else kp.data_ptr(), lib.stream_ptr()), "gat_edge_softmax_f32")
            torch.cuda.synchronize()
            a = out.view.double()
            assert out.outside_intact()
            assert bool((a[~kept] == 0).all()), "a dropped edge has a non-zero coefficient"
            ratio = (a - a64).abs()[kept] / (c * a64)[kept]
            assert bool(torch.isfinite(ratio).all())
            worst = max(worst, float(ratio.max()))
    print(f"\nedge softmax H={H} eps={eps}: worst |a - a64| / (c·a64) = {worst:.3g}")
    assert worst <= 1.0


# ====================================================================================== variant-knob families (tuning only)
# The families the automatic dispatch never selects, kept apart so that removing the knob removes this test and nothing
# else: 1 register-staged, 2 cp.async ring, 3-7 bulk-copy ring geometries, +16 evict_last, +32 the other barrier-group
# size, +64 two CTAs per SM, +128 eight gathers in flight in the narrow kernel; 8 (an unassigned low nibble) falls through
# to the automatic choice.  In scatter mode only the bulk-copy kernels (0, 3-7) and the narrow kernel may run: every other
# family must be refused before it launches a kernel that ignores the scatter.
KNOB_VARIANTS = [1, 2, 3, 4, 5, 6, 7, 8, 3 + 16, 4 + 32, 5 + 16 + 32, 3 + 64, 128]
KNOB_K = [16, 40, 128, 256, 384, 512]


def _scatter_c(G, val, xv, dst_ptrs, row_off, ld_dst, col_dst, K, reduce, bias, ws) -> int:
    import ctypes as C
    ptrs = (C.c_void_p * len(dst_ptrs))(*[C.c_void_p(int(p)) for p in dst_ptrs])
    offs = (C.c_int32 * len(row_off))(*[int(v) for v in row_off])
    return lib.load().b200gnn_spmm_csr_scatter_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), None if val is None else val.data_ptr(), xv.data_ptr(), xv.stride(0), ptrs,
        offs, len(dst_ptrs), ld_dst, col_dst, G.n_rows, G.n_cols, K, reduce, None if bias is None else bias.data_ptr(),
        G.chunk_rowptr.data_ptr(), G.n_chunks, G.hub_threshold, G.seg_len, G.hub_rows.data_ptr() if G.n_hub else None,
        G.hub_segptr.data_ptr() if G.n_hub else None, G.n_hub, G.n_seg, None if ws is None else ws.data_ptr(),
        lib.stream_ptr())


@pytest.fixture
def spmm_variant():
    L = lib.load()
    yield L.b200gnn_spmm_set_variant
    L.b200gnn_spmm_set_variant(0)


@pytest.mark.parametrize("variant", KNOB_VARIANTS)
def test_spmm_knob_families_exact(variant, spmm_variant):
    """Every knob family on two plans, with the exact check of the automatic paths (statistics slots included), and in
    scatter mode over two ranks: an exact scatter or B200GNN_ERR_UNSUPPORTED with nothing written."""
    for plan in (PLANS[0], PLANS[2]):
        for kind in GRAPH_KINDS:
            for K in KNOB_K:
                case = SpmmCase(plan, kind, K, 4, 0, 4, 0)
                spmm_variant(variant)
                for reduce in (SUM, MEAN):
                    for use_bias in (False, True):
                        for stats in (False, True):
                            case.check(reduce, use_bias, stats, True, f"variant {variant} K={K} {plan} {kind}")
                # scatter mode over 2 ranks, local buffers with a NaN canary block
                world, n = 2, case.n_rows
                off = [0, n // 2, n]
                ld = 2 * K + 4
                dst = [Boxed(off[q + 1] - off[q], K, ld, c0=K) for q in range(world)]
                for d in dst:
                    d.reset()
                case.ws.view(torch.int32).fill_(NAN_BITS)
                rc = _scatter_c(case.G, case.val, case.X.view, [d.flat.data_ptr() for d in dst], off, ld, K, K, SUM,
                                case.bias, case.ws)
                torch.cuda.synchronize()
                fam = variant & 15
                allowed = (K % 128 == 0 and (fam == 0 or 3 <= fam <= 7)) or (K <= 64 and fam not in (1, 2))
                if not allowed:
                    assert rc == ERR_UNSUPPORTED, (variant, K, rc)
                    assert all(bool(torch.isnan(d.view).all()) and d.outside_intact() for d in dst), (variant, K)
                else:
                    lib.check(rc, "spmm_csr_scatter_f32")
                    for q in range(world):
                        assert torch.equal(dst[q].view, case.refb[SUM][off[q]:off[q + 1]]), (variant, K, q)
                        assert dst[q].outside_intact(), (variant, K, q)
                spmm_variant(0)
                del case
