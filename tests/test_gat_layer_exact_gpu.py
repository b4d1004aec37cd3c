"""Contract of the fused GAT-layer kernels (gat.cu): the epilogue and ELU aggregations, the attention scores and their
backward, the ELU backward and the PPI logits / loss tail, through the C ABI with the pitches, alignments and plans chosen
here.  The designed graphs, the five plans and the poisoned buffers are test_sparse_exact_gpu.py's.

* gat_aggregate_epi: out = row_scale·Σ_e a[e,h]·src_scale[col_e]·ft[col_e] + res + bias.  On dyadic data (a in 2^-3 Z,
  src_scale and row_scale in {1/2, 1, 2}, ft in {-1, 0, 1}, res and bias in 2^-5 Z) every term is a multiple of 2^-4 and
  every output of 2^-5, so each sum is exact in fp32 whatever its order (`_assert_exact` checks the claim in fp64) and the
  output must equal the fp64 scatter sum bit for bit: each operand alone and all together, forward (eidx = NULL) and on the
  transposed graph with eidx = perm and the two scale vectors swapped (the engine's d ft call).  The statistics slots must
  hold exactly their own rows: slot c the non-hub rows of chunks [8c, 8c + 8), slot n_main + i hub row i; exact where
  the dyadic claim holds for the slot's sums, within gamma(rows + 8) of their magnitude where it does not.  On real data
  the output is bit-identical to gat_aggregate_f32 on a·src_scale followed by the fp32 epilogue in the kernel's order,
  with the plain aggregation run on views that select the same vector width (so the same U and hub-segment order).
  Every (V, NJ) instantiation is reached, by shape and by layout alone (odd ldr, an 8-byte res base, a 4-byte bias).
* gat_aggregate_elu: Z equals the epi output bit for bit; act = expm1f(Z) within 1 ulp (2u relative) of fp64 elu(Z).
  res nearly cancels the sum on half of the entries, so Z in (-1e-3, 0) on hub and chunk rows: expf(Z) - 1 loses every
  significant bit there to cancellation and must violate the bound.
* gat_scores / gat_scores_bwd: the fp64 bounds of test_engine_gat_gpu.py, at n = 1, 63, 64, 65, 3001 and 40,000 (past the
  2,112-CTA grid and the 528-slot cap), H = 16, K = 1536, D not a multiple of 32, NaN columns past K, no src_scale, no
  attn_r.
* elu_bwd: dZ = dA·(Z > 0 ? 1 : expf(Z)) within (1 + 4u)(1 + u) - 1 of fp64 (expf 2 ulp, one product), exact where
  Z > 0 or Z = ±0, on the float4 and the scalar path, past the 1,056-CTA grid.
* ppi_logits_loss: the logits equal a CPU fp32 restatement of the kernel's association bit for bit; d_agg = d_res / H bit
  for bit; the loss and d_res obey elementwise bounds derived below (`tail_reference`).

Poisoned views throughout: operands inside NaN buffers with wider pitches, outputs NaN-filled inside NaN canaries that must
survive bit for bit, NaN-filled workspaces and partial buffers; a second identical call gives identical bits; a refusal
returns its code with b200gnn_launch_count() unchanged and every output untouched.  The worst ratio of each bounded
family to its bound is printed at the end of the module."""
import math

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib
from test_sparse_exact_gpu import (DEV, ERR_UNSUPPORTED, GRAPH_KINDS, NAN_BITS, PLAN_IDS, PLANS, U, Boxed, _agg_c,
                                   _assert_exact, _dyadic, _gamma, _gen, _hub_args, _nan_flat, _row_index, _scatter,
                                   _slot_of_row, designed, device_graph, device_graph_t)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

ERR_BAD_ARG = -1                                      # B200GNN_ERR_BAD_ARG (include/b200gnn.h)
UD = 2.0 ** -53
TINY = 2.0 ** -148                                    # two ulps of the fp32 subnormal range
WORST = {}


def _record(family: str, r: float) -> None:
    assert r <= 1.0, (family, r)
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    if WORST:
        print("\nworst bound ratio per family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound; a zero bound demands an exact result."""
    assert bool(torch.isfinite(out).all()), "non-finite output"
    err = (out.double() - ref).abs()
    bound = torch.as_tensor(bound, dtype=torch.float64, device=err.device).expand_as(err)
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def _p(t):
    return None if t is None else t.data_ptr()


def _bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int32).clone()


def _boxed(x: torch.Tensor, ld: int, c0: int = 0, r0: int = 0) -> Boxed:
    b = Boxed(x.shape[0], x.shape[1], ld, c0=c0, r0=r0)
    b.reset(x)
    return b


def _untouched(*boxes: Boxed) -> bool:
    return all(b.outside_intact() and bool((b.view.contiguous().view(torch.int32) == NAN_BITS).all()) for b in boxes)


# ================================================================================== 1. epilogue and ELU aggregations
# (id, H, D, layout).  b200gnn_gat_aggregate_epi_f32 picks the vector width W from D, the pitches and the base alignments of
# ft / out / res / bias; launch_agg_epi the (NJ, U) shape from nj = ceil(K / W / 32): float4 NJ 1 / 2 / 4 / 8 / 12 for
# nj <= 1 / 2 / 4 / 8 / more, float2 and float NJ 4 / 12.  The last three reach a narrower width by layout alone.
EPI_SHAPES = [
    ("f4-nj1", 1, 40, "natural"),
    ("f4-nj2", 8, 32, "natural"),
    ("f4-nj4", 3, 128, "natural"),
    ("f4-nj8", 4, 256, "natural"),
    ("f4-nj8-ppi", 6, 124, "natural"),
    ("f4-nj8-arxiv", 3, 256, "natural"),
    ("f4-nj12", 16, 96, "natural"),
    ("f2-nj4", 5, 6, "natural"),
    ("f2-nj12", 3, 250, "natural"),
    ("f1-nj4", 3, 7, "natural"),
    ("f1-nj12-203", 7, 29, "natural"),        # nj = 7: a NJ = 4 instantiation would leave columns >= 128 unwritten
    ("f1-nj12-368", 16, 23, "natural"),
    ("f1-ldr-odd", 8, 32, "ldr-odd"),          # ldr = K + 1
    ("f2-res8", 8, 32, "res8"),                # res base 8 bytes into its buffer, ldr % 4 == 0
    ("f1-bias4", 8, 32, "bias4"),              # bias base 4 bytes into its buffer
]
EPI_IDS = [s[0] for s in EPI_SHAPES]
PAD_OF_W = {4: 4, 2: 2, 1: 1}                 # a pitch K + pad that lets exactly width W (and nothing wider) through


def _epi_width(D: int, layout: str) -> int:
    if layout in ("ldr-odd", "bias4"):
        return 1
    if layout == "res8":
        return 2
    return 4 if D % 4 == 0 else (2 if D % 2 == 0 else 1)


def _epi_c(G, eidx, a, ftv, outv, H, D, ss, rs, resv, bias, stat, slots, ws) -> int:
    return lib.load().b200gnn_gat_aggregate_epi_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), _p(eidx), a.data_ptr(), ftv.data_ptr(), ftv.stride(0), outv.data_ptr(),
        outv.stride(0), G.n_rows, H, D, _p(ss), _p(rs), _p(resv), 0 if resv is None else resv.stride(0), _p(bias), _p(stat),
        slots, G.chunk_rowptr.data_ptr(), G.n_chunks, *_hub_args(G, ws), lib.stream_ptr())


def _elu_c(G, eidx, a, ftv, outv, actv, H, D, resv, bias, ws) -> int:
    return lib.load().b200gnn_gat_aggregate_elu_f32(
        G.rowptr.data_ptr(), G.col.data_ptr(), _p(eidx), a.data_ptr(), ftv.data_ptr(), ftv.stride(0), outv.data_ptr(),
        outv.stride(0), actv.data_ptr(), actv.stride(0), G.n_rows, H, D, _p(resv), 0 if resv is None else resv.stride(0),
        _p(bias), G.chunk_rowptr.data_ptr(), G.n_chunks, *_hub_args(G, ws), lib.stream_ptr())


def stat_slots(G) -> int:
    return int(lib.load().b200gnn_gat_stat_slots(G.n_chunks, G.n_hub))


def near_zero(shape, g) -> torch.Tensor:
    """Values in (-1e-3, -1e-5): where elu(z) = expm1(z) ≈ z and expf(z) - 1 keeps almost none of its significant bits."""
    return -(1e-5 + (1e-3 - 2e-5) * torch.rand(shape, generator=g, device=g.device, dtype=torch.float64))


class EpiCase:
    """One (plan, graph kind, direction, H, D, layout): the graph in use (the designed graph, or its transpose with eidx =
    perm), the poisoned operand / output buffers, and the data sets.  a is indexed in forward edge order; the scale vectors
    live on the forward sources (s_src) and rows (s_dst): forward src_scale = s_src, row_scale = s_dst; transposed src_scale =
    s_dst, row_scale = s_src (engine_gat.py's backward)."""

    def __init__(self, plan, kind, transposed: bool, H: int, D: int, layout: str):
        rowptr, col, n_rows, n_src = designed(plan, kind)
        self.H, self.D, self.K, self.layout = H, D, H * D, layout
        self.W = _epi_width(D, layout)
        self.nnz = int(rowptr[-1])
        self.n_src, self.n_rows = n_src, n_rows
        self.fwd_rows, self.fwd_cols = _row_index(rowptr), torch.from_numpy(col).to(DEV)
        if transposed:
            self.G, self.eidx, rp, cl, _ = device_graph_t(plan, kind)
            self.n_in, self.n_out = n_rows, n_src
        else:
            self.G, self.eidx, rp, cl = device_graph(plan, kind), None, rowptr, col
            self.n_in, self.n_out = n_src, n_rows
        self.transposed = transposed
        self.rows, self.cols = _row_index(rp), torch.from_numpy(cl).to(DEV)
        self.key = (plan, kind, transposed, H, D, layout)
        K = self.K
        pad = 4 if D % 4 == 0 else (2 if D % 2 == 0 else 3)
        self.ft = Boxed(self.n_in, K, K + pad, extra_rows=4)
        self.out = Boxed(self.n_out, K, K + pad, r0=2)
        self.act = Boxed(self.n_out, K, K + pad + 4, r0=1)
        ldr, rc0 = {"ldr-odd": (K + 1, 0), "res8": (K + 4, 2)}.get(layout, (K + pad, 0))
        self.res = Boxed(self.n_out, K, ldr, c0=rc0, extra_rows=2)
        self.bias = Boxed(1, K, K + 4, c0=1 if layout == "bias4" else 0)
        self.slots = stat_slots(self.G)
        self.stat = Boxed(self.slots, 2 * K, 2 * K, r0=1, extra_rows=1)
        self.ws = _nan_flat(self.G.n_seg * K)

    def scales(self, s_src, s_dst):
        return (s_dst, s_src) if self.transposed else (s_src, s_dst)

    def a_of_edges(self, a):
        """a in the order of the graph in use (what the kernel reads through eidx)."""
        return a if self.eidx is None else a[self.eidx.long()]

    def run_epi(self, a, ss=None, rs=None, res=False, bias=False, stat=False, rc_only=False):
        self.out.reset()
        self.stat.reset()
        self.ws.view(torch.int32).fill_(NAN_BITS)
        rc = _epi_c(self.G, self.eidx, a, self.ft.view, self.out.view, self.H, self.D, ss, rs, self.res.view if res else None,
                    self.bias.view[0] if bias else None, self.stat.view if stat else None, self.slots if stat else 0, self.ws)
        if rc_only:
            return rc
        lib.check(rc, "gat_aggregate_epi_f32")
        torch.cuda.synchronize()
        assert self.out.outside_intact(), (self.key, "a store outside out")
        assert self.stat.outside_intact(), (self.key, "a store outside the statistics slots")
        return self.out.view

    def run_elu(self, a):
        self.out.reset()
        self.act.reset()
        self.ws.view(torch.int32).fill_(NAN_BITS)
        lib.check(_elu_c(self.G, self.eidx, a, self.ft.view, self.out.view, self.act.view, self.H, self.D, self.res.view,
                         self.bias.view[0], self.ws), "gat_aggregate_elu_f32")
        torch.cuda.synchronize()
        assert self.out.outside_intact() and self.act.outside_intact(), (self.key, "a store outside Z / act")
        return self.out.view, self.act.view

    # ------------------------------------------------------------------------------------------------ dyadic data
    def dyadic_data(self):
        g = _gen("epi-dyadic", *self.key)
        a = _dyadic((self.nnz, self.H), 0, 8, 3, g)
        ft = torch.randint(-4, 5, (self.n_in, self.K), generator=g, device=DEV).div(4, rounding_mode="trunc").float()
        s_src = torch.exp2(torch.randint(-1, 2, (self.n_src,), generator=g, device=DEV).float())
        s_dst = torch.exp2(torch.randint(-1, 2, (self.n_rows,), generator=g, device=DEV).float())
        res = _dyadic((self.n_out, self.K), -32, 32, 5, g)
        bias = _dyadic((self.K,), -32, 32, 5, g)
        return a, ft, s_src, s_dst, res, bias

    def exact_sum(self, a, ft, ss):
        """fp64 S = Σ a·ss·ft and M = Σ |a·ss·ft| over the graph in use; terms in 2^-4 Z."""
        w = self.a_of_edges(a).double()
        if ss is not None:
            w = w * ss.double()[self.cols][:, None]
        terms = w.repeat_interleave(self.D, dim=1) * ft.double()[self.cols]
        S = _scatter(self.rows, terms, self.n_out)
        terms.abs_()
        M = _scatter(self.rows, terms, self.n_out)
        del terms
        _assert_exact(M, 4, f"{self.key} S")
        return S, M

    def check_dyadic(self):
        a, ft, s_src, s_dst, res, bias = self.dyadic_data()
        ss, rs = self.scales(s_src, s_dst)
        self.ft.reset(ft)
        self.res.reset(res)
        self.bias.reset(bias[None])
        sums = {False: self.exact_sum(a, ft, None), True: self.exact_sum(a, ft, ss)}
        combos = [(), ("ss",), ("rs",), ("res",), ("bias",), ("ss", "rs", "res", "bias")]
        for combo in combos:
            S, M = sums["ss" in combo]
            y, mag = S, M
            if "rs" in combo:
                y, mag = y * rs.double()[:, None], mag * rs.double()[:, None]
            if "res" in combo:
                y, mag = y + res.double(), mag + res.double().abs()
            if "bias" in combo:
                y, mag = y + bias.double(), mag + bias.double().abs()
            _assert_exact(mag, 5, f"{self.key} {combo} out")
            want = y.float()
            stat = len(combo) == 4
            out = self.run_epi(a, ss if "ss" in combo else None, rs if "rs" in combo else None, "res" in combo,
                               "bias" in combo, stat)
            bad = (out != want).any(1)
            assert not bool(bad.any()), (self.key, combo, torch.nonzero(bad).flatten()[:8].tolist())
            if stat:
                first = (_bits(out), _bits(self.stat.view))
                self.check_slots(want)
                self.run_epi(a, ss, rs, True, True, True)
                assert torch.equal(first[0], _bits(self.out.view)) and torch.equal(first[1], _bits(self.stat.view)), \
                    (self.key, "a second identical call differs")

    def check_slots(self, y: torch.Tensor):
        """Slot ownership: each slot equals the (Σy, Σy²) of exactly its rows, exact where the dyadic claim holds for the
        slot (y in 2^-5 Z, y² in 2^-10 Z), otherwise within gamma(rows + 8): a chunk slot is one warp chain per chunk and
        the 8 warps added in order, a hub slot one row and one rounded square."""
        G, K = self.G, self.K
        part = self.stat.view.view(self.slots, 2, K).double()
        assert bool(torch.isfinite(part).all()), (self.key, "a statistics slot left unwritten")
        slot = _slot_of_row(G, self.n_out)
        y64 = y.double()
        s = _scatter(slot, y64, self.slots)
        q = _scatter(slot, y64 * y64, self.slots)
        A = _scatter(slot, y64.abs(), self.slots)
        cnt = _scatter(slot, torch.ones(self.n_out, 1, dtype=torch.float64, device=DEV), self.slots)
        gam = _gamma(cnt + 8)
        ex_s, ex_q = A * 2.0 ** 5 < 2.0 ** 24, q * 2.0 ** 10 < 2.0 ** 24
        ok_s = torch.where(ex_s, part[:, 0] == s, (part[:, 0] - s).abs() <= gam * A)
        ok_q = torch.where(ex_q, part[:, 1] == q, (part[:, 1] - q).abs() <= gam * q)
        bad = ~(ok_s & ok_q).all(1)
        assert not bool(bad.any()), (self.key, "statistics slots", torch.nonzero(bad).flatten()[:8].tolist())
        n_main = self.slots - G.n_hub
        assert bool(ex_s[:n_main].all()), (self.key, "the data leaves a chunk slot's Σy inexact: ownership unchecked")
        if G.n_hub:                                     # hub slots: Σy is the row itself
            assert bool(ex_s[n_main:].all()) and bool((part[n_main:, 0] == s[n_main:]).all())
        inexact = ~(ex_s & ex_q).all(1)
        if bool(inexact.any()):
            i = torch.nonzero(inexact).flatten()
            _record("epi statistics slot (not dyadic-exact)",
                    _ratio(part[i], torch.stack([s[i], q[i]], 1), gam[i][:, :, None] * torch.stack([A[i], q[i]], 1)))

    # -------------------------------------------------------------------------------------------------- real data
    def real_data(self):
        g = _gen("epi-real", *self.key)
        a = torch.rand(self.nnz, self.H, generator=g, device=DEV)
        ft = torch.randn(self.n_in, self.K, generator=g, device=DEV)
        s_src = torch.rand(self.n_src, generator=g, device=DEV) + 0.5
        s_dst = torch.rand(self.n_rows, generator=g, device=DEV) + 0.5
        res = torch.randn(self.n_out, self.K, generator=g, device=DEV)
        bias = torch.randn(self.K, generator=g, device=DEV)
        return a, ft, s_src, s_dst, res, bias

    def check_real(self):
        """Bit-identical to the unfused composition: gat_aggregate_f32 on fp32(a·src_scale), then ·row_scale, + res,
        + bias in fp32, the plain aggregation on views of width W."""
        a, ft, s_src, s_dst, res, bias = self.real_data()
        ss, rs = self.scales(s_src, s_dst)
        self.ft.reset(ft)
        self.res.reset(res)
        self.bias.reset(bias[None])
        out = self.run_epi(a, ss, rs, True, True).clone()
        # the column of forward edge e in the graph in use: its source forward, its destination on the transpose
        a_s = a * ss[(self.fwd_rows if self.transposed else self.fwd_cols)][:, None]
        pad = PAD_OF_W[self.W]
        fv = _boxed(ft, self.K + pad)
        pv = Boxed(self.n_out, self.K, self.K + pad)
        pv.reset()
        lib.check(_agg_c(self.G, self.eidx, a_s, fv.view, pv.view, self.H, self.D, _nan_flat(self.G.n_seg * self.K)),
                  "gat_aggregate_f32")
        torch.cuda.synchronize()
        want = ((pv.view * rs[:, None]) + res) + bias
        bad = (out != want).any(1)
        assert not bool(bad.any()), (self.key, "unfused composition", torch.nonzero(bad).flatten()[:8].tolist())

    # ------------------------------------------------------------------------------------------------------- ELU
    def check_elu(self):
        """Z = the epi output (res, bias) bit for bit; act within 1 ulp of fp64 elu(Z); Z in (-1e-3, 0) on hub and chunk
        rows, where expf(Z) - 1 must violate the bound."""
        a, ft, _, _, _, bias = self.dyadic_data()
        g = _gen("epi-elu", *self.key)
        S, _ = self.exact_sum(a, ft, None)
        mask = torch.rand(self.n_out, self.K, generator=g, device=DEV) < 0.5
        res = torch.where(mask, (near_zero((self.n_out, self.K), g) - S - bias.double()).float(),
                          torch.randn(self.n_out, self.K, generator=g, device=DEV))
        self.ft.reset(ft)
        self.res.reset(res)
        self.bias.reset(bias[None])
        ref = self.run_epi(a, None, None, True, True).clone()
        Z, A = self.run_elu(a)
        first = (_bits(Z), _bits(A))
        assert torch.equal(Z, ref), (self.key, "Z differs from the epi output")
        Z, A = self.run_elu(a)
        assert torch.equal(first[0], _bits(Z)) and torch.equal(first[1], _bits(A)), (self.key, "a second call differs")
        z64 = Z.double()
        e64 = torch.where(z64 > 0, z64, torch.expm1(z64))
        bound = 2 * U * e64.abs()
        _record("elu act (expm1f, 1 ulp)", _ratio(A, e64, bound))
        near = (Z < 0) & (Z > -1e-3)
        hub = torch.zeros(self.n_out, dtype=torch.bool, device=DEV)
        if self.G.n_hub:
            hub[self.G.hub_rows[:self.G.n_hub].long()] = True
            assert bool(near[hub].any()), (self.key, "no Z in (-1e-3, 0) on a hub row")
        if not bool(hub.all()):                        # the all-hubs plan can leave no chunk row at all
            assert bool(near[~hub].any()), (self.key, "no Z in (-1e-3, 0) on a chunk row")
        wrong = torch.exp(Z[near]) - 1.0                # the expf(z) - 1 formulation, in fp32
        viol = (wrong.double() - e64[near]).abs() > bound[near]
        assert float(viol.double().mean()) > 0.9, (self.key, "expf(z) - 1 stays within the bound: the data cannot see it")


def _cases(H, D, layout):
    for plan, pid in zip(PLANS, PLAN_IDS):
        for kind in GRAPH_KINDS:
            for transposed in (False, True):
                yield EpiCase(plan, kind, transposed, H, D, layout)


@pytest.mark.parametrize("shape", EPI_SHAPES, ids=EPI_IDS)
def test_gat_aggregate_epi_exact(shape):
    """Dyadic: bit-exact for each epilogue operand alone and all together, statistics slots owned row by row, repeatable;
    real: bit-identical to the unfused composition.  Both graph kinds, forward and transposed with eidx, every plan."""
    _, H, D, layout = shape
    for case in _cases(H, D, layout):
        case.check_dyadic()
        case.check_real()
        del case
        torch.cuda.empty_cache()


@pytest.mark.parametrize("shape", EPI_SHAPES, ids=EPI_IDS)
def test_gat_aggregate_elu_exact(shape):
    _, H, D, layout = shape
    for case in _cases(H, D, layout):
        case.check_elu()
        del case
        torch.cuda.empty_cache()


def _refusal_case(H, D):
    plan, kind = PLANS[0], "edges"
    rowptr, _, n_rows, n_src = designed(plan, kind)
    G = device_graph(plan, kind)
    K = H * D
    g = _gen("refuse", H, D)
    a = _dyadic((int(rowptr[-1]), H), 0, 8, 3, g)
    ft = _boxed(torch.randn(n_src, K, generator=g, device=DEV), K + 4)
    out, act = Boxed(n_rows, K, K + 4), Boxed(n_rows, K, K + 4)
    res = _boxed(torch.randn(n_rows, K, generator=g, device=DEV), K + 4)
    bias = torch.randn(K, generator=g, device=DEV)
    return G, a, ft, out, act, res, bias


@pytest.mark.parametrize("H,D", [(5, 308), (5, 154), (5, 77)], ids=["K1540-float4", "K770-float2", "K385-float"])
def test_gat_aggregate_epi_elu_refuse_wide_rows(H, D):
    """K past every width's limit (float4 1536, float2 768, float 384) for the data's widest vector: UNSUPPORTED from both
    entry points, nothing launched, nothing written."""
    G, a, ft, out, act, res, bias = _refusal_case(H, D)
    K = H * D
    slots = stat_slots(G)
    stat = Boxed(slots, 2 * K, 2 * K)
    for b in (out, act, stat):
        b.reset()
    ws = _nan_flat(G.n_seg * K)
    before = lib.launch_count()
    rc = _epi_c(G, None, a, ft.view, out.view, H, D, None, None, res.view, bias, stat.view, slots, ws)
    rc2 = _elu_c(G, None, a, ft.view, out.view, act.view, H, D, res.view, bias, ws)
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED and rc2 == ERR_UNSUPPORTED, (rc, rc2)
    assert lib.launch_count() == before
    assert _untouched(out, act, stat)


def test_gat_aggregate_epi_refuses_a_short_statistics_buffer():
    H, D = 8, 32
    G, a, ft, out, _, res, bias = _refusal_case(H, D)
    K = H * D
    slots = stat_slots(G) - 1
    stat = Boxed(slots, 2 * K, 2 * K)
    out.reset()
    stat.reset()
    before = lib.launch_count()
    rc = _epi_c(G, None, a, ft.view, out.view, H, D, None, None, res.view, bias, stat.view, slots, _nan_flat(G.n_seg * K))
    torch.cuda.synchronize()
    assert rc == ERR_BAD_ARG and lib.launch_count() == before
    assert _untouched(out, stat)


@pytest.mark.parametrize("H,D,act_c0", [(8, 32, 2), (5, 6, 1)], ids=["float4-act8", "float2-act4"])
def test_gat_aggregate_elu_refuses_an_act_narrower_than_the_width(H, D, act_c0):
    """act aligned below the width the epi operands select (float4 -> 8 bytes, float2 -> 4 bytes): BAD_ARG, no launch."""
    G, a, ft, out, _, res, bias = _refusal_case(H, D)
    K = H * D
    if D % 4:                                               # float2 operands
        ft = _boxed(ft.view.clone(), K + 2)
        res = _boxed(res.view.clone(), K + 2)
        out = Boxed(out.view.shape[0], K, K + 2)
    act = Boxed(out.view.shape[0], K, K + 4, c0=act_c0)
    out.reset()
    act.reset()
    before = lib.launch_count()
    rc = _elu_c(G, None, a, ft.view, out.view, act.view, H, D, res.view, bias, _nan_flat(G.n_seg * K))
    torch.cuda.synchronize()
    assert rc == ERR_BAD_ARG and lib.launch_count() == before
    assert _untouched(out, act)


# ========================================================================================= 2. attention scores
# (n, H, D, attn_r, src_scale).  n = 40,000: rows_grid caps the forward at 2,112 CTAs (16,896 rows per sweep) and
# gat_scores_slots the backward at 528 slots of 76 rows.
SCORE_CASES = [
    (40_000, 16, 96, True, True),
    (40_000, 3, 12, False, False),
    (40_000, 5, 45, True, False),
    (1, 16, 96, True, True),
    (63, 3, 12, True, True),
    (64, 8, 32, False, True),
    (65, 1, 40, True, False),
    (3001, 16, 7, True, True),
]


@pytest.mark.parametrize("n,H,D,with_r,with_sc", SCORE_CASES)
def test_gat_scores_and_backward_bounds(n, H, D, with_r, with_sc):
    """el / er within (D + 6)·u of Σ|f·attn|; dft within 4u of its magnitude; d attn within the slot chain's gamma.  ft is a
    view with NaN columns past K; outputs among canaries; two identical calls give identical bits."""
    K = H * D
    L = lib.load()
    g = _gen("scores", n, H, D, with_r, with_sc)
    ft = _boxed(torch.randn(n, K, generator=g, device=DEV), K + 5)
    al = torch.randn(K, generator=g, device=DEV)
    ar = torch.randn(K, generator=g, device=DEV) if with_r else None
    sc = (torch.rand(n, generator=g, device=DEV) + 0.2) if with_sc else None
    el, er = Boxed(n, H, H, r0=1), Boxed(n, H, H, r0=1)
    outs = []
    for _ in range(2):
        el.reset()
        er.reset()
        lib.check(L.b200gnn_gat_scores_f32(ft.view.data_ptr(), ft.view.stride(0), al.data_ptr(), _p(ar), _p(sc), n, H, D,
                                           el.view.data_ptr(), er.view.data_ptr(), lib.stream_ptr()), "gat_scores_f32")
        torch.cuda.synchronize()
        outs.append((_bits(el.view), _bits(er.view)))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    assert el.outside_intact() and er.outside_intact()
    f64 = ft.view.double().view(n, H, D)
    sc64 = sc.double().view(-1, 1) if with_sc else torch.ones(n, 1, dtype=torch.float64, device=DEV)
    gam = (D + 6) * U
    ref_l = (f64 * al.double().view(H, D)).sum(-1) * sc64
    _record("scores el", _ratio(el.view, ref_l, (f64.abs() * al.double().abs().view(H, D)).sum(-1) * sc64 * gam))
    if with_r:
        ref_r = (f64 * ar.double().view(H, D)).sum(-1)
        _record("scores er", _ratio(er.view, ref_r, (f64.abs() * ar.double().abs().view(H, D)).sum(-1) * gam))
    else:
        assert _untouched(er), "er written without attn_r"

    d_el = torch.randn(n, H, generator=g, device=DEV)
    d_er = torch.randn(n, H, generator=g, device=DEV) if with_r else torch.full((n, H), float("nan"), device=DEV)
    dft0 = torch.randn(n, K, generator=g, device=DEV)
    slots = int(L.b200gnn_gat_scores_slots(n))
    rows_per_cta = -(-n // slots)
    if n == 40_000:
        assert slots == 528 and rows_per_cta == 76
    dft = Boxed(n, K, K + 3)
    dal, dar = Boxed(1, K, K, r0=1), Boxed(1, K, K, r0=1)
    part = _nan_flat(slots * 2 * K)
    outs = []
    for _ in range(2):
        dft.reset(dft0)
        dal.reset()
        dar.reset()
        part.view(torch.int32).fill_(NAN_BITS)
        lib.check(L.b200gnn_gat_scores_bwd_f32(ft.view.data_ptr(), ft.view.stride(0), al.data_ptr(), _p(ar), _p(sc),
                                               d_el.data_ptr(), d_er.data_ptr(), n, H, D, dft.view.data_ptr(),
                                               dft.view.stride(0), dal.view.data_ptr(), dar.view.data_ptr(), part.data_ptr(),
                                               slots, lib.stream_ptr()), "gat_scores_bwd_f32")
        torch.cuda.synchronize()
        outs.append((_bits(dft.view), _bits(dal.view), _bits(dar.view)))
    assert all(torch.equal(x, y) for x, y in zip(*outs)), "a second identical call differs"
    assert dft.outside_intact() and dal.outside_intact() and dar.outside_intact()
    gl = (d_el.double() * sc64).view(n, H, 1)
    ref = dft0.double().view(n, H, D) + gl * al.double().view(H, D)
    mag = dft0.double().abs().view(n, H, D) + gl.abs() * al.double().abs().view(H, D)
    if with_r:
        ref = ref + d_er.double().view(n, H, 1) * ar.double().view(H, D)
        mag = mag + d_er.double().abs().view(n, H, 1) * ar.double().abs().view(H, D)
    _record("scores_bwd dft", _ratio(dft.view.reshape(n, H, D), ref, 4 * U * mag))
    gam_n = _gamma(rows_per_cta + slots + 4)
    _record("scores_bwd d attn_l", _ratio(dal.view[0], (gl * f64).sum(0).view(-1), gam_n * (gl.abs() * f64.abs()).sum(0).view(-1)))
    if with_r:
        gr = d_er.double().view(n, H, 1)
        _record("scores_bwd d attn_r", _ratio(dar.view[0], (gr * f64).sum(0).view(-1),
                                              gam_n * (gr.abs() * f64.abs()).sum(0).view(-1)))
    else:
        assert _untouched(dar), "d attn_r written without attn_r"


def test_gat_scores_bwd_refuses_k1537():
    """K = 1537 is past the 6 columns per thread of gat_scores_bwd_kernel: UNSUPPORTED, nothing launched or written."""
    n, H, D = 100, 1, 1537
    L = lib.load()
    g = _gen("scores-refuse")
    ft = torch.randn(n, D, generator=g, device=DEV)
    al = torch.randn(D, generator=g, device=DEV)
    d_el = torch.randn(n, H, generator=g, device=DEV)
    dft0 = torch.randn(n, D, generator=g, device=DEV)
    dft = _boxed(dft0, D + 3)
    dal = Boxed(1, D, D, r0=1)
    dal.reset()
    slots = int(L.b200gnn_gat_scores_slots(n))
    before = lib.launch_count()
    rc = L.b200gnn_gat_scores_bwd_f32(ft.data_ptr(), D, al.data_ptr(), None, None, d_el.data_ptr(), None, n, H, D,
                                      dft.view.data_ptr(), dft.view.stride(0), dal.view.data_ptr(), None,
                                      _nan_flat(slots * 2 * D).data_ptr(), slots, lib.stream_ptr())
    torch.cuda.synchronize()
    assert rc == ERR_UNSUPPORTED and lib.launch_count() == before
    assert torch.equal(dft.view, dft0) and dft.outside_intact() and _untouched(dal)


# ============================================================================================== 3. ELU backward
# (id, n, K, pad of dA, pad of Z, pad of dZ): n·K / W past the 1,056 × 256 threads of the capped grid.
ELU_BWD_CASES = [
    ("float4", 5000, 256, 4, 8, 4),
    ("scalar-odd-K", 3001, 121, 3, 1, 5),
    ("scalar-ldz", 5000, 256, 4, 2, 4),
]


@pytest.mark.parametrize("case", ELU_BWD_CASES, ids=[c[0] for c in ELU_BWD_CASES])
def test_elu_bwd_bound(case):
    """Z uniform in [-30, 30] with exact zeros and -0.0: exact dA where Z > 0 or Z = ±0, else within
    ((1 + 4u)(1 + u) - 1)·|dA·exp(Z)| (expf 2 ulp, one product rounding)."""
    _, n, K, pa, pz, po = case
    g = _gen("elu-bwd", *case)
    z = (torch.rand(n, K, generator=g, device=DEV) * 60 - 30)
    sel = torch.rand(n, K, generator=g, device=DEV)
    z[sel < 0.02] = 0.0
    z[sel > 0.98] = -0.0
    dA = torch.randn(n, K, generator=g, device=DEV)
    Zb, Gb = _boxed(z, K + pz), _boxed(dA, K + pa)
    out = Boxed(n, K, K + po, r0=1)
    outs = []
    for _ in range(2):
        out.reset()
        lib.check(lib.load().b200gnn_elu_bwd_f32(Gb.view.data_ptr(), Gb.view.stride(0), Zb.view.data_ptr(), Zb.view.stride(0),
                                                 out.view.data_ptr(), out.view.stride(0), n, K, lib.stream_ptr()), "elu_bwd_f32")
        torch.cuda.synchronize()
        outs.append(_bits(out.view))
    assert torch.equal(outs[0], outs[1]) and out.outside_intact()
    z64 = z.double()
    ref = dA.double() * torch.where(z64 > 0, torch.ones_like(z64), torch.exp(z64))
    ident = (z > 0) | (z == 0)
    assert int((z == 0).sum()) > 0 and int(torch.signbit(z[z == 0]).sum()) > 0
    assert torch.equal(out.view[ident], dA[ident]), "dZ differs from dA where Z > 0 or Z = ±0"
    _record("elu_bwd", _ratio(out.view[~ident], ref[~ident], ((1 + 4 * U) * (1 + U) - 1) * ref[~ident].abs()))


# =========================================================================================== 4. PPI logits tail
# (n, H, C, Dp, T, alpha, kd).  n = 10,007 is past the 528-slot cap of ppi_tail_slots (the grid-stride loop runs).
TAIL_CASES = [
    (10_007, 6, 121, 124, 2.0, 0.3, True),
    (10_007, 3, 121, 121, 0.5, 1.0, True),
    (10_007, 1, 40, 44, 1.0, 0.0, True),
    (10_007, 6, 121, 124, 1.0, 0.5, False),
    (10_007, 3, 19, 20, 2.0, 1.0, True),
    (1, 3, 121, 124, 2.0, 0.3, True),
    (1, 1, 7, 7, 0.5, 0.0, False),
]
TAIL_IDS = [f"n{c[0]}-H{c[1]}-C{c[2]}-Dp{c[3]}-T{c[4]}-a{c[5]}-{'kd' if c[6] else 'cls'}" for c in TAIL_CASES]


def tail_data(n, H, C, Dp, kd, seed=0):
    """CPU tensors: agg [n, H, Dp] and res [n, Dp] randn with NaN in the padded columns (the kernel must not read them),
    res at ±20 and ±100 on 5% of the entries each (so are the logits), labels in {0, 1}, teacher logits randn·2 with ±100
    on 5%."""
    g = torch.Generator().manual_seed(seed * 1000 + n + 10 * H + C)
    agg = torch.randn(n, H, Dp, generator=g)
    agg[:, :, C:] = float("nan")
    res = torch.randn(n, Dp, generator=g)
    sel = torch.rand(n, C, generator=g)
    sign = torch.where(torch.rand(n, C, generator=g) < 0.5, -1.0, 1.0)
    res[:, :C] = torch.where(sel < 0.05, 20.0 * sign, torch.where(sel > 0.95, 100.0 * sign, res[:, :C]))
    res[:, C:] = float("nan")
    bc, bl = torch.randn(Dp, generator=g), torch.randn(Dp, generator=g)
    y = (torch.rand(n, C, generator=g) < 0.3).float()
    t = None
    if kd:
        t = torch.randn(n, C, generator=g) * 2
        s2 = torch.rand(n, C, generator=g)
        t = torch.where(s2 < 0.05, 100.0 * sign, t)
    return agg, res, bc, bl, y, t


def tail_logits(agg, res, bc, bl, H, C):
    """The kernel's association in fp32: heads summed in order, / H, + b_conv, + (res + b_lin)."""
    s = agg[:, 0, :C].clone()
    for h in range(1, H):
        s = s + agg[:, h, :C]
    return (s / float(H) + bc[:C]) + (res[:, :C] + bl[:C])


def _f32(x: float) -> float:
    return float(torch.tensor(x, dtype=torch.float32))


def tail_reference(z, y, t, alpha, T, kd):
    """fp64 loss / d_res at the fp32 logits z, and their bounds, with alpha and T as the kernel receives them (fp32).

    Elementwise, u = 2^-24: expf(-|z|) errs by 2 ulp (4u relative, plus 2^-148 in the subnormal range), log1pf by 1 ulp, so
        |sp - sp64| <= 2u·sp64 + e_e / (1 + e);
    the sigmoid 1 / (1 + expf(-z)) by 4u·E/(1 + E) + 2u <= 6u relative, and all of it (sig64 < 3e-39) where expf(-z)
    overflows (z < -88);  the BCE term fl(fl(mz - fl(z·y)) + sp) against mz - z·y + sp by
        |z|·e_y + u·|z·y| + u·|mz - z·y| + u·|term| + e_sp,
    e_y = 0 for labels, e_tv for the teacher's sigmoid (the cancellation of mz against z·t is in the u·|z·t| term).  The
    fp64 sums (any order, gamma_d(N)·Σ|term|), the fp64 scaling by 1/N (2 ud) and the fp32 rounding u·|mean| follow, then
    alpha·T·T (2 roundings), 1 - alpha (1), two products and one sum for the loss.
    d_res = w_c·(sig - y) + w_k·(sig - tv), w_c = fp32((1 - alpha) / N) (or 1 / N), w_k = fp32(alpha·T² / N): each weight
    rounded (u), each difference e_sig (+ e_tv) + u of itself, each product u, the sum u.  A factor 1.01 covers the
    second-order terms."""
    n, C = z.shape
    N = n * C
    a32, T32 = _f32(alpha), _f32(T)
    z = z.double()
    y = y.double()
    az = z.abs()
    e = torch.exp(-az)
    e_e = 4 * U * e + TINY
    sp = torch.log1p(e)
    e_sp = 2 * U * sp + e_e / (1 + e)
    mz = z.clamp(min=0)

    def sigm(x):
        s = torch.sigmoid(x)
        return s, 6 * U * s + torch.where(x < -88, s, torch.zeros_like(s)) + TINY

    sig, e_sig = sigm(z)

    def bce(target, e_target):
        p = z * target
        d = mz - p
        term = d + sp
        B = 1.01 * (az * e_target + U * p.abs() + U * d.abs() + U * term.abs() + e_sp) + TINY
        mean = float(term.sum()) / N
        Bm = 1.01 * (float(B.sum()) / N + (float(_gamma_d(N + 1024)) + 2 * UD) * float(term.abs().sum()) / N
                     + U * abs(mean))
        return mean, Bm

    cls, B_cls = bce(y, torch.zeros_like(y))
    out = dict(cls=cls, B_cls=B_cls, dis=0.0, B_dis=0.0)
    if kd:
        tv, e_tv = sigm(t.double())
        out["dis"], out["B_dis"] = bce(tv, e_tv)
        w_c, w_k = (1.0 - a32) / N, a32 * T32 * T32 / N
        A, B = a32 * T32 * T32, 1.0 - a32
        out["loss"] = out["dis"] * A + cls * B
        out["B_loss"] = 1.01 * (A * (out["B_dis"] + 3 * U * abs(out["dis"])) + abs(B) * (B_cls + 2 * U * abs(cls))
                                + U * abs(out["loss"]))
    else:
        w_c, w_k = 1.0 / N, 0.0
        out["loss"], out["B_loss"] = cls, B_cls
    d1 = sig - y
    dz = w_c * d1
    Bd = abs(w_c) * (e_sig + U * d1.abs()) + 2 * U * abs(w_c) * d1.abs()
    if kd:
        d2 = sig - tv
        dz = dz + w_k * d2
        Bd = Bd + abs(w_k) * (e_sig + e_tv + U * d2.abs()) + 2 * U * abs(w_k) * d2.abs()
    out["dres"], out["B_dres"] = dz, 1.01 * (Bd + U * dz.abs()) + TINY
    return out


def _gamma_d(n):
    return n * UD / (1 - n * UD)


def _tail_c(agg, res, bc, bl, n, H, Dp, C, logits, y, t, alpha, T, dagg, dres, loss, part, slots) -> int:
    return lib.load().b200gnn_ppi_logits_loss_f32(
        agg.data_ptr(), agg.stride(0), res.data_ptr(), res.stride(0), bc.data_ptr(), bl.data_ptr(), n, H, Dp, C,
        logits.data_ptr(), logits.stride(0), _p(y), C if y is None else y.stride(0), _p(t), C if t is None else t.stride(0),
        alpha, T, _p(dagg), H * Dp if dagg is None else dagg.stride(0), _p(dres), Dp if dres is None else dres.stride(0),
        _p(loss), _p(part), slots, lib.stream_ptr())


class TailBuffers:
    def __init__(self, n, H, C, Dp, kd, seed=0):
        agg, res, bc, bl, y, t = tail_data(n, H, C, Dp, kd, seed)
        self.cpu = (agg, res, bc, bl, y, t)
        self.agg = _boxed(agg.reshape(n, H * Dp).to(DEV), H * Dp + 4)
        self.res = _boxed(res.to(DEV), Dp + 3)
        self.bc, self.bl = bc.to(DEV), bl.to(DEV)
        self.y = _boxed(y.to(DEV), C + 2)
        self.t = _boxed(t.to(DEV), C + 5) if kd else None
        self.logits = Boxed(n, C, C + 3, r0=1)
        self.dagg = Boxed(n, H * Dp, H * Dp + 8, r0=1)
        self.dres = Boxed(n, Dp, Dp + 4, r0=1)
        self.loss = Boxed(1, 3, 3, r0=1)
        self.slots = int(lib.load().b200gnn_ppi_tail_slots(n))
        self.part = torch.full((2 * self.slots + 2,), float("nan"), dtype=torch.float64, device=DEV)
        self.n, self.H, self.C, self.Dp = n, H, C, Dp

    def run(self, alpha, T, train=True):
        for b in (self.logits, self.dagg, self.dres, self.loss):
            b.reset()
        self.part.fill_(float("nan"))
        rc = _tail_c(self.agg.view, self.res.view, self.bc, self.bl, self.n, self.H, self.Dp, self.C, self.logits.view,
                     self.y.view if train else None, None if (self.t is None or not train) else self.t.view, alpha, T,
                     self.dagg.view, self.dres.view, self.loss.view[0], self.part, self.slots)
        lib.check(rc, "ppi_logits_loss_f32")
        torch.cuda.synchronize()
        for b in (self.logits, self.dagg, self.dres, self.loss):
            assert b.outside_intact(), "a store outside an output"
        return [_bits(b.view) for b in (self.logits, self.dagg, self.dres, self.loss)]


@pytest.mark.parametrize("n,H,C,Dp,T,alpha,kd", TAIL_CASES, ids=TAIL_IDS)
def test_ppi_logits_loss(n, H, C, Dp, T, alpha, kd):
    """Logits bitwise against the CPU restatement, d_agg = d_res / H bitwise, padding exactly 0, nothing past Dp; loss and
    d_res within the derived bounds, the loss bound below 1e-5 relative; two calls identical."""
    tb = TailBuffers(n, H, C, Dp, kd)
    first = tb.run(alpha, T)
    assert all(torch.equal(x, y) for x, y in zip(first, tb.run(alpha, T))), "a second identical call differs"
    agg, res, bc, bl, y, t = tb.cpu
    z = tail_logits(agg, res, bc, bl, H, C)
    assert torch.equal(tb.logits.view.cpu(), z), "logits differ from the fp32 restatement of the kernel's association"
    dres = tb.dres.view.cpu()
    dagg = tb.dagg.view.cpu().view(n, H, Dp)
    assert bool((dres[:, C:] == 0).all()) and bool((dagg[:, :, C:] == 0).all()), "padded gradient columns are not 0"
    assert torch.equal(dagg[:, :, :C], (dres[:, :C] / float(H))[:, None, :].expand(n, H, C)), "d_agg != d_res / H"
    ref = tail_reference(z, y, t, alpha, T, kd)
    loss = tb.loss.view[0].double().cpu()
    _record("ppi loss", abs(float(loss[0]) - ref["loss"]) / ref["B_loss"])
    _record("ppi loss_cls", abs(float(loss[1]) - ref["cls"]) / ref["B_cls"])
    if kd:
        _record("ppi loss_kd", abs(float(loss[2]) - ref["dis"]) / ref["B_dis"])
    else:
        assert float(loss[2]) == 0.0
    assert ref["B_loss"] < 1e-5 * abs(ref["loss"]), ("the loss bound is not below 1e-5 relative", ref["B_loss"] / ref["loss"])
    _record("ppi d_res", _ratio(dres[:, :C], ref["dres"], ref["B_dres"]))


def test_ppi_logits_loss_eval_writes_only_the_logits():
    n, H, C, Dp = 10_007, 6, 121, 124
    tb = TailBuffers(n, H, C, Dp, kd=True)
    tb.run(0.3, 2.0, train=False)
    agg, res, bc, bl, _, _ = tb.cpu
    assert torch.equal(tb.logits.view.cpu(), tail_logits(agg, res, bc, bl, H, C))
    assert _untouched(tb.dagg, tb.dres, tb.loss) and bool(torch.isnan(tb.part).all())


def test_ppi_logits_loss_refuses_n0_with_labels():
    H, C, Dp = 3, 7, 8
    tb = TailBuffers(1, H, C, Dp, kd=False)
    for b in (tb.logits, tb.dagg, tb.dres, tb.loss):
        b.reset()
    before = lib.launch_count()
    rc = _tail_c(tb.agg.view, tb.res.view, tb.bc, tb.bl, 0, H, Dp, C, tb.logits.view, tb.y.view, None, 0.5, 1.0,
                 tb.dagg.view, tb.dres.view, tb.loss.view[0], tb.part, tb.slots)
    torch.cuda.synchronize()
    assert rc == ERR_BAD_ARG and lib.launch_count() == before
    assert _untouched(tb.logits, tb.dagg, tb.dres, tb.loss)
