"""The GSP kernels of the captured step through the C ABI: the chunked pair pass against the two one-sided passes it replaces,
the GSP operands and backward against fp64 on designed rows, the chunk loop criterion.gsp_chunks against the unchunked
sequence it replaced, and its memory.

- b200gnn_gsp_pair_chunk_f32 stores, chunk by chunk, exactly what b200gnn_gsp_pair_f32(dGs, Gt, ns, nt) and
  b200gnn_gsp_pair_f32(dGt, Gs, nt, ns) store over the whole S x S matrices: both gradients, both row coefficients and the
  per-row partials, bit for bit, and b200gnn_gsp_finish_f32 then gives the same loss bits for every chunk size.
- b200gnn_gsp_operands_f32 / b200gnn_gsp_backward_f32 lie within fp64 bounds built from the rounding of each step; the ReLU
  masks are exact; rows outside the sample keep their NaN canaries.
"""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion as C, lib, ops

pytestmark = pytest.mark.gpu

OK, ERR_BAD_ARG = 0, -1
U = 2.0 ** -24                       # fp32 unit roundoff
KERNELS = [0, 1, 2, 3]
PAIR_S = [1, 7, 257, 600]


def _L():
    return lib.load()


def _st():
    return lib.stream_ptr()


def _p(t):
    return None if t is None else t.data_ptr()


def _ceil4(n):
    return (n + 3) // 4 * 4


def _refused(call, code=ERR_BAD_ARG):
    """The call returns `code` and launches nothing."""
    torch.cuda.synchronize()
    before = lib.launch_count()
    assert call() == code
    assert lib.launch_count() == before


def _nan(*shape):
    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


# ============================================================================================ 1. the chunked pair pass
def _grams(S, F, kernel, seed):
    """fp32 Gram matrices and squared norms of two row sets; rows 0 and 1 of the student repeat (zero l2 distance off the
    diagonal), the teacher's do not."""
    g = torch.Generator().manual_seed(seed)
    xs, xt = torch.randn(S, F, generator=g), torch.randn(S, F, generator=g) * 0.7
    if S > 1:
        xs[1] = xs[0]
    if kernel <= 1:
        xs, xt = torch.nn.functional.normalize(xs, dim=1), torch.nn.functional.normalize(xt, dim=1)
    Gs, Gt = (xs.double() @ xs.double().T).float(), (xt.double() @ xt.double().T).float()
    ns, nt = xs.double().pow(2).sum(1).float(), xt.double().pow(2).sum(1).float()
    return Gs.cuda(), Gt.cuda(), ns.cuda(), nt.cuda()


def _two_calls(Gs, Gt, ns, nt, S, kernel):
    """The sequence the chunk pass replaces: one one-sided pass per side over the whole matrices."""
    raw = kernel >= 2
    dGs, dGt = Gs.clone(), Gt.clone()
    rc_s, rc_t = (_nan(S), _nan(S)) if raw else (None, None)
    loss, loss2, part, part2 = _nan(1), _nan(1), _nan(S), _nan(S)
    assert _L().b200gnn_gsp_pair_f32(dGs.data_ptr(), Gt.data_ptr(), _p(ns if raw else None), _p(nt if raw else None), S, kernel,
                                     _p(rc_s), loss.data_ptr(), part.data_ptr(), _st()) == OK
    assert _L().b200gnn_gsp_pair_f32(dGt.data_ptr(), Gs.data_ptr(), _p(nt if raw else None), _p(ns if raw else None), S, kernel,
                                     _p(rc_t), loss2.data_ptr(), part2.data_ptr(), _st()) == OK
    return dGs, dGt, rc_s, rc_t, loss, part


def _chunk_sizes(S):
    return sorted({1, 4, 7, max(1, S // 3 + 1), S} & set(range(1, S + 1)))


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("S", PAIR_S)
def test_pair_chunk_equals_the_two_one_sided_passes_bitwise(S, kernel):
    Gs, Gt, ns, nt = _grams(S, 24, kernel, seed=S + 11 * kernel)
    dGs, dGt, rc_s, rc_t, loss, part = _two_calls(Gs, Gt, ns, nt, S, kernel)
    raw = kernel >= 2
    ld = _ceil4(S) + 4                                       # padding columns S..ld-1 come out zero
    for R in _chunk_sizes(S):
        out_s, out_t = _nan(S, ld), _nan(S, ld)
        c_rs, c_rt, c_part = (_nan(S), _nan(S), _nan(S))
        for r0 in range(0, S, R):
            r = min(R, S - r0)
            cs, ct = _nan(r, ld), _nan(r, ld)
            cs[:, :S].copy_(Gs[r0:r0 + r])
            ct[:, :S].copy_(Gt[r0:r0 + r])
            before = c_part.clone()
            assert _L().b200gnn_gsp_pair_chunk_f32(cs.data_ptr(), ct.data_ptr(), ld, r, S, r0, _p(ns if raw else None),
                                                   _p(nt if raw else None), kernel, _p(c_rs if raw else None),
                                                   _p(c_rt if raw else None), c_part.data_ptr(), _st()) == OK
            # partials of other rows are left alone: stored at the global row only
            outside = torch.ones(S, dtype=torch.bool, device="cuda")
            outside[r0:r0 + r] = False
            assert torch.equal(c_part[outside].isnan(), before[outside].isnan())
            out_s[r0:r0 + r], out_t[r0:r0 + r] = cs, ct
        assert torch.equal(out_s[:, :S], dGs), R
        assert torch.equal(out_t[:, :S], dGt), R
        assert not out_s[:, S:].any() and not out_t[:, S:].any(), R
        assert torch.equal(c_part, part), R
        if raw:
            assert torch.equal(c_rs, rc_s) and torch.equal(c_rt, rc_t), R
        else:
            assert c_rs.isnan().all() and c_rt.isnan().all()
        got = _nan(1)
        assert _L().b200gnn_gsp_finish_f32(c_part.data_ptr(), S, got.data_ptr(), _st()) == OK
        assert torch.equal(got, loss), R                    # the loss bits do not depend on the chunk size


def test_pair_chunk_refusals():
    S, ld = 8, 8
    G, part, v = torch.zeros(S, ld, device="cuda"), torch.zeros(S, device="cuda"), torch.zeros(S, device="cuda")

    def call(**kw):
        a = {**dict(Gs=G.data_ptr(), Gt=G.data_ptr(), ld=ld, n=4, S=S, r0=0, ns=v.data_ptr(), nt=v.data_ptr(), k=3,
                    rs=v.data_ptr(), rt=v.data_ptr(), part=part.data_ptr()), **kw}
        return _L().b200gnn_gsp_pair_chunk_f32(a["Gs"], a["Gt"], a["ld"], a["n"], a["S"], a["r0"], a["ns"], a["nt"], a["k"],
                                               a["rs"], a["rt"], a["part"], _st())
    torch.cuda.synchronize()
    assert call() == OK
    for kw in (dict(Gs=None), dict(Gt=None), dict(part=None), dict(S=0), dict(ld=S - 1), dict(n=0), dict(r0=-1),
               dict(r0=5), dict(k=-1), dict(k=4), dict(ns=None), dict(nt=None), dict(rs=None), dict(rt=None), dict(S=1 << 31)):
        _refused(lambda: call(**kw))
    assert call(k=0, ns=None, nt=None, rs=None, rt=None) == OK      # cosine / poly read no norms
    _refused(lambda: _L().b200gnn_gsp_finish_f32(None, S, part.data_ptr(), _st()))
    _refused(lambda: _L().b200gnn_gsp_finish_f32(part.data_ptr(), 0, part.data_ptr(), _st()))


# ============================================================================================ 2. operands and backward
def _designed_heads(n, P, g):
    """pre [n, P] and bn [4, P] whose rows exercise the kernels' branches: row 0 all cut by the ReLU (zero row), row 1 with
    norm inside (0, eps), row 2 half of the columns cut, the rest random."""
    pre = torch.randn(n, P, generator=g)
    mean, invstd = torch.randn(P, generator=g) * 0.1, torch.rand(P, generator=g) + 0.5
    scale = torch.rand(P, generator=g) + 0.5
    shift = torch.zeros(P)                                     # so that the designed rows below land where intended
    pre[0] = -1.0                                              # fma(y, scale, shift) < 0 everywhere
    pre[1] = 1e-14                                             # relu(bn) ~ 1e-14: norm below eps = 1e-12
    half = torch.arange(P) % 2 == 0
    pre[2] = torch.where(half, torch.ones(P), -torch.ones(P))
    bn = torch.stack([mean, invstd, scale, shift])
    return pre.cuda(), bn.cuda()


def _act64(pre, bn):
    y, s, h = pre.double().cpu(), bn[2].double().cpu(), bn[3].double().cpu()
    return torch.relu(y * s + h)


def _operands(inds, S, P, kernel, pre_s, bn_s, pre_t, bn_t, Sp_extra=4):
    x_s, x_t = _nan(S + Sp_extra, P), _nan(S + Sp_extra, P)
    n_s, n_t = _nan(S + Sp_extra), _nan(S + Sp_extra)
    assert _L().b200gnn_gsp_operands_f32(inds.data_ptr(), S, P, kernel, pre_s.data_ptr(), bn_s.data_ptr(), pre_t.data_ptr(),
                                         bn_t.data_ptr(), 1e-12, x_s.data_ptr(), x_t.data_ptr(), n_s.data_ptr(),
                                         n_t.data_ptr(), _st()) == OK
    return x_s, x_t, n_s, n_t


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("P", [4, 64, 132, 256])
def test_operands_within_fp64_bounds(kernel, P):
    g = torch.Generator().manual_seed(P + kernel)
    n, S = 40, 24
    pre_s, bn_s = _designed_heads(n, P, g)
    pre_t, bn_t = _designed_heads(n, P, g)
    inds = torch.cat([torch.tensor([0, 1, 2]), torch.randperm(n - 3, generator=g)[:S - 3] + 3]).to(torch.int32).cuda()
    x_s, x_t, n_s, n_t = _operands(inds, S, P, kernel, pre_s, bn_s, pre_t, bn_t)
    for x, nrm, pre, bn in ((x_s, n_s, pre_s, bn_s), (x_t, n_t, pre_t, bn_t)):
        a = _act64(pre, bn)[inds.long().cpu()]
        sq = a.pow(2).sum(1)
        assert x[S:].isnan().all() and nrm[S:].isnan().all()            # canaries past the sample
        assert torch.equal((x[:S] > 0).cpu(), (a > 0))                  # the ReLU mask, exactly
        if kernel >= 2:
            # raw: x = relu(fma(y, s, h)), one rounding (plus the fp64 product's); squared norm an fp32 fma chain
            assert ((x[:S].double().cpu() - a).abs() <= 2 * U * a.abs() + 1e-45).all()
            assert ((nrm[:S].double().cpu() - sq).abs() <= (P + 2) * U * sq * 1.01 + 1e-45).all()
        else:
            nr = sq.sqrt()
            ref = a / nr.clamp_min(1e-12)[:, None]
            bound = (P // 2 + 6) * U * ref.abs() + 1e-45
            assert ((x[:S].double().cpu() - ref).abs() <= bound).all()
            assert ((nrm[:S].double().cpu() - nr).abs() <= (P // 2 + 4) * U * nr + 1e-45).all()
            assert float(nrm[0]) == 0 and not x[0].any()                                   # the zero row
            assert 0 < float(nrm[1]) < 1e-12 and float(x[1].abs().max()) > 0               # through the eps clamp


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("P", [64, 256])
def test_backward_within_fp64_bounds(kernel, P):
    g = torch.Generator().manual_seed(100 + P + kernel)
    n, S, beta = 50, 30, float(np.float32(0.7))
    pre_s, bn_s = _designed_heads(n, P, g)
    pre_t, bn_t = _designed_heads(n, P, g)
    inds = torch.cat([torch.tensor([0, 1, 2]), torch.randperm(n - 3, generator=g)[:S - 3] + 3]).to(torch.int32).cuda()
    x_s, x_t, n_s, n_t = _operands(inds, S, P, kernel, pre_s, bn_s, pre_t, bn_t)
    g_s, g_t = torch.randn(S, P, generator=g).cuda(), torch.randn(S, P, generator=g).cuda()
    rc_s, rc_t = torch.randn(S, generator=g).cuda(), torch.randn(S, generator=g).cuda()
    dz_s, dz_t = _nan(n, P), _nan(n, P)
    slots = int(_L().b200gnn_gcrd_bwd_slots())
    part_s, part_t = _nan(slots, 2, P), _nan(slots, 2, P)
    loss_aux, total = torch.tensor([0.25], device="cuda"), torch.tensor([1.5], device="cuda")
    assert _L().b200gnn_gsp_backward_f32(inds.data_ptr(), S, P, kernel, g_s.data_ptr(), g_t.data_ptr(), x_s.data_ptr(),
                                         x_t.data_ptr(), n_s.data_ptr(), n_t.data_ptr(), rc_s.data_ptr(), rc_t.data_ptr(), 1e-12,
                                         pre_s.data_ptr(), bn_s.data_ptr(), pre_t.data_ptr(), bn_t.data_ptr(), beta,
                                         dz_s.data_ptr(), dz_t.data_ptr(), part_s.data_ptr(), part_t.data_ptr(),
                                         loss_aux.data_ptr(), total.data_ptr(), _st()) == OK
    assert abs(float(total) - (1.5 + np.float32(beta) * np.float32(0.25))) <= 2 * U * 1.7
    il = inds.long().cpu()
    rows_out = torch.ones(n, dtype=torch.bool)
    rows_out[il] = False
    for x, nrm, gg, rc, pre, bn, dz, part in ((x_s, n_s, g_s, rc_s, pre_s, bn_s, dz_s, part_s),
                                              (x_t, n_t, g_t, rc_t, pre_t, bn_t, dz_t, part_t)):
        xd, gd = x[:S].double().cpu(), gg.double().cpu()
        mask = _act64(pre, bn)[il] > 0
        if kernel >= 2:
            # operand gradient 2 g + 4 rc x (the raw path has no normalise step)
            v = 2 * gd + 4 * rc.double().cpu()[:, None] * xd
            mag = 2 * gd.abs() + 4 * rc.double().cpu().abs()[:, None] * xd.abs()
            bound = 3 * U * mag
        else:
            nr = nrm[:S].double().cpu()
            inv = 1.0 / nr.clamp_min(1e-12)
            g2 = 2 * gd
            dot = (xd * g2).sum(1, keepdim=True)
            clamped = (nr < 1e-12)[:, None]
            v = torch.where(clamped, g2 * inv[:, None], inv[:, None] * (g2 - xd * dot))
            mag = inv[:, None] * (g2.abs() + xd.abs() * (xd.abs() * g2.abs()).sum(1, keepdim=True))
            bound = (P // 2 + 8) * U * mag
        ref = torch.where(mask, v * beta, torch.zeros_like(v))
        got = dz.double().cpu()[il]
        assert ((got - ref).abs() <= bound * beta + 1e-45).all(), float(((got - ref).abs() / (bound * beta + 1e-300)).max())
        assert (got[~mask] == 0).all()                                  # the ReLU mask, exactly
        assert dz[rows_out.cuda()].isnan().all()                        # rows outside the sample keep their canaries
        # pass 1 of the BatchNorm backward: the slots' column sums of dz and dz * xhat
        xhat = (pre.double()[il].cpu() - bn[0].double().cpu()) * bn[1].double().cpu()
        s1, s2 = part[:, 0].double().sum(0).cpu(), part[:, 1].double().sum(0).cpu()
        r1, r2 = got.sum(0), (got * xhat).sum(0)
        assert ((s1 - r1).abs() <= (S + 2) * U * got.abs().sum(0) + 1e-30).all()
        assert ((s2 - r2).abs() <= (S + 4) * U * (got * xhat).abs().sum(0) + 1e-30).all()


def test_operands_and_backward_refusals():
    n, S, P = 8, 4, 64
    inds = torch.arange(S, dtype=torch.int32, device="cuda")
    b = lambda *s: torch.zeros(*s, device="cuda")
    pre, bn, x, nrm, dz = b(n, P), b(4, P), b(S, P), b(S), b(n, P)
    part = b(int(_L().b200gnn_gcrd_bwd_slots()), 2, P)

    def ops_call(**kw):
        a = {**dict(inds=inds.data_ptr(), S=S, P=P, k=0, pre=pre.data_ptr(), bn=bn.data_ptr(), x=x.data_ptr(),
                    nrm=nrm.data_ptr(), eps=1e-12), **kw}
        return _L().b200gnn_gsp_operands_f32(a["inds"], a["S"], a["P"], a["k"], a["pre"], a["bn"], a["pre"], a["bn"], a["eps"],
                                             a["x"], a["x"], a["nrm"], a["nrm"], _st())

    def bwd_call(**kw):
        a = {**dict(inds=inds.data_ptr(), S=S, P=P, k=0, g=x.data_ptr(), x=x.data_ptr(), nrm=nrm.data_ptr(), rc=nrm.data_ptr(),
                    pre=pre.data_ptr(), bn=bn.data_ptr(), dz=dz.data_ptr(), part=part.data_ptr(), eps=1e-12, la=None,
                    lt=None), **kw}
        return _L().b200gnn_gsp_backward_f32(a["inds"], a["S"], a["P"], a["k"], a["g"], a["g"], a["x"], a["x"], a["nrm"], a["nrm"],
                                             a["rc"], a["rc"], a["eps"], a["pre"], a["bn"], a["pre"], a["bn"], 0.5, a["dz"],
                                             a["dz"], a["part"], a["part"], a["la"], a["lt"], _st())
    torch.cuda.synchronize()
    assert ops_call() == OK and bwd_call() == OK
    for kw in (dict(inds=None), dict(S=0), dict(P=0), dict(P=6), dict(P=260), dict(k=-1), dict(k=4), dict(pre=None),
               dict(bn=None), dict(x=None), dict(nrm=None), dict(eps=0.0), dict(x=x.data_ptr() + 4)):
        _refused(lambda: ops_call(**kw))
    for kw in (dict(inds=None), dict(S=0), dict(P=6), dict(P=260), dict(k=5), dict(g=None), dict(x=None), dict(pre=None),
               dict(dz=None), dict(part=None), dict(nrm=None), dict(k=2, rc=None), dict(eps=-1.0), dict(lt=nrm.data_ptr()),
               dict(dz=dz.data_ptr() + 4)):
        _refused(lambda: bwd_call(**kw))
    assert bwd_call(k=3, nrm=None) == OK and bwd_call(k=1, rc=None) == OK      # each path reads only what it needs


# ============================================================================================ 3. the chunk loop
def _unchunked(xs, xt, S, kernel):
    """The sequence criterion._GSP ran before the chunk loop, rebuilt from public entry points: full S x S Gram GEMMs, the
    two one-sided pair passes, the backward GEMM dG . x over the zero-padded contraction."""
    Sp = _ceil4(S)
    pad = lambda t: torch.nn.functional.pad(t, (0, _ceil4(t.shape[1]) - t.shape[1], 0, Sp - S)).contiguous()
    xs_p, xt_p = pad(xs), pad(xt)
    raw = kernel >= 2
    ns = nt = None
    if raw:
        ns, nt = _nan(S), _nan(S)
        lib.check(_L().b200gnn_row_sqnorm_f32(xs.data_ptr(), S, xs.shape[1], ns.data_ptr(), _st()), "sq")
        lib.check(_L().b200gnn_row_sqnorm_f32(xt.data_ptr(), S, xt.shape[1], nt.data_ptr(), _st()), "sq")
    G = []
    for x in (xs_p, xt_p):
        hi, lo = ops.split_tf32(x[:S])
        G.append(ops.gemm_tf32x3(x[:S], hi, lo))
    dGs, dGt, rc_s, rc_t, loss, _ = _two_calls(G[0], G[1], ns, nt, S, kernel)
    out = []
    for dG, x, F_ in ((dGs, xs_p, xs.shape[1]), (dGt, xt_p, xt.shape[1])):
        hi, lo = ops.split_tf32(x[:, :F_].contiguous(), transpose=True)    # [F, Sp]
        A = torch.nn.functional.pad(dG, (0, Sp - S)).contiguous()
        out.append(ops.gemm_tf32x3(A, hi, lo))
    return ns, nt, out[0], out[1], rc_s, rc_t, loss


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("S,F,F_t,R", [(1, 8, 8, None), (7, 64, 90, None), (600, 64, 64, 128), (600, 90, 750, 124),
                                       (5000, 128, 128, None)])
def test_gsp_chunks_equals_the_unchunked_sequence(kernel, S, F, F_t, R):
    g = torch.Generator().manual_seed(S + F + kernel)
    xs, xt = torch.randn(S, F, generator=g).cuda(), torch.randn(S, F_t, generator=g).cuda()
    if kernel <= 1:
        xs, xt = torch.nn.functional.normalize(xs, dim=1), torch.nn.functional.normalize(xt, dim=1)
    else:
        xs, xt = xs * 0.3, xt * 0.3
    ns, nt, ref_s, ref_t, rc_s, rc_t, loss = _unchunked(xs, xt, S, kernel)
    Sp, Fp, Fp_t = _ceil4(S), _ceil4(F), _ceil4(F_t)
    b = C.GspBuffers(Sp, Fp, xs.device, Fp_t)
    if R is not None:                                    # smaller chunks than the L2 budget gives, ending in a partial one
        b.Gs, b.Gt = b.Gs[:R], b.Gt[:R]
    for t in (b.g_s, b.g_t, b.rc_s, b.rc_t, b.part):
        t.fill_(float("nan"))
    if kernel >= 2:
        b.ns[:S].copy_(ns)
        b.nt[:S].copy_(nt)
    pad = lambda t: torch.nn.functional.pad(t, (0, _ceil4(t.shape[1]) - t.shape[1], 0, Sp - S)).contiguous()
    C.gsp_chunks(pad(xs), pad(xt), S, kernel, b)
    assert torch.equal(b.loss, loss)
    assert torch.equal(b.g_s[:S, :F], ref_s[:S]) and torch.equal(b.g_t[:S, :F_t], ref_t[:S])
    assert not b.g_s[:S, F:].any() and not b.g_t[:S, F_t:].any()
    if kernel >= 2:
        assert torch.equal(b.rc_s[:S], rc_s) and torch.equal(b.rc_t[:S], rc_t)


def test_gsp_chunk_rows_share_the_nce_budget():
    for Sp in (4, 128, 4096, 8192, 16384, 65536):
        R = C.gsp_chunk_rows(Sp)
        assert R == Sp or (R % 128 == 0 and (2 * R * Sp * 4 <= C.NCE_CHUNK_BYTES or R == 128))


def test_gsp_chunks_peak_memory_is_far_below_the_square():
    S, F = 8192, 256
    g = torch.Generator().manual_seed(0)
    xs = torch.nn.functional.normalize(torch.randn(S, F, generator=g), dim=1).cuda()
    xt = torch.nn.functional.normalize(torch.randn(S, F, generator=g), dim=1).cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    b = C.GspBuffers(S, F, xs.device)
    C.gsp_chunks(xs, xt, S, 0, b)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 0.6 * S * S * 4, peak
    assert torch.isfinite(b.loss).all()
