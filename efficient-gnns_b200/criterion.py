"""Drop-in for the reference's ``criterion.py`` (arxiv_pyg/criterion.py:8-149 and the identical mag_pyg/ copy; the PPI
variant with binary cross-entropy is ``criterion_ppi.py``).

Same function names, argument order and return convention ``(loss, loss_cls, loss_aux)``; every loss is computed
by b200gnn kernels (fused row losses, edge-list passes, wgmma 3xTF32 GEMMs for the S x S contractions) and is
differentiable through small ``torch.autograd.Function`` wrappers.  ``from efficient_gnns_b200.criterion import *``
in place of ``from criterion import *`` is the whole integration (INTEGRATION.md).

Sampling (``max_samples``) draws from numpy's global RNG exactly like the reference (criterion.py:63,135) so that a
seeded run selects the same rows; ``sampled_inds=`` lets tests inject the draw.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import lib, ops

__all__ = ["kd_criterion", "fitnet_criterion", "at_criterion", "gpw_criterion", "lpw_criterion", "nce_criterion"]

_KERNELS = {"cosine": 0, "poly": 1, "l2": 2, "rbf": 3}
_NORM_EPS = 1e-12  # F.normalize default


def _L():
    return lib.load()


def _f32(t, name):
    return lib.dptr(t, torch.float32, name)


def _new(*shape, like):
    return torch.empty(*shape, dtype=torch.float32, device=like.device)


# ----------------------------------------------------------------------------------------- CE / logit KD
class _RowLoss(torch.autograd.Function):
    """CE (teacher None) or the fused Hinton KD loss over all rows of logits [n,C]; grad w.r.t. logits only."""

    @staticmethod
    def forward(ctx, logits, labels, teacher, alpha, T):
        logits = logits.contiguous()
        out, d_logits = ops.kd_loss_fwd_bwd(logits, labels.contiguous(), None,
                                            None if teacher is None else teacher.contiguous(), alpha, T)
        ctx.save_for_backward(d_logits)
        ctx.mark_non_differentiable(out)
        return out[0].clone(), out

    @staticmethod
    def backward(ctx, g_loss, _g_all):
        (d_logits,) = ctx.saved_tensors
        return d_logits * g_loss, None, None, None, None


def cross_entropy(logits, labels):
    return _RowLoss.apply(logits, labels, None, 0.0, 1.0)[0]


class _BCE(torch.autograd.Function):
    """F.binary_cross_entropy_with_logits(z, target) (mean over all elements); target_is_logits => sigmoid(target)."""

    @staticmethod
    def forward(ctx, z, target, target_is_logits: bool):
        z, target = z.contiguous(), target.contiguous().to(torch.float32)
        n = z.numel()
        loss, d_z = _new(1, like=z), torch.empty_like(z)
        part = _new(int(_L().b200gnn_reduce_slots(n)), like=z)
        lib.check(_L().b200gnn_bce_logits_fwd_bwd_f32(_f32(z, "z"), _f32(target, "target"), int(target_is_logits), n, 1.0,
                                                     _f32(d_z, "d_z"), _f32(loss, "loss"), _f32(part, "partial"),
                                                     lib.stream_ptr()), "bce_logits_fwd_bwd_f32")
        ctx.save_for_backward(d_z)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        (d_z,) = ctx.saved_tensors
        return d_z * g, None, None


def bce_with_logits(logits, labels):
    """ppi_pyg/criterion.py:11 — multi-label classification loss of the PPI student."""
    return _BCE.apply(logits, labels, False)


def kd_criterion(logits, labels, teacher_logits, alpha=0.9, T=4):
    """criterion.py:8-21."""
    loss, parts = _RowLoss.apply(logits, labels, teacher_logits, float(alpha), float(T))
    return loss, parts[1], parts[2]


# ----------------------------------------------------------------------------------------- row helpers
def _normalize(x, scale: float = 1.0):
    n, F = x.shape
    out, norm = torch.empty_like(x), _new(n, like=x)
    lib.check(_L().b200gnn_row_normalize_fwd_f32(_f32(x, "x"), n, F, _NORM_EPS, scale, _f32(out, "out"), _f32(norm, "norm"),
                                                lib.stream_ptr()), "row_normalize_fwd_f32")
    return out, norm


def _normalize_bwd(out, norm, d_out, scale: float = 1.0):
    n, F = out.shape
    d_x = torch.empty_like(out)
    lib.check(_L().b200gnn_row_normalize_bwd_f32(_f32(out, "out"), _f32(norm, "norm"), _f32(d_out.contiguous(), "d_out"), n, F,
                                                _NORM_EPS, scale, _f32(d_x, "d_x"), 0, lib.stream_ptr()),
              "row_normalize_bwd_f32")
    return d_x


def _mse(a, b, want_grad: bool = True):
    """(loss[1], d_a) with d_a = d mse / d a."""
    n = a.numel()
    loss = _new(1, like=a)
    d_a = torch.empty_like(a) if want_grad else None
    part = _new(int(_L().b200gnn_reduce_slots(n)), like=a)
    lib.check(_L().b200gnn_mse_fwd_bwd_f32(_f32(a, "a"), _f32(b, "b"), n, 1.0, _f32(d_a, "d_a"), _f32(loss, "loss"),
                                          _f32(part, "partial"), lib.stream_ptr()), "mse_fwd_bwd_f32")
    return loss, d_a


def _pad_k(t, dim: int):
    """Zero-pad the contraction dimension to a multiple of 4 floats (TMA needs 16-byte row pitches); exact."""
    k = t.shape[dim]
    if k % 4 == 0:
        return t.contiguous()
    pad = 4 - k % 4
    return torch.nn.functional.pad(t, (0, pad) if dim == 1 else (0, 0, 0, pad)).contiguous()


def _gemm_nt(a, b):
    """a[M,K] @ b[N,K]^T on the tensor cores with fp32 fidelity."""
    hi, lo = ops.split_tf32(_pad_k(b, 1))
    return ops.gemm_tf32x3(_pad_k(a, 1), hi, lo)


def _gemm_nn(a, b):
    """a[M,K] @ b[K,N]."""
    hi, lo = ops.split_tf32(_pad_k(b, 0), transpose=True)
    return ops.gemm_tf32x3(_pad_k(a, 1), hi, lo)


def _sample(n: int, max_samples: int, device, sampled_inds=None):
    if max_samples >= n:
        return None
    if sampled_inds is None:
        sampled_inds = np.random.choice(n, max_samples, replace=False)      # reference: criterion.py:63,135
    return torch.as_tensor(sampled_inds, dtype=torch.long, device=device)


# ----------------------------------------------------------------------------------------- FitNet / AT
class _NormalizedMSE(torch.autograd.Function):
    """mse(normalize(a), normalize(b)) — fitnet_criterion's auxiliary term (criterion.py:30-33)."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        an, na = _normalize(a)
        bn, nb = _normalize(b)
        loss, d_an = _mse(an, bn)
        ctx.save_for_backward(an, na, bn, nb, d_an)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        an, na, bn, nb, d_an = ctx.saved_tensors
        da = _normalize_bwd(an, na, d_an) * g if ctx.needs_input_grad[0] else None
        db = _normalize_bwd(bn, nb, -d_an) * g if ctx.needs_input_grad[1] else None
        return da, db


def fitnet_criterion(logits, labels, feat, teacher_feat, beta=1000, _cls=None):
    """criterion.py:24-36."""
    loss_cls = (_cls or cross_entropy)(logits, labels)
    loss_aux = _NormalizedMSE.apply(feat, teacher_feat)
    return loss_cls + beta * loss_aux, loss_cls, loss_aux


class _AttentionMSE(torch.autograd.Function):
    """mse(normalize(||f_i||^2 over nodes), normalize(||t_i||^2 over nodes)) — at_criterion (criterion.py:44-50)."""

    @staticmethod
    def forward(ctx, a, b):
        a, b = a.contiguous(), b.contiguous()
        L, st = _L(), lib.stream_ptr()
        n = a.shape[0]
        sa, sb = _new(n, like=a), _new(n, like=a)
        lib.check(L.b200gnn_row_sqnorm_f32(_f32(a, "a"), n, a.shape[1], _f32(sa, "sa"), st), "row_sqnorm_f32")
        lib.check(L.b200gnn_row_sqnorm_f32(_f32(b, "b"), n, b.shape[1], _f32(sb, "sb"), st), "row_sqnorm_f32")
        san, na = _normalize(sa.view(1, n))
        sbn, nb = _normalize(sb.view(1, n))
        loss, d_san = _mse(san, sbn)
        ctx.save_for_backward(a, b, san, na, sbn, nb, d_san)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        a, b, san, na, sbn, nb, d_san = ctx.saved_tensors
        L, st = _L(), lib.stream_ptr()
        out = []
        for x, xn, nx, sign, need in ((a, san, na, 1.0, ctx.needs_input_grad[0]), (b, sbn, nb, -1.0, ctx.needs_input_grad[1])):
            if not need:
                out.append(None)
                continue
            d_s = _normalize_bwd(xn, nx, d_san * sign).view(-1)
            d_x = torch.empty_like(x)
            lib.check(L.b200gnn_row_sqnorm_bwd_f32(_f32(x, "x"), _f32(d_s, "d_s"), x.shape[0], x.shape[1], _f32(d_x, "d_x"), st),
                      "row_sqnorm_bwd_f32")
            out.append(d_x * g)
        return tuple(out)


def at_criterion(logits, labels, feat, teacher_feat, beta=1000, _cls=None):
    """criterion.py:39-54."""
    loss_cls = (_cls or cross_entropy)(logits, labels)
    loss_aux = _AttentionMSE.apply(feat, teacher_feat)
    return loss_cls + beta * loss_aux, loss_cls, loss_aux


# ----------------------------------------------------------------------------------------- GSP
# Rows R of the two [R, Sp] Gram chunks of one GSP pass: together they take the InfoNCE chunk's budget (NCE_CHUNK_BYTES),
# so the loss never holds the four S x S matrices (Grams and their gradients) the direct form needs: 1 GiB at S = 8192.
def gsp_chunk_rows(Sp: int) -> int:
    """Rows R of one pair of [R, Sp] Gram chunks (2 * R * Sp * 4 <= NCE_CHUNK_BYTES, a multiple of 128, at most Sp)."""
    return min(max(128, (NCE_CHUNK_BYTES // (8 * Sp)) // 128 * 128), Sp)


class GspBuffers:
    """Every buffer of one GSP forward + gradient over [Sp, Fp] student and [Sp, Fp_t] teacher operands (Fp_t = Fp unless
    given: each side only meets itself), allocated once so that a captured step (gsp.py) reuses them on every replay.
    ns / nt [Sp]: the operands' squared row norms, filled by the caller for l2 / rbf.  g_s [Sp, Fp] / g_t [Sp, Fp_t]: dG . x
    per side (rows < S), the operand gradient before the factor 2 and the norm terms."""

    def __init__(self, Sp: int, Fp: int, device, Fp_t: Optional[int] = None):
        R = gsp_chunk_rows(Sp)
        Ft = Fp if Fp_t is None else Fp_t
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=device)
        self.Gs, self.Gt = e(R, Sp), e(R, Sp)
        self.xs_split, self.xt_split = (e(Sp, Fp), e(Sp, Fp)), (e(Sp, Ft), e(Sp, Ft))          # B of G_c = x_c . x^T
        self.xsT_split, self.xtT_split = (e(Fp, Sp), e(Fp, Sp)), (e(Ft, Sp), e(Ft, Sp))      # B of g_c = dG_c . x
        self.ns, self.nt, self.rc_s, self.rc_t, self.part = e(Sp), e(Sp), e(Sp), e(Sp), e(Sp)
        self.loss = e(1)
        self.g_s, self.g_t = e(Sp, Fp), e(Sp, Ft)


def gsp_chunks(x_s: torch.Tensor, x_t: torch.Tensor, S: int, kernel: int, b: GspBuffers) -> None:
    """The GSP loss over zero-padded operands x_s [Sp, Fp], x_t [Sp, Fp_t] (S real rows; normalised for cosine / poly, raw for l2 / rbf
    with b.ns / b.nt holding their squared norms) in row chunks: per chunk the two Gram GEMMs x_c . x^T, the pair pass
    (both gradients in place, the padding columns zeroed), then g[c] = dG_c . x per side.  dG is symmetric, so d x = 2 dG x
    needs only the chunk's own rows.  b.loss = mse(sim_s, sim_t); b.rc_s / b.rc_t the l2 / rbf row coefficients.  Only
    launches on preallocated buffers, so it can be captured."""
    L, st = _L(), lib.stream_ptr()
    Sp = x_s.shape[0]
    R = b.Gs.shape[0]
    sides = ((x_s, b.xs_split, b.xsT_split, b.Gs, b.g_s), (x_t, b.xt_split, b.xtT_split, b.Gt, b.g_t))
    for x, sp, spT, _, _ in sides:
        ops.split_tf32(x, hi=sp[0], lo=sp[1])
        ops.split_tf32(x, transpose=True, hi=spT[0], lo=spT[1])
    raw = kernel >= 2
    for r0 in range(0, S, R):
        r = min(R, S - r0)
        for x, sp, _, G, _ in sides:
            ops.gemm_tf32x3(x[r0:r0 + r], sp[0], sp[1], out=G[:r])
        lib.check(L.b200gnn_gsp_pair_chunk_f32(_f32(b.Gs, "Gs"), _f32(b.Gt, "Gt"), Sp, r, S, r0, _f32(b.ns if raw else None, "ns"),
                                               _f32(b.nt if raw else None, "nt"), kernel, _f32(b.rc_s if raw else None, "rc_s"),
                                               _f32(b.rc_t if raw else None, "rc_t"), _f32(b.part, "part"), st),
                  "gsp_pair_chunk_f32")
        for _, _, spT, G, g in sides:
            ops.gemm_tf32x3(G[:r], spT[0], spT[1], out=g[r0:r0 + r])
    lib.check(L.b200gnn_gsp_finish_f32(_f32(b.part, "part"), S, _f32(b.loss, "loss"), st), "gsp_finish_f32")


class _GSP(torch.autograd.Function):
    """mse(pairwise_k(fs), pairwise_k(ft)) over an S-row sample (criterion.py:66-86) by gsp_chunks: the S x S Gram
    matrices exist only as L2-sized row chunks, and both gradients are complete when the forward returns."""

    @staticmethod
    def forward(ctx, fs, ft, kernel: int):
        fs, ft = fs.contiguous(), ft.contiguous()
        L, st = _L(), lib.stream_ptr()
        S, F_, F_t = fs.shape[0], fs.shape[1], ft.shape[1]
        if kernel <= 1:
            xs, ns = _normalize(fs)
            xt, nt = _normalize(ft)
        else:
            xs, xt, ns, nt = fs, ft, None, None
        xs_p, xt_p = _pad_k(_pad_k(xs, 1), 0), _pad_k(_pad_k(xt, 1), 0)
        b = GspBuffers(xs_p.shape[0], xs_p.shape[1], fs.device, xt_p.shape[1])
        if kernel >= 2:
            lib.check(L.b200gnn_row_sqnorm_f32(_f32(xs, "xs"), S, F_, _f32(b.ns, "sq"), st), "row_sqnorm_f32")
            lib.check(L.b200gnn_row_sqnorm_f32(_f32(xt, "xt"), S, F_t, _f32(b.nt, "sq"), st), "row_sqnorm_f32")
        gsp_chunks(xs_p, xt_p, S, kernel, b)
        ctx.kernel = kernel
        ctx.save_for_backward(xs, xt, ns if ns is not None else xs, nt if nt is not None else xt, b.g_s[:S, :F_], b.g_t[:S, :F_t],
                              b.rc_s[:S], b.rc_t[:S])
        return b.loss[0]

    @staticmethod
    def backward(ctx, g):
        xs, xt, ns, nt, g_s, g_t, rc_s, rc_t = ctx.saved_tensors
        L, st = _L(), lib.stream_ptr()
        out = []
        for x, nrm, dGx, rc, need in ((xs, ns, g_s, rc_s, ctx.needs_input_grad[0]), (xt, nt, g_t, rc_t, ctx.needs_input_grad[1])):
            if not need:
                out.append(None)
                continue
            d = (dGx * 2.0).contiguous()            # d x = 2 dG x (+ norm terms)
            if ctx.kernel >= 2:
                lib.check(L.b200gnn_row_axpy_f32(_f32(x, "x"), _f32(rc, "rc"), x.shape[0], x.shape[1], 4.0, _f32(d, "d"), st),
                          "row_axpy_f32")
            else:
                d = _normalize_bwd(x, nrm, d)
            out.append(d * g)
        return out[0], out[1], None


def gpw_criterion(logits, labels, feat, teacher_feat, kernel='cosine', beta=1, max_samples=8192, sampled_inds=None, _cls=None):
    """criterion.py:57-92."""
    if kernel not in _KERNELS:
        raise NotImplementedError
    loss_cls = (_cls or cross_entropy)(logits, labels)
    inds = _sample(feat.shape[0], max_samples, feat.device, sampled_inds)
    if inds is not None:
        feat, teacher_feat = feat[inds], teacher_feat[inds]
    loss_aux = _GSP.apply(feat, teacher_feat, _KERNELS[kernel])
    return loss_cls + beta * loss_aux, loss_cls, loss_aux


# ----------------------------------------------------------------------------------------- LSP
class LspPlan:
    """Edge list sorted by destination (the PyG-softmax group index, criterion.py:100-104) — built once per edge_index."""
    _cache = {}

    def __init__(self, edge_index: torch.Tensor):
        src, dst = edge_index[0], edge_index[1]
        E = int(src.numel())
        if E and int(max(src.max(), dst.max())) >= 2 ** 31 - 1:
            raise lib.B200GnnError("edge_index exceeds the engine's int32 range")
        perm = torch.argsort(dst, stable=True)
        self.E = E
        self.src = src[perm].to(torch.int32).contiguous()
        self.dst = dst[perm].to(torch.int32).contiguous()
        self.n_seg = int(dst.max()) + 1 if E else 0          # PyG softmax: N = index.max() + 1
        counts = torch.bincount(dst, minlength=self.n_seg) if E else torch.zeros(0, dtype=torch.long, device=dst.device)
        rowptr = torch.zeros(self.n_seg + 1, dtype=torch.long, device=dst.device)
        torch.cumsum(counts, 0, out=rowptr[1:])
        self.rowptr = rowptr.to(torch.int32).contiguous()
        self.edge_index = edge_index          # keeps the keyed storage alive: its address cannot be recycled while cached
        self._bwd = {}

    def backward_matrix(self, n_nodes: int):
        """CSR structure of the backward matrix C (csrc/loss_edge.cu, b200gnn_lsp_bwd_values_f32) for `n_nodes` feature
        rows: (CsrGraph with an in-place updatable value array, pos_dst, pos_src, diag_pos, selfc scratch)."""
        hit = self._bwd.get(n_nodes)
        if hit is not None:
            return hit
        from .sparse import csr_graph_from
        dev, E = self.src.device, self.E
        src, dst = self.src.long(), self.dst.long()
        if E and int(max(src.max(), dst.max())) >= n_nodes:
            raise lib.B200GnnError("LSP: edge_index refers to a node beyond the feature matrix")
        ar = torch.arange(n_nodes, device=dev)
        rows = torch.cat([dst, src, ar])
        cols = torch.cat([src, dst, ar])
        perm = torch.argsort(rows, stable=True)
        inv = torch.empty_like(perm)
        inv[perm] = torch.arange(perm.numel(), device=dev)
        rowptr = torch.zeros(n_nodes + 1, dtype=torch.long, device=dev)
        torch.cumsum(torch.bincount(rows, minlength=n_nodes), 0, out=rowptr[1:])
        val = torch.zeros(perm.numel(), device=dev)
        G = csr_graph_from(rowptr, cols[perm], val, n_nodes, n_nodes)
        pos = inv.to(torch.int32)
        hit = (G, pos[:E].contiguous(), pos[E:2 * E].contiguous(), pos[2 * E:].contiguous(), torch.zeros_like(val))
        self._bwd[n_nodes] = hit
        return hit

    @classmethod
    def of(cls, edge_index: torch.Tensor) -> "LspPlan":
        key = (edge_index.data_ptr(), tuple(edge_index.shape), edge_index._version, str(edge_index.device))
        plan = cls._cache.get(key)
        if plan is not None and plan.edge_index.data_ptr() != edge_index.data_ptr():
            plan = None
        if plan is None:
            if len(cls._cache) > 8:
                cls._cache.clear()
            plan = cls._cache[key] = cls(edge_index)
        return plan


class _LSP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, teacher_feat, plan: LspPlan, kernel: int, criterion: int):
        feat, teacher_feat = feat.contiguous(), teacher_feat.contiguous()
        L, st = _L(), lib.stream_ptr()
        E = plan.E
        sim_s, sim_t, g = _new(E, like=feat), _new(E, like=feat), _new(E, like=feat)
        for f, sim in ((feat, sim_s), (teacher_feat, sim_t)):
            lib.check(L.b200gnn_edge_sim_f32(_f32(f, "feat"), f.shape[1], plan.src.data_ptr(), plan.dst.data_ptr(), E, kernel,
                                             _f32(sim, "sim"), st), "edge_sim_f32")
        loss = _new(1, like=feat)
        part = _new(int(L.b200gnn_lsp_partials(plan.n_seg)), like=feat)
        lib.check(L.b200gnn_lsp_segment_f32(_f32(sim_s, "sim_s"), _f32(sim_t, "sim_t"), plan.rowptr.data_ptr(), plan.n_seg, E,
                                            criterion, _f32(g, "g"), _f32(loss, "loss"), _f32(part, "part"), st),
                  "lsp_segment_f32")
        ctx.plan, ctx.kernel = plan, kernel
        ctx.save_for_backward(feat, sim_s, g)
        return loss[0]

    @staticmethod
    def backward(ctx, gout):
        feat, sim_s, g = ctx.saved_tensors
        plan = ctx.plan
        n, F_ = feat.shape
        G, pos_dst, pos_src, diag_pos, selfc = plan.backward_matrix(n)
        lib.check(_L().b200gnn_lsp_bwd_values_f32(_f32(feat, "feat"), F_, plan.src.data_ptr(), plan.dst.data_ptr(), plan.E,
                                                  ctx.kernel, _f32(sim_s, "sim"), _f32(g, "g"), pos_dst.data_ptr(),
                                                  pos_src.data_ptr(), G.rowptr.data_ptr(), diag_pos.data_ptr(), n,
                                                  _f32(G.val, "val"), _f32(selfc, "selfc"), lib.stream_ptr()),
                  "lsp_bwd_values_f32")
        from . import ops
        d = ops.spmm_csr(G, feat, "sum")             # d feat = C · feat: fixed summation order, no atomics
        return d * gout, None, None, None, None


def lpw_criterion(logits, labels, feat, teacher_feat, edge_index, kernel='cosine', beta=100, criterion='kld', _cls=None):
    """criterion.py:95-126 (teacher features are constants of the loss, as in the reference's call sites)."""
    if kernel not in _KERNELS or criterion not in ("kld", "mse"):
        raise NotImplementedError
    loss_cls = (_cls or cross_entropy)(logits, labels)
    plan = LspPlan.of(edge_index)
    loss_aux = _LSP.apply(feat, teacher_feat.detach(), plan, _KERNELS[kernel], 0 if criterion == "kld" else 1)
    return loss_cls + beta * loss_aux, loss_cls, loss_aux


# ----------------------------------------------------------------------------------------- G-CRD
# Logits chunk [R, S] of the G-CRD loss.  What sets the size is how many rows R the chunk's three GEMMs get, not L2
# residency (at 32 MB the chunk and its transpose exceed the 50 MB L2 of an H100): at S = 16384, F = 256 one forward +
# backward takes 75 / 42 / 22 / 14 ms with 8 / 16 / 32 / 64 MB chunks (tools/bench_nce_chunk.py, H100).  32 MB keeps the
# loss's peak memory well under that of the S x S logits it avoids (tests/test_criterion_gpu.py bounds it at S = 8192).
NCE_CHUNK_BYTES = 32 << 20


def nce_chunk_rows(Sp: int) -> int:
    """Rows R of one [R, Sp] logits chunk (R * Sp * 4 <= NCE_CHUNK_BYTES, a multiple of 128, at most Sp)."""
    return min(max(128, (NCE_CHUNK_BYTES // (4 * Sp)) // 128 * 128), Sp)


class NceBuffers:
    """Every buffer of one InfoNCE forward + gradient over [Sp, Fp] operands: allocated once, so that a captured step (gcrd.py)
    reuses them on every replay.  g_s / g_t (d loss / d xs, d xt, [Sp, Fp]) exist when requested."""

    def __init__(self, Sp: int, Fp: int, device, need_s: bool = True, need_t: bool = True, alloc=None):
        """alloc(*shape): where the buffers come from (default torch.empty; gcrd.PerGraphGCRD passes views that several
        row sets share)."""
        R = nce_chunk_rows(Sp)
        e = alloc or (lambda *shape: torch.empty(*shape, dtype=torch.float32, device=device))
        self.Z, self.part, self.loss = e(R, Sp), e(Sp), e(1)
        self.xt_split = (e(Sp, Fp), e(Sp, Fp))                                    # B of Z_c = xs_c · xt^T
        self.g_s = e(Sp, Fp) if need_s else None
        self.xtT_split = (e(Fp, Sp), e(Fp, Sp)) if need_s else None                # B of dZ_c · xt
        self.g_t = e(Sp, Fp) if need_t else None
        self.Zt = e(Sp * R) if need_t else None
        self.xsT_split = (e(Fp * R), e(Fp * R)) if need_t else None                # B of dZ_c^T · xs_c, per chunk


def nce_chunks(xs_p: torch.Tensor, xt_p: torch.Tensor, S: int, b: NceBuffers) -> None:
    """The chunk loop of the G-CRD loss over zero-padded operands xs_p, xt_p [Sp, Fp] (S real rows; xs_p already carries
    1 / nce_T): b.loss = InfoNCE, and b.g_s / b.g_t = its gradients w.r.t. xs_p / xt_p when allocated.  Only launches on
    preallocated buffers, so it can be captured."""
    L, st = _L(), lib.stream_ptr()
    Sp, Fp = xs_p.shape
    R = b.Z.shape[0]
    xt_hi, xt_lo = ops.split_tf32(xt_p, hi=b.xt_split[0], lo=b.xt_split[1])
    if b.g_s is not None:
        xtT_hi, xtT_lo = ops.split_tf32(xt_p, transpose=True, hi=b.xtT_split[0], lo=b.xtT_split[1])
    if b.g_t is not None:
        b.g_t.zero_()
    for r0 in range(0, Sp, R):
        r = min(R, Sp - r0)                                          # multiple of 4
        Zc = b.Z[:r]
        ops.gemm_tf32x3(xs_p[r0:r0 + r], xt_hi, xt_lo, out=Zc)
        if r0 < S:
            lib.check(L.b200gnn_nce_rows_chunk_f32(_f32(Zc, "Z"), Sp, min(r, S - r0), S, r0, _f32(b.part, "part"), st),
                      "nce_rows_chunk_f32")
        if b.g_s is not None:
            ops.gemm_tf32x3(Zc, xtT_hi, xtT_lo, out=b.g_s[r0:r0 + r])
        if b.g_t is not None:
            Ztc = b.Zt[:Sp * r].view(Sp, r)
            lib.check(L.b200gnn_transpose_f32(_f32(Zc, "Z"), r, Sp, _f32(Ztc, "Zt"), st), "transpose_f32")
            hi, lo = ops.split_tf32(xs_p[r0:r0 + r], transpose=True, hi=b.xsT_split[0][:Fp * r].view(Fp, r),
                                    lo=b.xsT_split[1][:Fp * r].view(Fp, r))                  # [Fp, r]
            ops.gemm_tf32x3(Ztc, hi, lo, out=b.g_t, accumulate=True)
    lib.check(L.b200gnn_nce_finish_f32(_f32(b.part, "part"), S, _f32(b.loss, "loss"), st), "nce_finish_f32")


class _NCE(torch.autograd.Function):
    """InfoNCE between normalised student rows and teacher rows (criterion.py:139-146) WITHOUT the S x S logits tensor
    (1 GiB at the scripts' S = 16384, arxiv_pyg/scripts/run_gcn.sh:144).  The rows are streamed in chunks of R (R*S*4 <=
    NCE_CHUNK_BYTES): per chunk one [R,S] logits GEMM on the tensor cores, the
    fused row pass (log-sum-exp, loss term, d/dlogits in place), and the two gradient contractions
    d fs[chunk] = dZ_c · x_t and d f_t += dZ_c^T · x_s[chunk] (accumulating epilogue) — the gradients are complete when
    the forward returns, so the backward only scales them."""

    @staticmethod
    def forward(ctx, fs, ft, nce_T: float):
        fs, ft = fs.contiguous(), ft.contiguous()
        S, F_ = fs.shape
        xs, ns = _normalize(fs, 1.0 / nce_T)          # logits / T folded into the student operand
        xt, nt = _normalize(ft)
        # every matrix is zero-padded to multiples of 4 rows / columns (TMA row pitches): zero feature rows give zero
        # logits, the row pass only visits the S real rows and columns, so the padding never reaches the result
        xs_p, xt_p = _pad_k(_pad_k(xs, 1), 0), _pad_k(_pad_k(xt, 1), 0)
        need_s, need_t = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        bufs = NceBuffers(xs_p.shape[0], xs_p.shape[1], fs.device, need_s, need_t)
        nce_chunks(xs_p, xt_p, S, bufs)
        loss, g_s, g_t = bufs.loss, bufs.g_s, bufs.g_t
        saved = []
        if need_s:
            saved.append(_normalize_bwd(xs, ns, g_s[:S, :F_], 1.0 / nce_T))
        if need_t:
            saved.append(_normalize_bwd(xt, nt, g_t[:S, :F_]))
        ctx.flags = (need_s, need_t)
        ctx.save_for_backward(*saved)
        return loss[0]

    @staticmethod
    def backward(ctx, g):
        need_s, need_t = ctx.flags
        saved = list(ctx.saved_tensors)
        d_fs = saved.pop(0) * g if need_s else None
        d_ft = saved.pop(0) * g if need_t else None
        return d_fs, d_ft, None


def nce_criterion(logits, labels, feat, teacher_feat, beta=0.5, nce_T=0.075, max_samples=8192, sampled_inds=None, _cls=None):
    """criterion.py:129-149."""
    loss_cls = (_cls or cross_entropy)(logits, labels)
    inds = _sample(feat.shape[0], max_samples, feat.device, sampled_inds)
    if inds is not None:
        feat, teacher_feat = feat[inds], teacher_feat[inds]
    loss_aux = _NCE.apply(feat, teacher_feat, float(nce_T))
    return loss_cls + beta * loss_aux, loss_cls, loss_aux
