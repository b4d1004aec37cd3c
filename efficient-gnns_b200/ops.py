"""Operators: thin, checked launches of the C ABI plus their autograd wiring.

Every function here ends in a ``libb200gnn.so`` call on the current CUDA stream;
PyTorch only provides the device buffers and the autograd tape.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from . import lib
from .sparse import CsrGraph, SparseTensor

_REDUCE = {"sum": lib.REDUCE_SUM, "add": lib.REDUCE_SUM, "mean": lib.REDUCE_MEAN}


def set_spmm_variant(variant: int) -> None:
    """0 = automatic kernel choice, 1 = force the register-staged SpMM kernel (A/B measurements)."""
    lib.load().b200gnn_spmm_set_variant(int(variant))


def stat_slots(g: CsrGraph) -> int:
    return int(lib.load().b200gnn_spmm_stat_slots(g.n_chunks, g.n_hub))


def spmm_csr(g: CsrGraph, x: torch.Tensor, reduce: str = "sum", bias: Optional[torch.Tensor] = None,
             out: Optional[torch.Tensor] = None, stat_partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Y = reduce_e val[e]·X[col[e]] (+bias), optional fused column statistics. No autograd."""
    if reduce not in _REDUCE:
        raise ValueError(f"reduce={reduce!r}: the engine implements sum/add/mean (what the reference path uses)")
    if x.dim() != 2:
        raise lib.B200GnnError("spmm: dense operand must be [n_src, K]")
    if x.shape[0] < g.n_cols:   # extra trailing rows are harmless (upstream accepts them: mag_pyg/gnn.py:151-162 infers
        raise lib.B200GnnError(  # the sparse sizes as max+1 and multiplies by the full per-type feature matrix)
            f"spmm: dense operand has {x.shape[0]} rows, matrix has {g.n_cols} columns")
    K = x.shape[1]
    if out is None:
        out = torch.empty(g.n_rows, K, dtype=torch.float32, device=x.device)
    if g.n_rows == 0 or K == 0:
        return out
    L = lib.load()
    ws = g.hub_workspace(K)
    rc = L.b200gnn_spmm_csr_f32(
        lib.dptr(g.rowptr, torch.int32, "rowptr"), lib.dptr(g.col, torch.int32, "col"),
        lib.dptr(g.val, torch.float32, "val"), lib.dptr(x, torch.float32, "x"), x.stride(0),
        lib.dptr(out, torch.float32, "out"), out.stride(0), g.n_rows, g.n_cols, K, _REDUCE[reduce],
        lib.dptr(bias, torch.float32, "bias"), lib.dptr(stat_partial, torch.float32, "stat_partial"),
        g.chunk_rowptr.data_ptr(), g.n_chunks, g.hub_threshold, g.seg_len,
        g.hub_rows.data_ptr() if g.n_hub else None, g.hub_segptr.data_ptr() if g.n_hub else None,
        g.n_hub, g.n_seg, None if ws is None else ws.data_ptr(), lib.stream_ptr())
    lib.check(rc, "spmm_csr_f32")
    return out


def _host_ptr_array(ptrs):
    import ctypes as C
    return (C.c_void_p * len(ptrs))(*[C.c_void_p(int(p)) for p in ptrs])


def _host_i32_array(vals):
    import ctypes as C
    return (C.c_int32 * len(vals))(*[int(v) for v in vals])


def spmm_csr_scatter(g: CsrGraph, x: torch.Tensor, dst_ptrs, row_off, ld_dst: int, col_dst: int, reduce: str = "sum",
                     bias: Optional[torch.Tensor] = None) -> None:
    """Y = A·X (+bias) with output row i stored to the R-layout buffer of the rank that owns it (raw device addresses
    dst_ptrs[q], rows row_off[q]..row_off[q+1], pitch ld_dst floats, column offset col_dst): the aggregation's epilogue performs
    the multi-GPU engine's C->R exchange."""
    K = x.shape[1]
    L = lib.load()
    ws = g.hub_workspace(K)
    rc = L.b200gnn_spmm_csr_scatter_f32(
        lib.dptr(g.rowptr, torch.int32, "rowptr"), lib.dptr(g.col, torch.int32, "col"), lib.dptr(g.val, torch.float32, "val"),
        lib.dptr(x, torch.float32, "x"), x.stride(0), _host_ptr_array(dst_ptrs), _host_i32_array(row_off), len(dst_ptrs),
        int(ld_dst), int(col_dst), g.n_rows, g.n_cols, K, _REDUCE[reduce], lib.dptr(bias, torch.float32, "bias"),
        g.chunk_rowptr.data_ptr(), g.n_chunks, g.hub_threshold, g.seg_len,
        g.hub_rows.data_ptr() if g.n_hub else None, g.hub_segptr.data_ptr() if g.n_hub else None,
        g.n_hub, g.n_seg, None if ws is None else ws.data_ptr(), lib.stream_ptr())
    lib.check(rc, "spmm_csr_scatter_f32")


class _SpMM(torch.autograd.Function):
    """matmul(adj, x, reduce): backward is the same kernel on the cached CSC view
    (upstream torch_sparse spmm backward, SURVEY Appendix A.4)."""

    @staticmethod
    def forward(ctx, x, adj: SparseTensor, reduce: str):
        st = adj.storage
        g = st.engine_csr() if st.value() is not None else st.engine_csr_unweighted()
        ctx.adj, ctx.reduce = adj, reduce
        return spmm_csr(g, x.contiguous(), reduce)

    @staticmethod
    def backward(ctx, grad_out):
        st = ctx.adj.storage
        if ctx.reduce == "mean":
            gt = st.engine_csc("mean" if st.value() is None else "mean_value")
        else:
            gt = st.engine_csc("value")
        return spmm_csr(gt, grad_out.contiguous(), "sum"), None, None


def matmul(adj: SparseTensor, x: torch.Tensor, reduce: str = "sum") -> torch.Tensor:
    """torch_sparse.matmul(adj, dense, reduce) for reduce in {sum, add, mean}."""
    if reduce not in _REDUCE:
        raise ValueError(f"reduce={reduce!r} not implemented (reference path uses add/mean)")
    v = adj.storage.value()
    if v is not None and v.requires_grad:
        raise NotImplementedError("gradients w.r.t. sparse values are never taken on the reference path")
    if x.dim() == 1:
        return matmul(adj, x.unsqueeze(-1), reduce).squeeze(-1)
    return _SpMM.apply(x, adj, reduce)


# ----------------------------------------------------------------------------- dense row passes (raw launches)
def _f32(t, name):
    return lib.dptr(t, torch.float32, name)


def rows_slots(n_rows: int) -> int:
    return int(lib.load().b200gnn_rows_slots(n_rows))


def col_stats(y: torch.Tensor, partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    """partial[slots][2][K]: per-slot column sums / sums of squares of y [n,K]."""
    n, K = y.shape
    slots = rows_slots(n)
    if partial is None:
        partial = torch.empty(slots, 2, K, dtype=torch.float32, device=y.device)
    lib.check(lib.load().b200gnn_col_stats_f32(_f32(y, "y"), n, K, _f32(partial, "partial"), slots, lib.stream_ptr()),
              "col_stats_f32")
    return partial


def col_sum(y: torch.Tensor, out: Optional[torch.Tensor] = None, partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    n, K = y.shape
    slots = rows_slots(n)
    if out is None:
        out = torch.empty(K, dtype=torch.float32, device=y.device)
    if partial is None:
        partial = torch.empty(slots, 2, K, dtype=torch.float32, device=y.device)
    lib.check(lib.load().b200gnn_col_sum_f32(_f32(y, "y"), n, K, _f32(out, "out"), _f32(partial, "partial"), slots,
                                             lib.stream_ptr()), "col_sum_f32")
    return out


def bn_finalize(partial: torch.Tensor, n_rows: int, gamma, beta, eps: float = 1e-5, momentum: float = 0.1,
                running_mean=None, running_var=None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Returns a [4,K] tensor: rows = mean, invstd, scale, shift."""
    slots, _, K = partial.shape
    if out is None:
        out = torch.empty(4, K, dtype=torch.float32, device=partial.device)
    lib.check(lib.load().b200gnn_bn_finalize_f32(
        _f32(partial, "partial"), slots, K, n_rows, _f32(gamma, "gamma"), _f32(beta, "beta"), eps, momentum,
        _f32(running_mean, "running_mean"), _f32(running_var, "running_var"),
        out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), lib.stream_ptr()), "bn_finalize_f32")
    return out


def affine_relu_dropout(y: torch.Tensor, scale=None, shift=None, relu: bool = True, p: float = 0.0, seed: int = 0,
                        offset: int = 0, out: Optional[torch.Tensor] = None, step_dev: Optional[torch.Tensor] = None,
                        step_mul: int = 0, row_offset: int = 0) -> torch.Tensor:
    n, K = y.shape
    if out is None:
        out = torch.empty_like(y)
    lib.check(lib.load().b200gnn_affine_relu_dropout_f32(
        _f32(y, "y"), _f32(out, "out"), n, K, _f32(scale, "scale"), _f32(shift, "shift"), int(relu), p, seed, offset,
        lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, row_offset, lib.stream_ptr()), "affine_relu_dropout_f32")
    return out


def affine_relu_dropout_mapped(y: torch.Tensor, scale=None, shift=None, relu: bool = True, p: float = 0.0, seed: int = 0,
                               offset: int = 0, out: Optional[torch.Tensor] = None, step_dev: Optional[torch.Tensor] = None,
                               step_mul: int = 0, rowmap: Optional[torch.Tensor] = None, row_offset: int = 0,
                               k_global: Optional[int] = None, col_offset: int = 0) -> torch.Tensor:
    """affine_relu_dropout on a row/column BLOCK of an [N, k_global] activation matrix: local row r is node
    rowmap[r] (int32) or r + row_offset, local columns start at col_offset.  Masks match the full-matrix call."""
    n, K = y.shape
    if out is None:
        out = torch.empty_like(y)
    lib.check(lib.load().b200gnn_affine_relu_dropout_mapped_f32(
        _f32(y, "y"), _f32(out, "out"), n, K, _f32(scale, "scale"), _f32(shift, "shift"), int(relu), p, seed, offset,
        lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, lib.dptr(rowmap, torch.int32, "rowmap"), row_offset,
        K if k_global is None else k_global, col_offset, lib.stream_ptr()), "affine_relu_dropout_mapped_f32")
    return out


def affine_relu_dropout_scatter(y: torch.Tensor, scale, shift, relu: bool, p: float, seed: int, offset: int, out: torch.Tensor,
                                step_dev, step_mul: int, rowmap, k_global: int, col_offset: int, dst_ptrs, row_off,
                                ld_dst: int) -> torch.Tensor:
    """affine_relu_dropout_mapped that ALSO stores every output row into the R-layout buffer of the rank owning the node
    (the multi-GPU engine's C->R exchange fused into the activation pass)."""
    n, K = y.shape
    lib.check(lib.load().b200gnn_affine_relu_dropout_scatter_f32(
        _f32(y, "y"), _f32(out, "out"), n, K, _f32(scale, "scale"), _f32(shift, "shift"), int(relu), p, seed, offset,
        lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, lib.dptr(rowmap, torch.int32, "rowmap"), 0, k_global, col_offset,
        _host_ptr_array(dst_ptrs), _host_i32_array(row_off), len(dst_ptrs), int(ld_dst), lib.stream_ptr()),
        "affine_relu_dropout_scatter_f32")
    return out


def dropout_mask(n_rows: int, K: int, p: float, seed: int, offset: int, device="cuda") -> torch.Tensor:
    """The keep-mask (uint8 [n,K]) that affine_relu_dropout uses for (seed, offset)."""
    mask = torch.empty(n_rows, K, dtype=torch.uint8, device=device)
    lib.check(lib.load().b200gnn_dropout_mask_u8(mask.data_ptr(), n_rows, K, p, seed, offset, lib.stream_ptr()),
              "dropout_mask_u8")
    return mask


def dropout_bits(bits: torch.Tensor, p: float, seed: int, offset: int, step_dev: Optional[torch.Tensor] = None,
                 step_mul: int = 0, K: Optional[int] = None) -> torch.Tensor:
    """Fill int32 bits[L, n, ceil(K/32)] with the keep decisions of affine_relu_dropout, one bit per element: layer l uses
    offset + l (+ step_dev * step_mul).  K defaults to 32 * bits.shape[2]."""
    n_layers, n, words = bits.shape
    K = 32 * words if K is None else K
    assert bits.dtype == torch.int32 and bits.is_contiguous() and words == (K + 31) // 32
    lib.check(lib.load().b200gnn_dropout_bits_u32(bits.data_ptr(), n_layers, n, K, p, seed, offset,
                                                  lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, lib.stream_ptr()),
              "dropout_bits_u32")
    return bits


def _bits(bits: torch.Tensor, n: int, K: int) -> int:
    if bits.dtype != torch.int32 or not bits.is_cuda or not bits.is_contiguous() or tuple(bits.shape) != (n, (K + 31) // 32):
        raise lib.B200GnnError(f"keep bits: expected a contiguous CUDA int32 [{n}, {(K + 31) // 32}] tensor")
    return bits.data_ptr()


def affine_relu_bits(y: torch.Tensor, bits: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, p: float,
                     out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dropout(relu(y*scale + shift)) with the keep decisions of ``dropout_bits`` (bit-identical to affine_relu_dropout)."""
    n, K = y.shape
    if out is None:
        out = torch.empty_like(y)
    lib.check(lib.load().b200gnn_affine_relu_bits_f32(_f32(y, "y"), _bits(bits, n, K), _f32(scale, "scale"), _f32(shift, "shift"),
                                                      p, _f32(out, "out"), n, K, lib.stream_ptr()), "affine_relu_bits_f32")
    return out


def gather_rows_act(x: torch.Tensor, idx: torch.Tensor, out: torch.Tensor, bits: Optional[torch.Tensor] = None,
                    scale: Optional[torch.Tensor] = None, shift: Optional[torch.Tensor] = None, p: float = 0.0) -> torch.Tensor:
    """out[i] = x[idx[i]] (idx int64), or with ``bits`` the activation dropout(relu(x[idx[i]]*scale + shift)) of
    ``affine_relu_bits`` (bit-identical) without materialising it for every row."""
    n, K = out.shape
    assert x.shape[1] == K and idx.numel() == n
    lib.check(lib.load().b200gnn_gather_rows_act_f32(
        _f32(x, "x"), x.stride(0), lib.dptr(idx, torch.int64, "idx"),
        n, K, None if bits is None else _bits(bits, x.shape[0], K), _f32(scale, "scale"), _f32(shift, "shift"), float(p),
        _f32(out, "out"), lib.stream_ptr()), "gather_rows_act_f32")
    return out


def lsp_student(feat: torch.Tensor, src: torch.Tensor, dst: torch.Tensor, rowptr: torch.Tensor, sim_t: torch.Tensor, kernel: int,
                pos_dst: torch.Tensor, pos_src: torch.Tensor, comb_rowptr: torch.Tensor, diag_pos: torch.Tensor,
                sim_s: torch.Tensor, scratch: torch.Tensor, val: torch.Tensor, selfc: torch.Tensor, loss: torch.Tensor,
                partial: torch.Tensor) -> None:
    """The student side of the LSP loss (kld) over a dst-sorted edge list (criterion.LspPlan) and its backward matrix: sim_s,
    the backward matrix's values val (selfc scratch) and loss[0], bit-identical to edge_sim -> lsp_segment -> lsp_bwd_values.
    feat [n_nodes, F] with F <= lib.LSP_MAX_F; scratch [2E]."""
    E, n_seg, n_nodes = src.numel(), rowptr.numel() - 1, comb_rowptr.numel() - 1
    assert dst.numel() == E and sim_t.numel() == E and sim_s.numel() == E and scratch.numel() >= 2 * E
    assert pos_dst.numel() == E and pos_src.numel() == E and diag_pos.numel() == n_nodes and feat.shape[0] >= n_nodes
    assert val.numel() == selfc.numel() == 2 * E + n_nodes and partial.numel() >= int(lib.load().b200gnn_lsp_partials(n_seg))
    i32 = lambda t, name: lib.dptr(t, torch.int32, name)
    lib.check(lib.load().b200gnn_lsp_student_f32(
        _f32(feat, "feat"), feat.shape[1], i32(src, "src"), i32(dst, "dst"), i32(rowptr, "rowptr"), n_seg, E,
        _f32(sim_t, "sim_t"), int(kernel), i32(pos_dst, "pos_dst"), i32(pos_src, "pos_src"), i32(comb_rowptr, "comb_rowptr"),
        i32(diag_pos, "diag_pos"), n_nodes, _f32(sim_s, "sim_s"), _f32(scratch, "scratch"), _f32(val, "val"),
        _f32(selfc, "selfc"), _f32(loss, "loss"), _f32(partial, "partial"), lib.stream_ptr()), "lsp_student_f32")


def scatter_rows_scaled(src: torch.Tensor, idx: torch.Tensor, scale: float, out: torch.Tensor,
                        loss_aux: Optional[torch.Tensor] = None, loss_total: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[idx[i]] = src[i] * scale (fp32 product; idx int64); no other row of out is written.  With loss_total, also
    loss_total[0] += loss_aux[0] * scale (fp32 product, then fp32 add)."""
    n, K = src.shape
    assert idx.numel() == n and out.dim() == 2 and out.shape[1] == K and out.stride(1) == 1
    if out.dtype != torch.float32 or not out.is_cuda:
        raise lib.B200GnnError("scatter_rows_scaled: out must be a float32 CUDA tensor")
    lib.check(lib.load().b200gnn_scatter_rows_scaled_f32(
        _f32(src, "src"), lib.dptr(idx, torch.int64, "idx"), n, K, float(scale), out.data_ptr(), out.stride(0),
        _f32(loss_aux, "loss_aux"), _f32(loss_total, "loss_total"), lib.stream_ptr()), "scatter_rows_scaled_f32")
    return out


def gsp_contract_workspace(n_rows: int, S: int, F: int, device) -> Optional[torch.Tensor]:
    """The workspace gsp_contract_narrow needs for n_rows rows (None when S fits one slab)."""
    nbytes = int(lib.load().b200gnn_gsp_contract_workspace_bytes(n_rows, S, F))
    return torch.empty(nbytes, dtype=torch.uint8, device=device) if nbytes else None


def gsp_contract_narrow(dG: torch.Tensor, S: int, x: torch.Tensor, out: torch.Tensor,
                        workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[i, :F] = sum_{j<S} dG[i, j] x[j, :F] in fp32 FMA (b200gnn_gsp_contract_narrow_f32): dG [n_rows, >= S] rows at a
    row pitch, x [>= S, F] with F a multiple of 4 up to lib.GSP_CONTRACT_MAX_F, out [n_rows, F] at a row pitch.  Row i of
    out depends on row i of dG and on x only.  workspace: gsp_contract_workspace(n_rows, S, F) or larger."""
    n_rows, F = dG.shape[0], x.shape[1]
    assert out.shape[0] == n_rows and out.shape[1] == F and x.shape[0] >= S
    for t, name in ((dG, "dG"), (x, "x"), (out, "out")):
        if t.dtype != torch.float32 or not t.is_cuda or t.stride(1) != 1:
            raise lib.B200GnnError(f"gsp_contract_narrow: {name} must be float32 CUDA rows with unit column stride")
    ws = 0 if workspace is None else workspace.numel() * workspace.element_size()
    lib.check(lib.load().b200gnn_gsp_contract_narrow_f32(
        dG.data_ptr(), dG.stride(0), n_rows, int(S), x.data_ptr(), x.stride(0), F, out.data_ptr(), out.stride(0),
        None if workspace is None else workspace.data_ptr(), ws, lib.stream_ptr()), "gsp_contract_narrow_f32")
    return out


def bn_act_bwd(d_out, x_out, y, mean, invstd, gamma, p: float, d_y=None, d_gamma=None, d_beta=None, d_bias=None,
               partial=None, coef=None, want_dbias: bool = True):
    """Backward of x_out = dropout_p(relu(BN_train(y))). Returns (d_y, d_gamma, d_beta, d_bias)."""
    n, K = y.shape
    dev = y.device
    slots = rows_slots(n)
    d_y = torch.empty_like(y) if d_y is None else d_y
    d_gamma = torch.empty(K, device=dev) if d_gamma is None else d_gamma
    d_beta = torch.empty(K, device=dev) if d_beta is None else d_beta
    if want_dbias and d_bias is None:
        d_bias = torch.empty(K, device=dev)
    partial = torch.empty(slots, 2, K, device=dev) if partial is None else partial
    coef = torch.empty(3, K, device=dev) if coef is None else coef
    lib.check(lib.load().b200gnn_bn_act_bwd_f32(
        _f32(d_out, "d_out"), _f32(x_out, "x_out"), _f32(y, "y"), _f32(mean, "mean"), _f32(invstd, "invstd"),
        _f32(gamma, "gamma"), n, K, p, _f32(d_y, "d_y"), _f32(d_gamma, "d_gamma"), _f32(d_beta, "d_beta"),
        _f32(d_bias, "d_bias") if want_dbias else None, _f32(partial, "partial"), slots, _f32(coef, "coef"),
        lib.stream_ptr()), "bn_act_bwd_f32")
    return d_y, d_gamma, d_beta, d_bias


def adam_step(params, grads, exp_avg, exp_avg_sq, step: torch.Tensor, lr: float, betas=(0.9, 0.999), eps: float = 1e-8):
    lib.check(lib.load().b200gnn_adam_step_f32(
        _f32(params, "params"), _f32(grads, "grads"), _f32(exp_avg, "exp_avg"), _f32(exp_avg_sq, "exp_avg_sq"),
        params.numel(), lr, betas[0], betas[1], eps, lib.dptr(step, torch.int32, "step"), lib.stream_ptr()),
        "adam_step_f32")


def kd_loss_fwd_bwd(logits, labels, train_idx, teacher_logits=None, alpha: float = 0.9, T: float = 4.0,
                    d_logits=None, loss_out=None, partial=None, n_norm: int = 0):
    """Fused CE / logit-KD over rows train_idx of FULL [N,C] matrices; returns (loss_out[3], d_logits [N,C])."""
    N, C = logits.shape
    n_train = train_idx.numel() if train_idx is not None else N
    L = lib.load()
    if d_logits is None:
        d_logits = torch.zeros_like(logits)
    if loss_out is None:
        loss_out = torch.empty(3, dtype=torch.float32, device=logits.device)
    if partial is None:
        partial = torch.empty(2 * int(L.b200gnn_kd_partials(max(n_train, 1))), dtype=torch.float32, device=logits.device)
    lib.check(L.b200gnn_kd_loss_fwd_bwd_f32(
        _f32(logits, "logits"), logits.stride(0), lib.dptr(train_idx, torch.int64, "train_idx"), n_train,
        lib.dptr(labels, torch.int64, "labels"), _f32(teacher_logits, "teacher_logits"),
        teacher_logits.stride(0) if teacher_logits is not None else 0, C, alpha, T, n_norm, _f32(d_logits, "d_logits"),
        d_logits.stride(0), _f32(loss_out, "loss_out"), _f32(partial, "partial"), lib.stream_ptr()), "kd_loss_fwd_bwd_f32")
    return loss_out, d_logits


# ----------------------------------------------------------------------------- wgmma 3xTF32 GEMM
def split_tf32(w: torch.Tensor, transpose: bool = False, hi: Optional[torch.Tensor] = None,
               lo: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """(hi, lo) tf32 split of a small [rows, cols] matrix; transposed ([cols, rows]) output if requested."""
    rows, cols = w.shape
    shape = (cols, rows) if transpose else (rows, cols)
    hi = torch.empty(shape, dtype=torch.float32, device=w.device) if hi is None else hi
    lo = torch.empty(shape, dtype=torch.float32, device=w.device) if lo is None else lo
    lib.check(lib.load().b200gnn_split_tf32_f32(_f32(w, "w"), rows, cols, int(transpose), _f32(hi, "hi"), _f32(lo, "lo"),
                                                lib.stream_ptr()), "split_tf32_f32")
    return hi, lo


def gemm_tf32x3(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, bias: Optional[torch.Tensor] = None,
                out: Optional[torch.Tensor] = None, accumulate: bool = False) -> torch.Tensor:
    """out[M,N] (+)= a[M,K] @ b[N,K]^T (+bias) with fp32 fidelity on the tensor cores (b pre-split by split_tf32)."""
    M, K = a.shape
    N = b_hi.shape[0]
    assert b_hi.shape == b_lo.shape and b_hi.shape[1] == K
    if out is None:
        assert not accumulate
        out = torch.empty(M, N, dtype=torch.float32, device=a.device)
    L = lib.load()
    if accumulate:
        assert bias is None
        lib.check(L.b200gnn_gemm_tf32x3_acc_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K, lib.stream_ptr()),
                  "gemm_tf32x3_acc_f32")
        return out
    lib.check(L.b200gnn_gemm_tf32x3_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                        b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K,
                                        _f32(bias, "bias"), lib.stream_ptr()), "gemm_tf32x3_f32")
    return out


def gemm_stat_slots(m: int, n: int) -> int:
    """Slots of the [slots, 2, n] partial buffer the statistics-fused GEMMs fill."""
    return int(lib.load().b200gnn_gemm_stat_slots(m, n))


def gemm_stats_supported(n: int) -> bool:
    return n % 32 == 0 and 48 < n <= 256


def gemm_tf32x3_stats(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                      partial: torch.Tensor, accumulate: bool = False) -> torch.Tensor:
    """out = a @ b^T + bias (or out += a @ b^T) with the BatchNorm batch statistics of the final ``out`` reduced in the epilogue:
    partial[slots, 2, N] = per-slot (column sum, column sum of squares) — feed to ``bn_finalize`` (no sweep over out)."""
    M, K = a.shape
    N = b_hi.shape[0]
    lib.check(lib.load().b200gnn_gemm_tf32x3_stats_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                       b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K, _f32(bias, "bias"),
                                                       int(accumulate), _f32(partial, "partial"), partial.shape[0], lib.stream_ptr()),
              "gemm_tf32x3_stats_f32")
    return out


def gemm_tf32x3_bnbwd(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, out: torch.Tensor, x_out: torch.Tensor,
                      y: torch.Tensor, mean: torch.Tensor, invstd: torch.Tensor, p: float, partial: torch.Tensor,
                      accumulate: bool = False) -> torch.Tensor:
    """Input-gradient GEMM with pass 1 of the BatchNorm/ReLU/dropout backward in its epilogue: d_out = a @ b^T (+ out),
    and what is STORED to ``out`` is dz = d_out * [x_out > 0] / (1-p); partial[slots, 2, N] = per-slot (sum dz, sum dz*xhat).
    Follow with ``bn_act_bwd_apply(out, None, y, ..., sums=partial, ...)``."""
    M, K = a.shape
    N = b_hi.shape[0]
    assert out.shape == x_out.shape == y.shape and out.stride(0) == x_out.stride(0) == y.stride(0)
    lib.check(lib.load().b200gnn_gemm_tf32x3_bnbwd_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                       b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K, int(accumulate),
                                                       _f32(x_out, "x_out"), _f32(y, "y"), _f32(mean, "mean"),
                                                       _f32(invstd, "invstd"), float(p), _f32(partial, "partial"),
                                                       partial.shape[0], lib.stream_ptr()), "gemm_tf32x3_bnbwd_f32")
    return out


def gemm_tf32x3_bnbwd_bits(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, out: torch.Tensor, bits: torch.Tensor,
                           y: torch.Tensor, mean: torch.Tensor, invstd: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor,
                           p: float, partial: torch.Tensor, accumulate: bool = False) -> torch.Tensor:
    """gemm_tf32x3_bnbwd for an activation that is not materialised: [x_out > 0] is taken as bit && y*scale + shift > 0."""
    M, K = a.shape
    N = b_hi.shape[0]
    assert out.shape == y.shape and out.stride(0) == y.stride(0)
    lib.check(lib.load().b200gnn_gemm_tf32x3_bnbwd_bits_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                            b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K, int(accumulate),
                                                            _bits(bits, M, N), _f32(y, "y"), _f32(mean, "mean"), _f32(invstd, "invstd"),
                                                            _f32(scale, "scale"), _f32(shift, "shift"), float(p),
                                                            _f32(partial, "partial"), partial.shape[0], lib.stream_ptr()),
              "gemm_tf32x3_bnbwd_bits_f32")
    return out


def gemm_tf32x3_act(y: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, bits: torch.Tensor, p: float, b_hi: torch.Tensor,
                    b_lo: torch.Tensor, bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = dropout(relu(y*scale + shift)) @ b^T (+bias), the activation formed in the GEMM's registers from y and the keep
    bits of ``dropout_bits``: bit for bit gemm_tf32x3 of the materialised activation."""
    M, K = y.shape
    N = b_hi.shape[0]
    assert b_hi.shape == b_lo.shape and b_hi.shape[1] == K
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=y.device)
    lib.check(lib.load().b200gnn_gemm_tf32x3_act_f32(_f32(y, "y"), y.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                     b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K, _f32(bias, "bias"),
                                                     _f32(scale, "scale"), _f32(shift, "shift"), _bits(bits, M, K), float(p),
                                                     lib.stream_ptr()), "gemm_tf32x3_act_f32")
    return out


def gemm_tf32x3_rowidx(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, out: torch.Tensor,
                       row_idx: torch.Tensor) -> torch.Tensor:
    """out[row_idx[m]] = (a @ b^T)[m] (row_idx int64, distinct); rows of out that row_idx does not name are left as they are."""
    M, K = a.shape
    N = b_hi.shape[0]
    assert b_hi.shape == b_lo.shape and b_hi.shape[1] == K and row_idx.numel() == M and out.shape[1] == N
    lib.check(lib.load().b200gnn_gemm_tf32x3_rowidx_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                        b_hi.stride(0), _f32(out, "out"), out.stride(0), M, N, K,
                                                        lib.dptr(row_idx, torch.int64, "row_idx"), lib.stream_ptr()),
              "gemm_tf32x3_rowidx_f32")
    return out


def gemm_tf32x3_scatter(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, dst_ptrs, row_off: int,
                        bias: Optional[torch.Tensor] = None) -> None:
    """a[M,K] @ b[N,K]^T with column block q of the result stored to the [*, N/world] matrix at raw device address
    dst_ptrs[q] (rows row_off + m): the GEMM epilogue performs the multi-GPU engine's R->C exchange (peer-mapped targets)."""
    import ctypes as C
    M, K = a.shape
    N = b_hi.shape[0]
    world = len(dst_ptrs)
    arr = (C.c_void_p * world)(*[C.c_void_p(int(p)) for p in dst_ptrs])
    lib.check(lib.load().b200gnn_gemm_tf32x3_scatter_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                         b_hi.stride(0), arr, world, int(row_off), M, N, K, _f32(bias, "bias"),
                                                         lib.stream_ptr()), "gemm_tf32x3_scatter_f32")


def gemm_tf32x3_bcast(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, dst_ptrs, row_off: int, ldc: int,
                      bias: Optional[torch.Tensor] = None) -> None:
    """a[M,K] @ b[N,K]^T stored to EVERY buffer at raw address dst_ptrs[q] (rows row_off + m, pitch ldc): the multi-GPU
    engine's row all-gather of a narrow result fused into the GEMM epilogue."""
    M, K = a.shape
    N = b_hi.shape[0]
    lib.check(lib.load().b200gnn_gemm_tf32x3_bcast_f32(_f32(a, "a"), a.stride(0), _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"),
                                                       b_hi.stride(0), _host_ptr_array(dst_ptrs), len(dst_ptrs), int(row_off), int(ldc),
                                                       M, N, K, _f32(bias, "bias"), lib.stream_ptr()), "gemm_tf32x3_bcast_f32")


def wgrad_supported(k_in: int, n_out: int) -> bool:
    """Shapes gemm_wgrad_tf32x3 accepts by default: the 128/256-row tilings of the GCN / SAGE layers."""
    return k_in in (128, 256) and n_out % 4 == 0 and 0 < n_out <= 256


def wgrad_workspace_floats(k_in: int, n_out: int) -> int:
    """Size of the workspace gemm_wgrad_tf32x3 fills (fp32 elements)."""
    return int(lib.load().b200gnn_wgrad_workspace_floats(k_in, n_out))


def gemm_wgrad_tf32x3(x: torch.Tensor, g: torch.Tensor, out: Optional[torch.Tensor] = None,
                      workspace: Optional[torch.Tensor] = None, wide: bool = False) -> torch.Tensor:
    """out[Kin,Nout] = x[Nn,Kin]^T @ g[Nn,Nout] on the tensor cores with fp32 fidelity (split-K over nodes).

    By default only the shapes of ``wgrad_supported`` are accepted (others raise B200GnnError), so a caller that picks its
    path by that predicate never reaches a padded tiling by accident.  ``wide=True`` accepts everything the kernel takes:
    Kin and Nout multiples of 4 up to 2048 and 512, ragged 128-row / 32-column tiles zero-filled (the R-GCN's
    [Wroot | W_r1 | ...] blocks)."""
    nn_, k_in = x.shape
    n_out = g.shape[1]
    assert g.shape[0] == nn_
    if not wide and not wgrad_supported(k_in, n_out):
        raise lib.B200GnnError(f"gemm_wgrad_tf32x3: Kin={k_in}, Nout={n_out} is outside the 128/256-row tilings "
                               "(pass wide=True for the padded ones)")
    L = lib.load()
    if out is None:
        out = torch.empty(k_in, n_out, dtype=torch.float32, device=x.device)
    if workspace is None:
        n_ws = int(L.b200gnn_wgrad_workspace_floats(k_in, n_out))
        if n_ws < 0:
            lib.check(n_ws, "wgrad_workspace_floats")
        workspace = torch.empty(n_ws, dtype=torch.float32, device=x.device)
    lib.check(L.b200gnn_gemm_wgrad_tf32x3_f32(_f32(x, "x"), x.stride(0), _f32(g, "g"), g.stride(0), _f32(out, "out"), nn_,
                                              k_in, n_out, _f32(workspace, "workspace"), lib.stream_ptr()),
              "gemm_wgrad_tf32x3_f32")
    return out


def gemm_wgrad_tf32x3_act(y: torch.Tensor, scale: torch.Tensor, shift: torch.Tensor, bits: torch.Tensor, p: float,
                          g: torch.Tensor, out: Optional[torch.Tensor] = None,
                          workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemm_wgrad_tf32x3 of x = dropout(relu(y*scale + shift)), x formed in registers from y and the keep bits."""
    nn_, k_in = y.shape
    n_out = g.shape[1]
    assert g.shape[0] == nn_
    if not wgrad_supported(k_in, n_out):
        raise lib.B200GnnError(f"gemm_wgrad_tf32x3_act: Kin={k_in}, Nout={n_out} is outside the 128/256-row tilings")
    L = lib.load()
    if out is None:
        out = torch.empty(k_in, n_out, dtype=torch.float32, device=y.device)
    if workspace is None:
        workspace = torch.empty(int(L.b200gnn_wgrad_workspace_floats(k_in, n_out)), dtype=torch.float32, device=y.device)
    lib.check(L.b200gnn_gemm_wgrad_tf32x3_act_f32(_f32(y, "y"), y.stride(0), _f32(g, "g"), g.stride(0), _f32(out, "out"), nn_,
                                                  k_in, n_out, _f32(scale, "scale"), _f32(shift, "shift"), _bits(bits, nn_, k_in),
                                                  float(p), _f32(workspace, "workspace"), lib.stream_ptr()),
              "gemm_wgrad_tf32x3_act_f32")
    return out


def partial_reduce(partial: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[slots, 2, K] (or [slots, K2]) partial sums -> [2, K] / [K2] totals (before a cross-rank all-reduce)."""
    slots = partial.shape[0]
    k2 = partial.numel() // slots
    if out is None:
        out = torch.empty(partial.shape[1:], dtype=torch.float32, device=partial.device)
    lib.check(lib.load().b200gnn_partial_reduce_f32(_f32(partial, "partial"), slots, k2, _f32(out, "out"), lib.stream_ptr()),
              "partial_reduce_f32")
    return out


def bn_act_bwd_reduce(d_out, x_out, y, mean, invstd, p: float, partial: torch.Tensor) -> torch.Tensor:
    n, K = y.shape
    lib.check(lib.load().b200gnn_bn_act_bwd_reduce_f32(_f32(d_out, "d_out"), _f32(x_out, "x_out"), _f32(y, "y"),
                                                       _f32(mean, "mean"), _f32(invstd, "invstd"), n, K, p,
                                                       _f32(partial, "partial"), partial.shape[0], lib.stream_ptr()),
              "bn_act_bwd_reduce_f32")
    return partial


def bn_act_bwd_apply(d_out, x_out, y, mean, invstd, gamma, sums, n_norm: int, p: float, d_y, d_gamma, d_beta, d_bias,
                     partial, coef):
    n, K = y.shape
    sum_slots = sums.numel() // (2 * K)
    lib.check(lib.load().b200gnn_bn_act_bwd_apply_f32(
        _f32(d_out, "d_out"), _f32(x_out, "x_out"), _f32(y, "y"), _f32(mean, "mean"), _f32(invstd, "invstd"),
        _f32(gamma, "gamma"), _f32(sums, "sums"), sum_slots, n_norm, n, K, p, _f32(d_y, "d_y"), _f32(d_gamma, "d_gamma"),
        _f32(d_beta, "d_beta"), _f32(d_bias, "d_bias"), _f32(partial, "partial"), partial.shape[0], _f32(coef, "coef"),
        lib.stream_ptr()), "bn_act_bwd_apply_f32")


# ----------------------------------------------------------------------------- R-GCN training passes
def relu_dropout_bwd(d_out: torch.Tensor, x_out: torch.Tensor, p: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Backward of x_out = dropout_p(relu(y)): d_y = d_out * [x_out > 0] / (1-p) (contiguous [n, K]; out may be d_out)."""
    n, K = x_out.shape
    out = torch.empty_like(x_out) if out is None else out
    if d_out.shape != x_out.shape or out.shape != x_out.shape:
        raise lib.B200GnnError(f"relu_dropout_bwd: d_out {tuple(d_out.shape)} and out {tuple(out.shape)} must have the shape "
                               f"of x_out {tuple(x_out.shape)}")
    lib.check(lib.load().b200gnn_relu_dropout_bwd_f32(_f32(d_out, "d_out"), _f32(x_out, "x_out"), _f32(out, "out"), n, K, float(p),
                                                      lib.stream_ptr()), "relu_dropout_bwd_f32")
    return out


MAX_TABLES = 16                         # Tables::ptr in csrc/hetero.cu


def _table(t, name: str, F: int, dev: torch.device) -> None:
    """The typed kernels index a table as fp32 rows of exactly F floats: anything else would be read as wrong rows."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.device != dev:
        raise lib.B200GnnError(f"{name}: expected a CUDA tensor on {dev}")
    if t.dtype != torch.float32 or t.dim() != 2 or not t.is_contiguous() or t.shape[1] != F:
        raise lib.B200GnnError(f"{name}: expected a contiguous float32 [rows, {F}] table, got {t.dtype} "
                               f"{tuple(t.shape)} with strides {t.stride()}")


def _index(t, name: str, n: int, dev: torch.device) -> int:
    """Device pointer of a contiguous int64 vector of length n (node types, local indices, sort orders)."""
    if not isinstance(t, torch.Tensor) or t.dim() != 1 or t.numel() != n:
        raise lib.B200GnnError(f"{name}: expected a 1-D int64 tensor of length {n}, got shape "
                               f"{None if not isinstance(t, torch.Tensor) else tuple(t.shape)}")
    if t.device != dev:
        raise lib.B200GnnError(f"{name}: expected a tensor on {dev}, got {t.device}")
    return lib.dptr(t, torch.int64, name)


def _node_type_key(k, n_types: int, what: str) -> int:
    import operator
    try:
        k = operator.index(k)
    except TypeError:
        raise lib.B200GnnError(f"{what} {k!r} is not an integer node type") from None
    if not 0 <= k < n_types:
        raise lib.B200GnnError(f"{what} {k} is not a node type in [0, {n_types})")
    return k


def _table_arrays(tables: dict, n_tables: int, F: int, dev: torch.device):
    """Host arrays (pointer, rows) indexed by node type; types without a table get a null pointer."""
    import ctypes as C
    if not 1 <= n_tables <= MAX_TABLES:
        raise lib.B200GnnError(f"typed tables: n_tables = {n_tables}, the kernels take 1..{MAX_TABLES} node types")
    ptrs = (C.c_void_p * n_tables)()
    rows = (C.c_int64 * n_tables)()
    for k, t in tables.items():
        k = _node_type_key(k, n_tables, "typed tables: key")
        _table(t, f"table of type {k}", F, dev)
        ptrs[k], rows[k] = t.data_ptr(), t.shape[0]
    return ptrs, rows


def typed_gather(tables: dict, n_tables: int, node_type: torch.Tensor, local_idx: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[i] = tables[node_type[i]][local_idx[i]] (zero rows for types without a table); tables: {type: [rows, F] fp32}.

    A local index outside its table raises B200GnnError naming the first such position, as the reference's indexing does.
    Reading the kernel's error flag waits for the stream; the R-GCN step already reads the host while it builds its batch
    plan, so this adds a wait but no new constraint (no caller captures the gather in a CUDA graph)."""
    if not isinstance(out, torch.Tensor) or out.dim() != 2:
        raise lib.B200GnnError("typed_gather: out must be a [n, F] tensor")
    n, F_ = out.shape
    ptrs, rows = _table_arrays(tables, n_tables, F_, out.device)
    err = torch.zeros(1, dtype=torch.int32, device=out.device)
    lib.check(lib.load().b200gnn_typed_gather_f32(ptrs, rows, n_tables, _index(node_type, "node_type", n, out.device),
                                                  _index(local_idx, "local_idx", n, out.device), n, F_,
                                                  _f32(out, "out"), out.stride(0), err.data_ptr(), lib.stream_ptr()),
              "typed_gather_f32")
    if int(err.item()):
        bad = torch.zeros(n, dtype=torch.bool, device=out.device)
        for k, t in tables.items():
            bad |= (node_type == k) & ((local_idx < 0) | (local_idx >= t.shape[0]))
        i = int(bad.nonzero()[0, 0])
        raise lib.B200GnnError(f"typed_gather: local index {int(local_idx[i])} at position {i} is outside the "
                               f"{tables[int(node_type[i])].shape[0]}-row table of node type {int(node_type[i])}")
    return out


def typed_scatter(d_out: torch.Tensor, node_type: torch.Tensor, local_idx: torch.Tensor, order: torch.Tensor, grads: dict,
                  n_tables: int) -> None:
    """grads[t][j] = sum of d_out[i] over nodes (node_type, local_idx) == (t, j), added in ``order`` (rows outside the batch are
    left untouched: pass zeroed tables for a dense gradient)."""
    if not isinstance(d_out, torch.Tensor) or d_out.dim() != 2:
        raise lib.B200GnnError("typed_scatter: d_out must be a [n, F] tensor")
    n, F_ = d_out.shape
    ptrs, rows = _table_arrays(grads, n_tables, F_, d_out.device)
    lib.check(lib.load().b200gnn_typed_scatter_f32(_f32(d_out, "d_out"), d_out.stride(0), _index(node_type, "node_type", n, d_out.device),
                                                   _index(local_idx, "local_idx", n, d_out.device),
                                                   _index(order, "order", n, d_out.device), n, F_, ptrs, rows, n_tables,
                                                   lib.stream_ptr()),
              "typed_scatter_f32")


def embedding_adam(d_out: torch.Tensor, node_type: torch.Tensor, local_idx: torch.Tensor, order: torch.Tensor, table_type: int,
                   table: torch.Tensor, exp_avg: torch.Tensor, exp_avg_sq: torch.Tensor, head: torch.Tensor, step: torch.Tensor,
                   lr: float, betas=(0.9, 0.999), eps: float = 1e-8) -> None:
    """Adam over one embedding table whose gradient is typed_scatter(d_out) (``order``: the rows of d_out sorted by
    (node_type, local_idx)); bit-identical to the scatter into a zeroed dense gradient + adam_step, reads ``step`` without
    advancing it.  head: int32 [rows] scratch, all -1 (restored on return)."""
    if not isinstance(d_out, torch.Tensor) or d_out.dim() != 2:
        raise lib.B200GnnError("embedding_adam: d_out must be a [n, F] tensor")
    n, F_ = d_out.shape
    dev = d_out.device
    table_type = _node_type_key(table_type, MAX_TABLES, "embedding_adam: table_type")
    for name, t in (("table", table), ("exp_avg", exp_avg), ("exp_avg_sq", exp_avg_sq)):
        _table(t, name, F_, dev)
    rows = table.shape[0]
    if exp_avg.shape != table.shape or exp_avg_sq.shape != table.shape:
        raise lib.B200GnnError(f"embedding_adam: moments {tuple(exp_avg.shape)}, {tuple(exp_avg_sq.shape)} do not match the "
                               f"table {tuple(table.shape)}")
    if not isinstance(head, torch.Tensor) or head.dim() != 1 or head.numel() < rows or head.device != dev:
        raise lib.B200GnnError(f"embedding_adam: head must be an int32 vector of at least {rows} entries on {dev}")
    if not isinstance(step, torch.Tensor) or step.numel() != 1 or step.device != dev:
        raise lib.B200GnnError(f"embedding_adam: step must be a one-element int32 tensor on {dev}")
    lib.check(lib.load().b200gnn_embedding_adam_f32(
        _f32(d_out, "d_out"), d_out.stride(0), _index(node_type, "node_type", n, dev), _index(local_idx, "local_idx", n, dev),
        _index(order, "order", n, dev), n, table_type,
        _f32(table, "table"), _f32(exp_avg, "exp_avg"), _f32(exp_avg_sq, "exp_avg_sq"), rows, F_,
        lib.dptr(head, torch.int32, "head"), lr, betas[0], betas[1], eps, lib.dptr(step, torch.int32, "step"), lib.stream_ptr()),
        "embedding_adam_f32")


# ----------------------------------------------------------------------------- SIGN (PReLU FeedForwardNet layers)
def _rows(t: torch.Tensor, name: str):
    """(device pointer, row pitch) of an fp32 CUDA matrix whose rows are contiguous (column blocks of a wider matrix pass)."""
    if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 2 or t.stride(1) != 1:
        raise lib.B200GnnError(f"{name}: expected a CUDA float32 matrix with contiguous rows")
    return t.data_ptr(), t.stride(0)


def _bits_rows(bits: torch.Tensor, n: int, K: int):
    """(pointer, row pitch in words) of int32 keep bits covering rows [0, n) and columns [0, K)."""
    if bits.dtype != torch.int32 or not bits.is_cuda or bits.dim() != 2 or bits.stride(1) != 1 or bits.shape[0] != n \
            or bits.shape[1] < (K + 31) // 32:
        raise lib.B200GnnError(f"keep bits: expected CUDA int32 [{n}, >= {(K + 31) // 32}] with contiguous rows")
    return bits.data_ptr(), bits.stride(0)


def prelu_bits(z: torch.Tensor, bits: torch.Tensor, slope: torch.Tensor, p: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dropout(prelu(z)) with the keep decisions of ``dropout_bits`` and the slope scalar (device): what the PReLU GEMM
    prologues form in registers, materialised."""
    n, K = z.shape
    if out is None:
        out = torch.empty(n, K, dtype=torch.float32, device=z.device)
    zp, ldz = _rows(z, "z")
    op, ldo = _rows(out, "out")
    bp, ldb = _bits_rows(bits, n, K)
    lib.check(lib.load().b200gnn_prelu_bits_f32(zp, ldz, bp, ldb, _f32(slope, "slope"), float(p), op, ldo, n, K, lib.stream_ptr()),
              "prelu_bits_f32")
    return out


def gemm_tf32x3_prelu(z: torch.Tensor, slope: torch.Tensor, bits: torch.Tensor, p: float, b_hi: torch.Tensor, b_lo: torch.Tensor,
                      bias: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = dropout(prelu(z)) @ b^T (+bias), the activation formed in the GEMM's registers: bit for bit gemm_tf32x3 of
    ``prelu_bits``.  ``out`` may be a column block of a wider matrix (row pitch taken from its stride)."""
    M, K = z.shape
    N = b_hi.shape[0]
    assert b_hi.shape == b_lo.shape and b_hi.shape[1] == K
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=z.device)
    zp, lda = _rows(z, "z")
    op, ldc = _rows(out, "out")
    if bits.shape[1] != (K + 31) // 32:
        raise lib.B200GnnError("gemm_tf32x3_prelu: keep bits must be [M, ceil(K/32)]")
    lib.check(lib.load().b200gnn_gemm_tf32x3_prelu_f32(zp, lda, _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"), b_hi.stride(0), op, ldc, M, N, K,
                                                       _f32(bias, "bias"), _f32(slope, "slope"), _bits(bits, M, K), float(p),
                                                       lib.stream_ptr()), "gemm_tf32x3_prelu_f32")
    return out


def gemm_tf32x3_prelu_stats(z: torch.Tensor, slope: torch.Tensor, bits: torch.Tensor, p: float, b_hi: torch.Tensor,
                            b_lo: torch.Tensor, bias: Optional[torch.Tensor], out: torch.Tensor,
                            partial: torch.Tensor) -> torch.Tensor:
    """out = dropout(prelu(z)) @ b^T + bias with the BatchNorm batch statistics of ``out`` in the epilogue: output and
    partial[slots, 2, N] bit for bit ``gemm_tf32x3_stats`` of ``prelu_bits(z, bits, slope, p)``, the activation never
    materialised.  N a multiple of 32 in (48, 256]."""
    M, K = z.shape
    N = b_hi.shape[0]
    assert b_hi.shape == b_lo.shape and b_hi.shape[1] == K
    zp, lda = _rows(z, "z")
    if bits.shape[1] != (K + 31) // 32:
        raise lib.B200GnnError("gemm_tf32x3_prelu_stats: keep bits must be [M, ceil(K/32)]")
    lib.check(lib.load().b200gnn_gemm_tf32x3_prelu_stats_f32(zp, lda, _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"), b_hi.stride(0),
                                                             _f32(out, "out"), out.stride(0), M, N, K, _f32(bias, "bias"),
                                                             _f32(slope, "slope"), _bits(bits, M, K), float(p),
                                                             _f32(partial, "partial"), partial.shape[0], lib.stream_ptr()),
              "gemm_tf32x3_prelu_stats_f32")
    return out


def gemm_tf32x3_prelu_bwd(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, out: torch.Tensor, z: torch.Tensor,
                          bits: torch.Tensor, slope: torch.Tensor, p: float, slope_grad: torch.Tensor, partial: torch.Tensor,
                          accumulate: bool = False, slope_accumulate: bool = False) -> torch.Tensor:
    """Input-gradient GEMM behind x = dropout(prelu(z)): d_x = a @ b^T (+ out if accumulate); STORES
    dz = d_x * keep / (1-p) * (z > 0 ? 1 : slope) to ``out`` and writes (or adds, slope_accumulate) the slope gradient to
    slope_grad[0].  ``a`` may be a column block (row pitch from its stride); partial: float64 [gemm_stat_slots(M, N)]."""
    M, K = a.shape
    N = b_hi.shape[0]
    assert out.shape == z.shape == (M, N) and out.stride(0) == z.stride(0)
    if partial.dtype != torch.float64 or not partial.is_cuda or partial.numel() < gemm_stat_slots(M, N):
        raise lib.B200GnnError("gemm_tf32x3_prelu_bwd: partial must be CUDA float64 [>= gemm_stat_slots(M, N)]")
    ap, lda = _rows(a, "a")
    op, ldc = _rows(out, "out")
    lib.check(lib.load().b200gnn_gemm_tf32x3_prelu_bwd_f32(ap, lda, _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"), b_hi.stride(0), op, ldc,
                                                           M, N, K, int(accumulate), _rows(z, "z")[0], _bits(bits, M, N),
                                                           _f32(slope, "slope"), float(p), slope_grad.data_ptr(),
                                                           int(slope_accumulate), partial.data_ptr(), partial.numel(),
                                                           lib.stream_ptr()), "gemm_tf32x3_prelu_bwd_f32")
    return out


WGRAD_PRELU_BLOCK = 512   # column block of a Z wider than the kernel's 2048-column tiling


def gemm_wgrad_tf32x3_prelu(z: torch.Tensor, slope: torch.Tensor, bits: torch.Tensor, p: float, g: torch.Tensor,
                            out: Optional[torch.Tensor] = None, workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[Kin, Nout] = dropout(prelu(z))^T @ g, the activation formed in registers (bit for bit gemm_wgrad_tf32x3 of
    ``prelu_bits``).  Kin > 2048 runs as 512-column blocks of z.  z and g may be column blocks (row pitches from strides)."""
    nn_, k_in = z.shape
    n_out = g.shape[1]
    assert g.shape[0] == nn_
    if k_in % 4 or n_out % 4:
        raise lib.B200GnnError(f"gemm_wgrad_tf32x3_prelu: Kin={k_in}, Nout={n_out} must be multiples of 4")
    L = lib.load()
    if out is None:
        out = torch.empty(k_in, n_out, dtype=torch.float32, device=z.device)
    blk = k_in if k_in <= 2048 else WGRAD_PRELU_BLOCK
    if workspace is None:
        workspace = torch.empty(wgrad_workspace_floats(blk, n_out), dtype=torch.float32, device=z.device)
    bp, ldb = _bits_rows(bits, nn_, k_in)
    gp, ldg = _rows(g, "g")
    assert out.is_contiguous()
    for c0 in range(0, k_in, blk):
        kb = min(blk, k_in - c0)
        zb, ldz = _rows(z[:, c0:c0 + kb], "z")
        lib.check(L.b200gnn_gemm_wgrad_tf32x3_prelu_f32(zb, ldz, gp, ldg, out[c0:c0 + kb].data_ptr(), nn_, kb, n_out,
                                                        _f32(slope, "slope"), bp + 4 * (c0 // 32), ldb, float(p),
                                                        _f32(workspace, "workspace"), lib.stream_ptr()),
                  "gemm_wgrad_tf32x3_prelu_f32")
    return out


def gemm_wgrad_tf32x3_rows(x: torch.Tensor, g: torch.Tensor, out: torch.Tensor, workspace: torch.Tensor) -> torch.Tensor:
    """gemm_wgrad_tf32x3 (any tiling it accepts) on operands that may be column blocks of wider matrices."""
    nn_, k_in = x.shape
    xp, ldx = _rows(x, "x")
    gp, ldg = _rows(g, "g")
    lib.check(lib.load().b200gnn_gemm_wgrad_tf32x3_f32(xp, ldx, gp, ldg, _f32(out, "out"), nn_, k_in, g.shape[1],
                                                       _f32(workspace, "workspace"), lib.stream_ptr()), "gemm_wgrad_tf32x3_f32")
    return out


def gemm_tf32x3_rows(a: torch.Tensor, b_hi: torch.Tensor, b_lo: torch.Tensor, out: torch.Tensor,
                     bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """gemm_tf32x3 with ``a`` / ``out`` possibly column blocks of wider matrices (row pitches from strides)."""
    M, K = a.shape
    N = b_hi.shape[0]
    ap, lda = _rows(a, "a")
    op, ldc = _rows(out, "out")
    lib.check(lib.load().b200gnn_gemm_tf32x3_f32(ap, lda, _f32(b_hi, "b_hi"), _f32(b_lo, "b_lo"), b_hi.stride(0), op, ldc, M, N, K,
                                                 _f32(bias, "bias"), lib.stream_ptr()), "gemm_tf32x3_f32")
    return out


def col_sum_ld(y: torch.Tensor, out: torch.Tensor, partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[K] = column sums of y [n, K] (rows contiguous, any pitch), fixed summation order."""
    n, K = y.shape
    L = lib.load()
    slots = int(L.b200gnn_col_sum_ld_slots(n))
    if partial is None:
        partial = torch.empty(slots * K, dtype=torch.float32, device=y.device)
    yp, ldy = _rows(y, "y")
    lib.check(L.b200gnn_col_sum_ld_f32(yp, ldy, n, K, _f32(out, "out"), partial.data_ptr(), partial.numel() // K, lib.stream_ptr()),
              "col_sum_ld_f32")
    return out


def sign_gather(feats, idx: torch.Tensor, p: float, seed: int, offset: int, out: torch.Tensor,
                step_dev: Optional[torch.Tensor] = None, step_mul: int = 0, labels: Optional[torch.Tensor] = None,
                labels_out: Optional[torch.Tensor] = None, teacher: Optional[torch.Tensor] = None,
                teacher_out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[h, i] = input_dropout(feats[h][idx[i]]) for every hop (hop h: the mask of dropout_mask(B, F, p, seed,
    offset + h + step * step_mul)), plus the batch's label and teacher-logit rows."""
    H = len(feats)
    B = idx.numel()
    n, F_ = feats[0].shape
    for f in feats:
        if f.shape != (n, F_):
            raise lib.B200GnnError("sign_gather: every hop feature matrix must have the same shape")
        _f32(f, "feats")
    assert out.shape == (H, B, F_)
    C = teacher.shape[1] if teacher is not None else 0
    lib.check(lib.load().b200gnn_sign_gather_f32(
        _host_ptr_array([f.data_ptr() for f in feats]), H, n, F_, lib.dptr(idx, torch.int64, "idx"), B, float(p), int(seed),
        int(offset), lib.dptr(step_dev, torch.int32, "step_dev"), int(step_mul), _f32(out, "out"),
        lib.dptr(labels, torch.int64, "labels"), lib.dptr(labels_out, torch.int64, "labels_out"),
        _f32(teacher, "teacher"), teacher.stride(0) if teacher is not None else 0, C, _f32(teacher_out, "teacher_out"),
        lib.stream_ptr()), "sign_gather_f32")
    return out


# ----------------------------------------------------------------------------- fused GAT layer (engine_gat.py)
def dropout_mask_step(mask: torch.Tensor, p: float, seed: int, offset: int, step_dev: torch.Tensor, step_mul: int) -> torch.Tensor:
    """Fill the flat uint8 ``mask`` (a multiple of 4 elements) with the decisions of ``dropout_mask`` for the effective offset
    offset + step_dev * step_mul, read on the device."""
    assert mask.dtype == torch.uint8 and mask.is_contiguous() and mask.numel() % 4 == 0
    lib.check(lib.load().b200gnn_dropout_mask_step_u8(mask.data_ptr(), mask.numel() // 4, 4, p, seed, offset,
                                                      lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, lib.stream_ptr()),
              "dropout_mask_step_u8")
    return mask


def gat_scores(ft: torch.Tensor, attn_l: torch.Tensor, attn_r: Optional[torch.Tensor], src_scale: Optional[torch.Tensor],
               H: int, el: Optional[torch.Tensor] = None, er: Optional[torch.Tensor] = None):
    """el[n,h] = src_scale[n]·<ft[n,h,:], attn_l[h,:]>, er[n,h] = <ft[n,h,:], attn_r[h,:]>; ft [N, H*D] may be a column block."""
    n, K = ft.shape
    fp, ldf = _rows(ft, "ft")
    el = torch.empty(n, H, dtype=torch.float32, device=ft.device) if el is None else el
    if attn_r is not None and er is None:
        er = torch.empty(n, H, dtype=torch.float32, device=ft.device)
    lib.check(lib.load().b200gnn_gat_scores_f32(fp, ldf, _f32(attn_l, "attn_l"), _f32(attn_r, "attn_r"), _f32(src_scale, "src_scale"),
                                                n, H, K // H, _f32(el, "el"), _f32(er, "er") if attn_r is not None else None,
                                                lib.stream_ptr()), "gat_scores_f32")
    return el, (er if attn_r is not None else None)


def gat_scores_slots(n_rows: int) -> int:
    return int(lib.load().b200gnn_gat_scores_slots(n_rows))


def gat_scores_bwd(ft: torch.Tensor, attn_l: torch.Tensor, attn_r: Optional[torch.Tensor], src_scale: Optional[torch.Tensor],
                   d_el: torch.Tensor, d_er: Optional[torch.Tensor], H: int, dft: torch.Tensor, d_attn_l: torch.Tensor,
                   d_attn_r: Optional[torch.Tensor], partial: Optional[torch.Tensor] = None) -> None:
    """dft += d_el·src_scale·attn_l + d_er·attn_r in place; d_attn_l / d_attn_r reduced through per-CTA partials in slot order."""
    n, K = ft.shape
    fp, ldf = _rows(ft, "ft")
    dp, ldd = _rows(dft, "dft")
    if partial is None:
        partial = torch.empty(gat_scores_slots(n), 2, K, dtype=torch.float32, device=ft.device)
    lib.check(lib.load().b200gnn_gat_scores_bwd_f32(
        fp, ldf, _f32(attn_l, "attn_l"), _f32(attn_r, "attn_r"), _f32(src_scale, "src_scale"), _f32(d_el, "d_el"),
        _f32(d_er, "d_er") if attn_r is not None else None, n, H, K // H, dp, ldd, _f32(d_attn_l, "d_attn_l"),
        _f32(d_attn_r, "d_attn_r") if attn_r is not None else None, _f32(partial, "partial"), partial.shape[0],
        lib.stream_ptr()), "gat_scores_bwd_f32")


def gat_stat_slots(g: CsrGraph) -> int:
    return int(lib.load().b200gnn_gat_stat_slots(g.n_chunks, g.n_hub))


def gat_aggregate_epi(g: CsrGraph, eidx: Optional[torch.Tensor], a: torch.Tensor, ft: torch.Tensor, out: torch.Tensor, H: int,
                      src_scale: Optional[torch.Tensor] = None, row_scale: Optional[torch.Tensor] = None,
                      res: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
                      stat_partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out[i] = row_scale[i]·Σ_e a[e,h]·src_scale[col[e]]·ft[col[e],h,:] + res[i] + bias, with the BatchNorm partial sums of the
    output rows in stat_partial [gat_stat_slots(g), 2, K]; ft / res / out may be column blocks.  No operands: gat_aggregate."""
    K = ft.shape[1]
    fp, ldf = _rows(ft, "ft")
    op, ldo = _rows(out, "out")
    rp, ldr = _rows(res, "res") if res is not None else (None, 0)
    ws = g.hub_workspace(K)
    lib.check(lib.load().b200gnn_gat_aggregate_epi_f32(
        g.rowptr.data_ptr(), g.col.data_ptr(), lib.dptr(eidx, torch.int32, "eidx"), _f32(a, "a"), fp, ldf, op, ldo, g.n_rows, H,
        K // H, _f32(src_scale, "src_scale"), _f32(row_scale, "row_scale"), rp, ldr, _f32(bias, "bias"),
        _f32(stat_partial, "stat_partial"), 0 if stat_partial is None else stat_partial.shape[0],
        g.chunk_rowptr.data_ptr(), g.n_chunks, g.hub_threshold, g.seg_len,
        g.hub_rows.data_ptr() if g.n_hub else None, g.hub_segptr.data_ptr() if g.n_hub else None, g.n_hub, g.n_seg,
        None if ws is None else ws.data_ptr(), lib.stream_ptr()), "gat_aggregate_epi_f32")
    return out


# ----------------------------------------------------------------------------- PPI GAT layers (engine_ppi.py)
def gat_aggregate_elu(g: CsrGraph, a: torch.Tensor, ft: torch.Tensor, out: torch.Tensor, act: torch.Tensor, H: int,
                      res: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """out = Z = Σ_e a[e,h]·ft[col[e],h,:] + res + bias (gat_aggregate_epi's output bit for bit) and act = elu(Z); ft / res / out /
    act may be column blocks of wider matrices.  act must be aligned like out (same 16- or 8-byte vector width)."""
    K = ft.shape[1]
    fp, ldf = _rows(ft, "ft")
    op, ldo = _rows(out, "out")
    ap, lda = _rows(act, "act")
    rp, ldr = _rows(res, "res") if res is not None else (None, 0)
    ws = g.hub_workspace(K)
    lib.check(lib.load().b200gnn_gat_aggregate_elu_f32(
        g.rowptr.data_ptr(), g.col.data_ptr(), None, _f32(a, "a"), fp, ldf, op, ldo, ap, lda, g.n_rows, H, K // H, rp, ldr,
        _f32(bias, "bias"), g.chunk_rowptr.data_ptr(), g.n_chunks, g.hub_threshold, g.seg_len,
        g.hub_rows.data_ptr() if g.n_hub else None, g.hub_segptr.data_ptr() if g.n_hub else None, g.n_hub, g.n_seg,
        None if ws is None else ws.data_ptr(), lib.stream_ptr()), "gat_aggregate_elu_f32")
    return out, act


def elu_bwd(d_act: torch.Tensor, z: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = d_act · (z > 0 ? 1 : exp(z)) (torch's elu_backward); every operand may be a column block (own row pitch)."""
    n, K = z.shape
    if d_act.shape != (n, K):
        raise lib.B200GnnError("elu_bwd: d_act and z must have the same shape")
    out = torch.empty(n, K, dtype=torch.float32, device=z.device) if out is None else out
    gp, ldg = _rows(d_act, "d_act")
    zp, ldz = _rows(z, "z")
    op, ldo = _rows(out, "out")
    lib.check(lib.load().b200gnn_elu_bwd_f32(gp, ldg, zp, ldz, op, ldo, n, K, lib.stream_ptr()), "elu_bwd_f32")
    return out


def ppi_tail_slots(n_rows: int) -> int:
    return int(lib.load().b200gnn_ppi_tail_slots(n_rows))


def ppi_logits_loss(agg: torch.Tensor, res: torch.Tensor, b_conv: torch.Tensor, b_lin: torch.Tensor, H: int, C: int,
                    logits: torch.Tensor, labels: Optional[torch.Tensor] = None, teacher_logits: Optional[torch.Tensor] = None,
                    alpha: float = 0.5, T: float = 1.0, d_agg: Optional[torch.Tensor] = None, d_res: Optional[torch.Tensor] = None,
                    loss_out: Optional[torch.Tensor] = None, partial: Optional[torch.Tensor] = None) -> torch.Tensor:
    """logits[:, :C] = (mean_h agg + b_conv) + (res + b_lin) over agg [n, H·Dp] and res [n, >= Dp]; with labels also the BCE /
    logit-KD loss into loss_out[3] and the seed gradients d_agg [n, H·Dp] (dz/H per head), d_res [n, >= Dp] (dz), padded
    columns written as zero.  Every matrix may be a column block; partial: float64 [2·ppi_tail_slots(n)]."""
    n = agg.shape[0]
    Dp = agg.shape[1] // H
    gp, lda = _rows(agg, "agg")
    rp, ldr = _rows(res, "res")
    lp, ldl = _rows(logits, "logits")
    yp, ldy = _rows(labels, "labels") if labels is not None else (None, C)
    tp, ldt = _rows(teacher_logits, "teacher_logits") if teacher_logits is not None else (None, C)
    train = labels is not None
    if train:
        if d_agg is None or d_res is None or loss_out is None:
            raise lib.B200GnnError("ppi_logits_loss: labels need d_agg, d_res and loss_out")
        if partial is None:
            partial = torch.empty(2 * ppi_tail_slots(n), dtype=torch.float64, device=agg.device)
        if partial.dtype != torch.float64 or not partial.is_cuda or not partial.is_contiguous():
            raise lib.B200GnnError("ppi_logits_loss: partial must be a contiguous CUDA float64 buffer")
    dap, ldga = _rows(d_agg, "d_agg") if train else (None, H * Dp)
    drp, ldgr = _rows(d_res, "d_res") if train else (None, Dp)
    lib.check(lib.load().b200gnn_ppi_logits_loss_f32(
        gp, lda, rp, ldr, _f32(b_conv, "b_conv"), _f32(b_lin, "b_lin"), n, H, Dp, C, lp, ldl, yp, ldy, tp, ldt, float(alpha),
        float(T), dap, ldga, drp, ldgr, _f32(loss_out, "loss_out") if train else None,
        partial.data_ptr() if train else None, partial.numel() // 2 if train else 0, lib.stream_ptr()), "ppi_logits_loss_f32")
    return logits


# ---------------------------------------------------------------------------------------------- GAT teacher recipe
ROLE_NONE, ROLE_INPUT, ROLE_PRED, ROLE_EVAL = 0, 1, 2, 3


def rmsprop_step(params, grads, square_avg, step: torch.Tensor, lr: float, warmup: int = 0, alpha: float = 0.99,
                 eps: float = 1e-8, weight_decay: float = 0.0):
    """torch.optim.RMSprop (no momentum, not centred) over flat buffers; the rate is lr * min(step + 1, warmup) / warmup
    (warmup 0: lr) with the step read on the device, which is then incremented."""
    lib.check(lib.load().b200gnn_rmsprop_step_f32(
        _f32(params, "params"), _f32(grads, "grads"), _f32(square_avg, "square_avg"), params.numel(), float(lr), int(warmup),
        float(alpha), float(eps), float(weight_decay), lib.dptr(step, torch.int32, "step"), lib.stream_ptr()), "rmsprop_step_f32")


def teacher_slots(n_items: int) -> int:
    return int(lib.load().b200gnn_teacher_slots(n_items))


def label_inputs(X: Optional[torch.Tensor], col0: int, C: int, row_pos: torch.Tensor, labels: Optional[torch.Tensor],
                 role: torch.Tensor, cnt_part: torch.Tensor, eval: bool, use_labels: bool, mask_rate: float = 0.0,
                 seed: int = 0, offset: int = 0, step_dev: Optional[torch.Tensor] = None, step_mul: int = 0,
                 mask: Optional[torch.Tensor] = None):
    """Roles of every row and (use_labels) the label block X[:, col0:col0+C]: one-hot for the label rows, zero elsewhere;
    cnt_part[teacher_slots(N)] receives the per-CTA counts of loss rows.  mask (uint8 [n_train]) replaces the Philox
    label mask."""
    n = row_pos.numel()
    if role.dtype != torch.uint8 or role.numel() != n or cnt_part.dtype != torch.int32 or cnt_part.numel() != teacher_slots(n):
        raise lib.B200GnnError("label_inputs: role must be uint8[N] and cnt_part int32[teacher_slots(N)]")
    xp, ldx = _rows(X, "X") if C > 0 else (None, 0)
    lib.check(lib.load().b200gnn_label_inputs_f32(
        xp, ldx, col0, C if use_labels else 0, n, lib.dptr(row_pos, torch.int32, "row_pos"),
        lib.dptr(labels, torch.int64, "labels"), int(eval), float(mask_rate), seed, offset,
        lib.dptr(step_dev, torch.int32, "step_dev"), step_mul, lib.dptr(mask, torch.uint8, "mask"), int(use_labels),
        role.data_ptr(), cnt_part.data_ptr(),
        lib.stream_ptr()), "label_inputs_f32")


def label_softmax(logits: torch.Tensor, C: int, out: torch.Tensor, role: Optional[torch.Tensor] = None, role_mask: int = 0):
    """out[r, :C] = softmax(logits[r, :C]) for the rows whose role bit is in role_mask (all rows without roles)."""
    lp, ld = _rows(logits, "logits")
    op, ldo = _rows(out, "out")
    if role is not None and (role.dtype != torch.uint8 or role.numel() != logits.shape[0]):
        raise lib.B200GnnError("label_softmax: role must be uint8[N]")
    lib.check(lib.load().b200gnn_label_softmax_f32(lp, ld, C, logits.shape[0], None if role is None else role.data_ptr(),
                                                   int(role_mask), op, ldo, lib.stream_ptr()), "label_softmax_f32")
    return out


def logce_fwd_bwd(logits: torch.Tensor, C: int, train_idx: torch.Tensor, labels: torch.Tensor, role: torch.Tensor,
                  cnt_part: torch.Tensor, d_logits: torch.Tensor, loss_out: torch.Tensor, acc_out: torch.Tensor,
                  partial: torch.Tensor):
    """The log-CE loss of the role-2 rows (device-counted) with its gradient into d_logits, and the training accuracy."""
    lp, ld = _rows(logits, "logits")
    dp, ldd = _rows(d_logits, "d_logits")
    if partial.dtype != torch.float64 or partial.numel() < 6 * teacher_slots(train_idx.numel()):
        raise lib.B200GnnError("logce: partial must be float64[6 * teacher_slots(n_train)]")
    lib.check(lib.load().b200gnn_logce_fwd_bwd_f32(
        lp, ld, C, lib.dptr(train_idx, torch.int64, "train_idx"), train_idx.numel(), lib.dptr(labels, torch.int64, "labels"),
        role.data_ptr(), lib.dptr(cnt_part, torch.int32, "cnt_part"), cnt_part.numel(), dp, ldd, loss_out.data_ptr(),
        acc_out.data_ptr(), partial.data_ptr(), lib.stream_ptr()), "logce_fwd_bwd_f32")


def split_eval(logits: torch.Tensor, C: int, idx: torch.Tensor, sizes, labels: torch.Tensor, loss_out: torch.Tensor,
               acc_out: torch.Tensor, partial: torch.Tensor):
    """Log-CE loss and first-maximum accuracy of the three splits of idx = [train | val | test] (sizes n0, n1, n2)."""
    lp, ld = _rows(logits, "logits")
    n0, n1, n2 = (int(s) for s in sizes)
    if partial.dtype != torch.float64 or partial.numel() < 6 * teacher_slots(n0 + n1 + n2) or idx.numel() != n0 + n1 + n2:
        raise lib.B200GnnError("split_eval: partial must be float64[6 * teacher_slots(len(idx))]")
    lib.check(lib.load().b200gnn_split_eval_f32(lp, ld, C, lib.dptr(idx, torch.int64, "idx"), n0, n1, n2,
                                                lib.dptr(labels, torch.int64, "labels"), loss_out.data_ptr(), acc_out.data_ptr(),
                                                partial.data_ptr(), lib.stream_ptr()), "split_eval_f32")


def snapshot_if_better(cand: torch.Tensor, best: torch.Tensor, pairs):
    """If cand < best (a NaN never is): copy every (src, dst) pair of contiguous fp32 buffers, then best = cand."""
    args = []
    for s, d in list(pairs) + [(None, None)] * (3 - len(pairs)):
        if s is None:
            args += [None, None, 0]
        else:
            if s.numel() != d.numel():
                raise lib.B200GnnError("snapshot: source and destination sizes differ")
            args += [_f32(s, "src"), _f32(d, "dst"), s.numel()]
    lib.check(lib.load().b200gnn_snapshot_if_better_f32(cand.data_ptr(), best.data_ptr(), *args, lib.stream_ptr()),
              "snapshot_if_better_f32")
