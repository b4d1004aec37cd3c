"""`torch.ops.b200gnn.*` — the torch binding of the C ABI (SURVEY.md §8b "Operator ABI", item (2)).

The reference reaches its sparse kernels through dispatcher-registered operators
(`torch.ops.torch_sparse.spmm_sum(row?, rowptr, col, value?, colptr?, csr2csc?, mat)`, `spmm_mean(...)`, `ind2ptr`, `ptr2ind`;
called by `SparseTensor.matmul`, mag_pyg/gnn.py:162, and by GCNConv/SAGEConv's `matmul(adj_t, x)`, arxiv_pyg/gnn.py:47,79).
This module registers the same stateless forms under the `b200gnn` namespace with `torch.library`:

    torch.ops.b200gnn.spmm_sum (rowptr, col, value?, mat) -> Tensor      Y = A · mat
    torch.ops.b200gnn.spmm_mean(rowptr, col, value?, mat) -> Tensor      row-mean (A.4: divide by the row's entry count)
    torch.ops.b200gnn.ind2ptr  (ind, M) -> Tensor / ptr2ind(ptr, E) -> Tensor
    torch.ops.b200gnn.split_tf32(w, transpose) -> (hi, lo)
    torch.ops.b200gnn.gemm_tf32x3(a, b_hi, b_lo, bias?) -> Tensor        fp32-faithful wgmma GEMM  a · bᵀ (+bias)

Each has a fake (meta) implementation, so the ops trace under `torch.compile` / FakeTensorMode, and the two SpMMs carry
autograd (gradient w.r.t. `mat`: the same kernel on the transposed matrix, upstream's spmm backward).  int64 indices at the
API as upstream; the engine-side int32 copies, the chunk/hub plans and the transposed view are cached per (rowptr, col,
value) triple (the tensors are kept alive by the cache entry, so a data pointer cannot be recycled under it).
CUDA tensors only — a CPU tensor raises `B200GnnError` (no fallback).  The module path (`SparseTensor.matmul`, the fused
engines) calls the C ABI directly and does not pay the dispatcher; these ops are the binding for functional callers.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import lib, ops
from .sparse import SparseTensor, ind2ptr as _ind2ptr, ptr2ind as _ptr2ind

_CACHE: "OrderedDict[tuple, SparseTensor]" = OrderedDict()
_CACHE_MAX = 16


def _adj(rowptr: Tensor, col: Tensor, value: Optional[Tensor], n_cols: int) -> SparseTensor:
    key = (rowptr.data_ptr(), col.data_ptr(), None if value is None else value.data_ptr(), rowptr._version, col._version,
           None if value is None else value._version, rowptr.numel(), col.numel(), n_cols)
    adj = _CACHE.get(key)
    if adj is None:
        if not (rowptr.is_cuda and col.is_cuda):
            raise lib.B200GnnError(f"b200gnn operators need CUDA tensors (got {col.device}); there is no CPU fallback")
        adj = SparseTensor(rowptr=rowptr, col=col, value=value, sparse_sizes=(rowptr.numel() - 1, n_cols), is_sorted=True)
        adj._keepalive = (rowptr, col, value)
        _CACHE[key] = adj
        while len(_CACHE) > _CACHE_MAX:
            _CACHE.popitem(last=False)
    else:
        _CACHE.move_to_end(key)
    return adj


def _spmm(rowptr, col, value, mat, reduce):
    adj = _adj(rowptr, col, value, mat.size(0))
    st = adj.storage
    g = st.engine_csr() if value is not None else st.engine_csr_unweighted()
    return ops.spmm_csr(g, mat.contiguous(), reduce)


def _spmm_bwd(rowptr, col, value, grad, n_cols, reduce):
    st = _adj(rowptr, col, value, n_cols).storage
    if reduce == "mean":
        gt = st.engine_csc("mean" if value is None else "mean_value")
    else:
        gt = st.engine_csc("value")
    return ops.spmm_csr(gt, grad.contiguous(), "sum")


@torch.library.custom_op("b200gnn::spmm_sum", mutates_args=())
def spmm_sum(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tensor:
    return _spmm(rowptr, col, value, mat, "sum")


@torch.library.custom_op("b200gnn::spmm_mean", mutates_args=())
def spmm_mean(rowptr: Tensor, col: Tensor, value: Optional[Tensor], mat: Tensor) -> Tensor:
    return _spmm(rowptr, col, value, mat, "mean")


@torch.library.custom_op("b200gnn::spmm_transposed", mutates_args=())
def spmm_transposed(rowptr: Tensor, col: Tensor, value: Optional[Tensor], grad: Tensor, n_cols: int, mean: bool) -> Tensor:
    """d mat of spmm_sum / spmm_mean: Aᵀ · grad (mean: rows of A pre-scaled by 1 / count)."""
    return _spmm_bwd(rowptr, col, value, grad, n_cols, "mean" if mean else "sum")


def _fake_spmm(rowptr, col, value, mat):
    return mat.new_empty(rowptr.numel() - 1, mat.size(1))


spmm_sum.register_fake(_fake_spmm)
spmm_mean.register_fake(_fake_spmm)


@spmm_transposed.register_fake
def _(rowptr, col, value, grad, n_cols, mean):
    return grad.new_empty(n_cols, grad.size(1))


def _setup(ctx, inputs, output):
    rowptr, col, value, mat = inputs
    ctx.save_for_backward(rowptr, col, *([] if value is None else [value]))
    ctx.has_value, ctx.n_cols = value is not None, mat.size(0)


def _make_bwd(mean: bool):
    def bwd(ctx, grad):
        saved = ctx.saved_tensors
        value = saved[2] if ctx.has_value else None
        return None, None, None, torch.ops.b200gnn.spmm_transposed(saved[0], saved[1], value, grad, ctx.n_cols, mean)
    return bwd


spmm_sum.register_autograd(_make_bwd(False), setup_context=_setup)
spmm_mean.register_autograd(_make_bwd(True), setup_context=_setup)


@torch.library.custom_op("b200gnn::ind2ptr", mutates_args=())
def ind2ptr(ind: Tensor, M: int) -> Tensor:
    return _ind2ptr(ind, M)


@ind2ptr.register_fake
def _(ind, M):
    return ind.new_empty(M + 1)


@torch.library.custom_op("b200gnn::ptr2ind", mutates_args=())
def ptr2ind(ptr: Tensor, E: int) -> Tensor:
    return _ptr2ind(ptr, E)


@ptr2ind.register_fake
def _(ptr, E):
    return ptr.new_empty(E)


@torch.library.custom_op("b200gnn::split_tf32", mutates_args=())
def split_tf32(w: Tensor, transpose: bool) -> Tuple[Tensor, Tensor]:
    hi, lo = ops.split_tf32(w.contiguous(), transpose=transpose)
    return hi, lo


@split_tf32.register_fake
def _(w, transpose):
    shape = (w.size(1), w.size(0)) if transpose else tuple(w.shape)
    return w.new_empty(shape), w.new_empty(shape)


@torch.library.custom_op("b200gnn::gemm_tf32x3", mutates_args=())
def gemm_tf32x3(a: Tensor, b_hi: Tensor, b_lo: Tensor, bias: Optional[Tensor]) -> Tensor:
    return ops.gemm_tf32x3(a.contiguous(), b_hi, b_lo, bias)


@gemm_tf32x3.register_fake
def _(a, b_hi, b_lo, bias):
    return a.new_empty(a.size(0), b_hi.size(0))


OPS = ("spmm_sum", "spmm_mean", "spmm_transposed", "ind2ptr", "ptr2ind", "split_tf32", "gemm_tf32x3")
