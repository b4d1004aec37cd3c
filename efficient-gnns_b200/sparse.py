"""Sparse adjacency containers.

``SparseTensor`` mirrors the slice of ``torch_sparse.SparseTensor`` the reference
touches (SURVEY.md §8b): construction from ``row``/``col`` (arxiv_pyg/gnn.py:236-237
via ``T.ToSparseTensor``, mag_pyg/gnn.py:151), ``to_symmetric`` (arxiv_pyg/gnn.py:240),
``coo`` (:248), ``matmul(x, reduce=)`` (mag_pyg/gnn.py:162), ``.to(device)``.
API-side indices are int64 like upstream; ``CsrGraph`` is the engine-side view
(int32, plus the hub plan the SpMM kernels need), built lazily and cached the way
upstream's SparseStorage caches rowptr / colptr / csr2csc / rowcount.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import Optional, Tuple

import torch

from . import lib

HUB_THRESHOLD = 256   # rows with more non-zeros than this are split across CTAs
HUB_SEG_LEN = 256     # non-zeros per hub segment (one CTA each)
CHUNK_NNZ = 128       # non-zeros per warp-sized chunk of consecutive rows
CHUNK_ROW_COST = 4    # per-row cost (in non-zero equivalents) when cutting chunks


def _narrow_i32(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.numel() and int(t.max()) >= 2 ** 31 - 1:
        raise lib.B200GnnError(f"{what}: index >= 2^31-1 cannot be narrowed to the engine's int32")
    return t.to(torch.int32).contiguous()


@dataclass
class CsrGraph:
    """Engine-side CSR matrix: int32 indices, optional fp32 values, hub plan."""
    rowptr: torch.Tensor
    col: torch.Tensor
    val: Optional[torch.Tensor]
    n_rows: int
    n_cols: int
    hub_threshold: int = 0
    seg_len: int = 0
    chunk_nnz: int = 0
    row_cost: int = 0
    chunk_rowptr: Optional[torch.Tensor] = None
    n_chunks: int = 0
    hub_rows: Optional[torch.Tensor] = None
    hub_segptr: Optional[torch.Tensor] = None
    n_hub: int = 0
    n_seg: int = 0
    _ws: dict = field(default_factory=dict)

    @property
    def nnz(self) -> int:
        return int(self.col.numel())

    @property
    def device(self):
        return self.rowptr.device

    def build_plan(self, hub_threshold: Optional[int] = None, seg_len: Optional[int] = None,
                   chunk_nnz: Optional[int] = None, row_cost: Optional[int] = None) -> "CsrGraph":
        """Chunk plan (load balance) + hub plan (row splitting): C-ABI calls with one host read of the hub
        counts in between; one-off per graph, cached with the storage."""
        self.hub_threshold = HUB_THRESHOLD if hub_threshold is None else hub_threshold
        self.seg_len = HUB_SEG_LEN if seg_len is None else seg_len
        self.chunk_nnz = CHUNK_NNZ if chunk_nnz is None else chunk_nnz
        self.row_cost = CHUNK_ROW_COST if row_cost is None else row_cost
        self._ws.clear()
        L = lib.load()
        st = lib.stream_ptr()
        self.n_chunks = int(L.b200gnn_csr_chunk_count(self.n_rows, self.nnz, self.chunk_nnz, self.row_cost))
        self.chunk_rowptr = torch.zeros(self.n_chunks + 1, dtype=torch.int32, device=self.device)
        if self.n_rows > 0:
            lib.check(L.b200gnn_csr_chunk_plan(lib.dptr(self.rowptr, torch.int32, "rowptr"), self.n_rows, self.nnz,
                                               self.chunk_nnz, self.row_cost, self.chunk_rowptr.data_ptr(), st),
                      "csr_chunk_plan")
        counts = torch.zeros(2, dtype=torch.int32, device=self.device)
        lib.check(L.b200gnn_csr_hub_count(lib.dptr(self.rowptr, torch.int32, "rowptr"), self.n_rows,
                                          self.hub_threshold, self.seg_len, counts.data_ptr(), st), "csr_hub_count")
        n_hub, n_seg = (int(v) for v in counts.tolist())
        self.hub_segptr = torch.zeros(n_hub + 1, dtype=torch.int32, device=self.device)
        self.hub_rows = torch.zeros(max(n_hub, 1), dtype=torch.int32, device=self.device)
        lib.check(L.b200gnn_csr_hub_fill(self.rowptr.data_ptr(), self.n_rows, self.hub_threshold, self.seg_len,
                                         self.hub_rows.data_ptr(), self.hub_segptr.data_ptr(), n_hub, st),
                  "csr_hub_fill")
        self.n_hub, self.n_seg = n_hub, n_seg
        return self

    def hub_workspace(self, K: int) -> Optional[torch.Tensor]:
        """Scratch for hub-segment partials, cached per feature width (stream-ordered reuse)."""
        if self.n_seg == 0:
            return None
        ws = self._ws.get(K)
        if ws is None:
            ws = torch.empty(self.n_seg * K, dtype=torch.float32, device=self.device)
            self._ws[K] = ws
        return ws


def csr_graph_from(rowptr64: torch.Tensor, col64: torch.Tensor, val: Optional[torch.Tensor],
                   n_rows: int, n_cols: int) -> CsrGraph:
    if not rowptr64.is_cuda:
        raise lib.B200GnnError("engine graphs live on a CUDA device; there is no CPU fallback")
    g = CsrGraph(_narrow_i32(rowptr64, "rowptr"), _narrow_i32(col64, "col"),
                 None if val is None else val.to(torch.float32).contiguous(), n_rows, n_cols)
    return g.build_plan()


def ind2ptr(ind: torch.Tensor, size: int) -> torch.Tensor:
    """Sorted row indices -> rowptr (upstream torch_sparse ind2ptr, K6)."""
    counts = torch.bincount(ind, minlength=size) if ind.numel() else torch.zeros(size, dtype=torch.long, device=ind.device)
    ptr = torch.zeros(size + 1, dtype=torch.long, device=ind.device)
    torch.cumsum(counts, 0, out=ptr[1:])
    return ptr


def ptr2ind(ptr: torch.Tensor, nnz: int) -> torch.Tensor:
    counts = ptr[1:] - ptr[:-1]
    return torch.repeat_interleave(torch.arange(counts.numel(), device=ptr.device), counts, output_size=nnz)


# ----------------------------------------------------------------------------- device graph ingestion (csrc/graph_prep.cu)
def _on_engine_device(*ts) -> bool:
    return all(t is not None and t.is_cuda for t in ts)


def device_argsort(major: torch.Tensor, minor: torch.Tensor, major_size: int, minor_size: int) -> torch.Tensor:
    """Stable argsort of major*minor_size + minor: the hand-written radix sort on CUDA tensors (int64 out, same
    permutation as torch.argsort(stable=True)); torch on CPU tensors (host-side logic and its tests).  The CPU order is two
    stable passes, minor then major, so that key ranges of 2^63 and above (which the radix sort accepts) do not overflow."""
    n = int(major.numel())
    if not _on_engine_device(major, minor):
        p = torch.argsort(minor, stable=True)
        return p[torch.argsort(major[p], stable=True)]
    if n == 0:
        return torch.empty(0, dtype=torch.long, device=major.device)
    if n >= 2 ** 31 - 1 or float(major_size) * float(minor_size) >= 1.8e19:
        raise lib.B200GnnError(f"device_argsort: {n} keys in a range of {major_size} x {minor_size}: the radix sort takes fewer "
                               "than 2^31-1 keys and a key range below 1.8e19")
    L = lib.load()
    ws = torch.empty(int(L.b200gnn_graph_sort_workspace_bytes(n)), dtype=torch.uint8, device=major.device)
    perm = torch.empty(n, dtype=torch.int32, device=major.device)
    ma, mi = major.to(torch.long).contiguous(), minor.to(torch.long).contiguous()     # the kernel reads int64
    lib.check(L.b200gnn_graph_argsort_i64(ma.data_ptr(), mi.data_ptr(), n, int(major_size), int(minor_size), perm.data_ptr(),
                                          ws.data_ptr(), lib.stream_ptr()), "graph_argsort_i64")
    return perm.long()


def device_coalesce(row: torch.Tensor, col: torch.Tensor, n_rows: int, n_cols: int):
    """(row, col, rowptr, src) of the row-sorted duplicate-free matrix (src = input index of each kept entry)."""
    n = int(row.numel())
    L = lib.load()
    dev = row.device
    ws = torch.empty(int(L.b200gnn_graph_sort_workspace_bytes(n)), dtype=torch.uint8, device=dev)
    out_row, out_col = torch.empty(n, dtype=torch.long, device=dev), torch.empty(n, dtype=torch.long, device=dev)
    src = torch.empty(n, dtype=torch.int32, device=dev)
    rowptr = torch.empty(n_rows + 1, dtype=torch.long, device=dev)
    nnz = torch.zeros(1, dtype=torch.long, device=dev)
    r, c = row.to(torch.long).contiguous(), col.to(torch.long).contiguous()     # the kernel reads int64
    lib.check(L.b200gnn_graph_coalesce_i64(r.data_ptr(), c.data_ptr(), n, int(n_rows), int(n_cols), out_row.data_ptr(),
                                           out_col.data_ptr(), src.data_ptr(), rowptr.data_ptr(), nnz.data_ptr(), ws.data_ptr(),
                                           lib.stream_ptr()), "graph_coalesce_i64")
    k = int(nnz.item())                       # one host read per graph (set-up time)
    return out_row[:k], out_col[:k], rowptr, src[:k].long()


class SparseStorage:
    """row-sorted COO/CSR storage with lazily cached derived arrays (shared by reference between views)."""

    def __init__(self, row, rowptr, col, value, sparse_sizes, is_sorted):
        M, N = sparse_sizes
        if row is None:
            row = ptr2ind(rowptr, col.numel())
        if not is_sorted and row.numel() > 1:
            key = row * N + col
            if not bool((key[1:] >= key[:-1]).all()):
                perm = device_argsort(row, col, M, N)
                row, col = row[perm], col[perm]
                value = None if value is None else value[perm]
                rowptr = None
        self._row, self._col, self._value = row, col, value
        self._rowptr = rowptr
        self._sizes = (int(M), int(N))
        self._colptr = None
        self._csr2csc = None
        self._rowcount = None
        self._engine = {}

    # --- upstream-named accessors
    def row(self): return self._row
    def col(self): return self._col
    def value(self): return self._value
    def sparse_sizes(self): return self._sizes

    def rowptr(self):
        if self._rowptr is None:
            self._rowptr = ind2ptr(self._row, self._sizes[0])
        return self._rowptr

    def rowcount(self):
        if self._rowcount is None:
            p = self.rowptr()
            self._rowcount = p[1:] - p[:-1]
        return self._rowcount

    def csr2csc(self):
        if self._csr2csc is None:
            self._csr2csc = device_argsort(self._col, self._row, self._sizes[1], self._sizes[0])
        return self._csr2csc

    def colptr(self):
        if self._colptr is None:
            self._colptr = ind2ptr(self._col[self.csr2csc()], self._sizes[1])
        return self._colptr

    # --- engine views
    def engine_csr(self) -> CsrGraph:
        g = self._engine.get("csr")
        if g is None:
            g = csr_graph_from(self.rowptr(), self._col, self._value, *self._sizes)
            self._engine["csr"] = g
        return g

    def engine_csr_unweighted(self) -> CsrGraph:
        g = self._engine.get("csr_u")
        if g is None:
            base = self.engine_csr()
            g = replace(base, val=None, _ws={})
            self._engine["csr_u"] = g
        return g

    def engine_csc(self, mode: str) -> CsrGraph:
        """Transpose as CSR, for the SpMM backward (upstream: colptr, row[csr2csc], value[csr2csc]).
        mode 'value': carries value[csr2csc] (None if unweighted); 'mean': weights 1/max(rowcount[row],1);
        'mean_value': value[csr2csc]/max(rowcount[row],1) (mean of a WEIGHTED matrix: forward is sum(val*x)/rowcount)."""
        key = "csc_" + mode
        g = self._engine.get(key)
        if g is None:
            perm = self.csr2csc()
            row_t = self._row[perm]
            if mode == "value":
                val = None if self._value is None else self._value[perm]
            elif mode == "mean":
                val = (1.0 / self.rowcount().clamp(min=1).to(torch.float32))[row_t]
            elif mode == "mean_value":
                val = self._value[perm].to(torch.float32) / self.rowcount().clamp(min=1).to(torch.float32)[row_t]
            else:
                raise ValueError(mode)
            g = csr_graph_from(self.colptr(), row_t, val, self._sizes[1], self._sizes[0])
            self._engine[key] = g
        return g


class SparseTensor:
    def __init__(self, row: Optional[torch.Tensor] = None, rowptr: Optional[torch.Tensor] = None,
                 col: Optional[torch.Tensor] = None, value: Optional[torch.Tensor] = None,
                 sparse_sizes: Optional[Tuple[int, int]] = None, is_sorted: bool = False, _storage=None):
        if _storage is not None:
            self.storage = _storage
            return
        assert col is not None and (row is not None or rowptr is not None)
        if sparse_sizes is None or sparse_sizes[0] is None or sparse_sizes[1] is None:
            # upstream infers (max(row)+1, max(col)+1)
            M = (int(row.max()) + 1 if row is not None and row.numel() else (rowptr.numel() - 1 if rowptr is not None else 0))
            N = int(col.max()) + 1 if col.numel() else 0
            if sparse_sizes is not None:
                M = sparse_sizes[0] if sparse_sizes[0] is not None else M
                N = sparse_sizes[1] if sparse_sizes[1] is not None else N
            sparse_sizes = (M, N)
        self.storage = SparseStorage(row, rowptr, col, value, sparse_sizes, is_sorted)

    @classmethod
    def from_edge_index(cls, edge_index, edge_attr=None, sparse_sizes=None, is_sorted=False):
        return cls(row=edge_index[0], col=edge_index[1], value=edge_attr, sparse_sizes=sparse_sizes, is_sorted=is_sorted)

    # --- views
    def coo(self):
        s = self.storage
        return s.row(), s.col(), s.value()

    def csr(self):
        s = self.storage
        return s.rowptr(), s.col(), s.value()

    def sparse_sizes(self): return self.storage.sparse_sizes()
    def sparse_size(self, dim): return self.storage.sparse_sizes()[dim]
    def size(self, dim): return self.storage.sparse_sizes()[dim]
    def sizes(self): return list(self.storage.sparse_sizes())
    def nnz(self): return int(self.storage.col().numel())
    def has_value(self): return self.storage.value() is not None
    @property
    def device(self): return self.storage.col().device
    def is_cuda(self): return self.storage.col().is_cuda

    def to(self, device, *args, **kwargs):
        s = self.storage
        mv = lambda t: None if t is None else t.to(device)
        return SparseTensor(row=mv(s.row()), rowptr=mv(s._rowptr), col=mv(s.col()), value=mv(s.value()),
                            sparse_sizes=s.sparse_sizes(), is_sorted=True)

    def cuda(self): return self.to("cuda")
    def cpu(self): return self.to("cpu")

    def set_value(self, value, layout=None):
        s = self.storage
        st = SparseStorage(s.row(), s._rowptr, s.col(), value, s.sparse_sizes(), True)
        st._colptr, st._csr2csc, st._rowcount = s._colptr, s._csr2csc, s._rowcount
        if value is None and "csr" in s._engine:  # share the int32 structure + hub plan
            st._engine["csr_u"] = s.engine_csr_unweighted()
        return SparseTensor(_storage=st)

    def fill_value(self, v: float, dtype=torch.float32):
        return self.set_value(torch.full((self.nnz(),), v, dtype=dtype, device=self.device))

    def sum(self, dim: int):
        assert dim == 1, "only row sums are used by the reference path (gcn_norm)"
        s = self.storage
        if s.value() is None:
            return s.rowcount().to(torch.float32)
        out = torch.zeros(s.sparse_sizes()[0], dtype=s.value().dtype, device=self.device)
        return out.index_add_(0, s.row(), s.value())

    def t(self):
        s = self.storage
        perm = s.csr2csc()
        val = None if s.value() is None else s.value()[perm]
        M, N = s.sparse_sizes()
        return SparseTensor(row=s.col()[perm], rowptr=s.colptr(), col=s.row()[perm], value=val,
                            sparse_sizes=(N, M), is_sorted=True)

    def coalesce(self, reduce: str = "sum"):
        """Drop duplicate (row,col) pairs (values, if any, summed) — storage is already sorted."""
        s = self.storage
        row, col, val = s.row(), s.col(), s.value()
        if row.numel() <= 1:
            return self
        key = row * s.sparse_sizes()[1] + col
        keep = torch.ones_like(key, dtype=torch.bool)
        keep[1:] = key[1:] != key[:-1]
        if bool(keep.all()):
            return self
        if val is not None:
            seg = torch.cumsum(keep.to(torch.long), 0) - 1
            val = torch.zeros(int(seg[-1]) + 1, dtype=val.dtype, device=val.device).index_add_(0, seg, val)
        return SparseTensor(row=row[keep], col=col[keep], value=val, sparse_sizes=s.sparse_sizes(), is_sorted=True)

    def to_symmetric(self, reduce: str = "sum"):
        """upstream: cat([row,col]), cat([col,row]) -> sort -> coalesce (SURVEY Appendix A.1)."""
        row, col, val = self.coo()
        M, N = self.sparse_sizes()
        n = max(M, N)
        r2, c2 = torch.cat([row, col]), torch.cat([col, row])
        if val is None and _on_engine_device(r2) and 0 < r2.numel() < 2 ** 31 - 1:
            # sort + duplicate removal + row pointers in one pass of the ingestion kernels (csrc/graph_prep.cu)
            ro, co, rowptr, _ = device_coalesce(r2, c2, n, n)
            return SparseTensor(row=ro, rowptr=rowptr, col=co, sparse_sizes=(n, n), is_sorted=True)
        v2 = None if val is None else torch.cat([val, val])
        return SparseTensor(row=r2, col=c2, value=v2, sparse_sizes=(n, n), is_sorted=False).coalesce(reduce)

    def fill_diag(self, fill_value: float):
        """Set the main diagonal to ``fill_value`` (existing diagonal entries replaced, missing ones added)."""
        row, col, val = self.coo()
        M, N = self.sparse_sizes()
        n = min(M, N)
        off = row != col
        diag = torch.arange(n, device=row.device)
        r2 = torch.cat([row[off], diag])
        c2 = torch.cat([col[off], diag])
        if val is None:
            v2 = None
        else:
            v2 = torch.cat([val[off], torch.full((n,), fill_value, dtype=val.dtype, device=val.device)])
        return SparseTensor(row=r2, col=c2, value=v2, sparse_sizes=(M, N), is_sorted=False)

    def matmul(self, other: torch.Tensor, reduce: str = "sum"):
        from .ops import matmul
        return matmul(self, other, reduce)

    def __matmul__(self, other):
        return self.matmul(other, "sum")

    def spmm(self, other, reduce: str = "sum"):
        return self.matmul(other, reduce)

    def __repr__(self):
        return f"SparseTensor(sizes={self.sparse_sizes()}, nnz={self.nnz()}, device={self.device})"
