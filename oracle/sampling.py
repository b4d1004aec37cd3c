"""CPU restatement (numpy, test infrastructure only) of the reference's mini-batch sampling path (SURVEY.md §8 f4).

The reference drives `torch_geometric.data.GraphSAINTRandomWalkSampler(homo_data, batch_size, walk_length=num_layers,
num_steps, sample_coverage=0)` at mag_pyg/gnn.py:361-366 and consumes its batches at :187-190.  The algorithm itself lives in
third-party packages that are NOT vendored in the reference repository (torch_geometric 1.x `GraphSAINTSampler.__getitem__ /
__collate__`, torch_sparse `random_walk` and `SparseTensor.saint_subgraph`; versions per the reference README: PyG 1.6.x,
torch_sparse 0.6.x), so it is restated here from their published behaviour:

  * roots: `batch_size` node ids drawn uniformly with replacement;
  * walk: `walk_length` steps, each to a uniformly chosen out-neighbour of the current node (adjacency rows = edge_index[0]);
    a node without out-neighbours holds the walker;
  * node set: sorted unique of every visited node; sub-graph: all parent edges with BOTH endpoints in the set, kept in the
    parent's (row, col)-sorted order, endpoints relabelled to positions in the node set, parent edge ids carried along;
  * every parent attribute with first dimension N is indexed by the node set, with first dimension E by the edge ids.

Random streams cannot match upstream's (different generators): "parity unpinned" for the draws themselves — pinned are the
deterministic parts (induced sub-graph, relabelling, attribute slicing) and, because the CUDA kernel's draws are a pure
Philox4x32-10 function of (seed, offset, walker, step), this file replays them bit for bit.
"""
from __future__ import annotations

import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32(seed: int, offset: int, index: np.ndarray) -> np.ndarray:
    """Philox4x32-10 (Salmon et al., SC'11) — same key/counter layout as efficient-gnns_b200/csrc/philox.cuh.
    index: uint64 array -> uint32 array [len(index), 4]."""
    index = np.asarray(index, dtype=np.uint64)
    c0 = (index & np.uint64(MASK)).astype(np.uint64)
    c1 = (index >> np.uint64(32)).astype(np.uint64)
    c2 = np.full_like(c0, offset & MASK)
    c3 = np.full_like(c0, (offset >> 32) & MASK)
    k0, k1 = seed & MASK, (seed >> 32) & MASK
    for _ in range(10):
        p0 = np.uint64(M0) * c0
        p1 = np.uint64(M1) * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & np.uint64(MASK)
        hi1, lo1 = p1 >> np.uint64(32), p1 & np.uint64(MASK)
        n0 = hi1 ^ c1 ^ np.uint64(k0)
        n2 = hi0 ^ c3 ^ np.uint64(k1)
        c0, c1, c2, c3 = n0, lo1, n2, lo0
        k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
    return np.stack([c0, c1, c2, c3], axis=1).astype(np.uint32)


def csr_by_source(edge_index: np.ndarray, num_nodes: int):
    """(rowptr, col, eid): adjacency with rows = edge_index[0], sorted by (row, col), stable; eid = parent edge position."""
    row, col = edge_index[0].astype(np.int64), edge_index[1].astype(np.int64)
    order = np.lexsort((col, row))
    ptr = np.zeros(num_nodes + 1, dtype=np.int64)
    np.add.at(ptr, row + 1, 1)
    return np.cumsum(ptr), col[order], order.astype(np.int64)


def random_walk(rowptr, col, start, walk_length: int, seed: int, offset: int) -> np.ndarray:
    n_w = len(start)
    out = np.empty((n_w, walk_length + 1), dtype=np.int64)
    out[:, 0] = v = np.asarray(start, dtype=np.int64).copy()
    bpw = (walk_length + 3) // 4
    w = np.arange(n_w, dtype=np.uint64)
    r = None
    for s in range(walk_length):
        if s % 4 == 0:
            r = philox4x32(seed, offset, w * np.uint64(bpw) + np.uint64(s // 4))
        u = r[:, s % 4].astype(np.uint64)
        b, e = rowptr[v], rowptr[v + 1]
        deg = (e - b).astype(np.uint64)
        pick = b + ((u * deg) >> np.uint64(32)).astype(np.int64)
        v = np.where(deg > 0, col[np.minimum(pick, len(col) - 1)] if len(col) else v, v)
        out[:, s + 1] = v
    return out


def saint_subgraph(rowptr, col, eid, node_idx):
    """node_idx sorted unique -> (local row, local col, parent edge id), parent CSR order."""
    n = len(rowptr) - 1
    loc = np.full(n, -1, dtype=np.int64)
    loc[node_idx] = np.arange(len(node_idx))
    rows, cols, eids = [], [], []
    for i, v in enumerate(node_idx):
        b, e = rowptr[v], rowptr[v + 1]
        c = loc[col[b:e]]
        keep = c >= 0
        rows.append(np.full(int(keep.sum()), i, dtype=np.int64))
        cols.append(c[keep])
        eids.append(eid[b:e][keep])
    cat = lambda xs: np.concatenate(xs) if xs else np.empty(0, dtype=np.int64)  # noqa: E731
    return cat(rows), cat(cols), cat(eids)
