"""numpy restatement of the heterogeneous input kernels (csrc/hetero.cu): the typed gather, the typed scatter whose runs
of equal (type, idx) keys are added in `order`, and the run heads the embedding Adam marks.  Written from the
definitions: the typed gather is RGCN.group_input (mag_pyg/gnn.py:111-124), the scatter is the gradient of that gather
with every run summed left to right.

`tables` and `table_rows` are lists indexed by node type; None (or a type past the end of the list) means "no table"."""
from __future__ import annotations

import numpy as np


def _runs(node_type, local_idx, order):
    """(start, length, key type, key idx) of every run of consecutive equal (type, idx) keys in `order`."""
    order = np.asarray(order, np.int64)
    t = np.asarray(node_type, np.int64)[order]
    j = np.asarray(local_idx, np.int64)[order]
    if order.size == 0:
        e = np.zeros(0, np.int64)
        return e, e, e, e
    new = np.ones(order.size, bool)
    new[1:] = (t[1:] != t[:-1]) | (j[1:] != j[:-1])
    start = np.flatnonzero(new)
    length = np.diff(np.append(start, order.size))
    return start, length, t[start], j[start]


def _has_row(table_rows, t, j):
    return 0 <= t < len(table_rows) and table_rows[t] is not None and 0 <= j < table_rows[t]


def typed_gather(tables, node_type, local_idx, F: int):
    """(out [n, F] float32, positions whose local index is outside their type's table).  Row i is row local_idx[i] of the
    table of node_type[i], and zero when that type has no table or the index is out of range."""
    nt, li = np.asarray(node_type, np.int64), np.asarray(local_idx, np.int64)
    out = np.zeros((nt.size, F), np.float32)
    bad = np.zeros(nt.size, bool)
    for t, tab in enumerate(tables):
        if tab is None:
            continue
        m = nt == t
        ok = m & (li >= 0) & (li < tab.shape[0])
        out[ok] = tab[li[ok]]
        bad |= m & ~ok
    return out, np.flatnonzero(bad)


def typed_scatter_inorder(d_out, node_type, local_idx, order, table_rows):
    """{t: (rows [k] int64, sums [k, F] float32)}: for every run of key (t, j) in `order` whose row exists, the fp32 sum of
    d_out[order[p]] over the run, added one term at a time in `order`, starting from +0.  The positions within a run are
    walked in step and the additions vectorised across the runs still going."""
    d = np.asarray(d_out, np.float32)
    order = np.asarray(order, np.int64)
    start, length, kt, kj = _runs(node_type, local_idx, order)
    keep = np.array([_has_row(table_rows, int(t), int(j)) for t, j in zip(kt, kj)], bool)
    start, length, kt, kj = start[keep], length[keep], kt[keep], kj[keep]
    by_len = np.argsort(-length, kind="stable")             # the runs still going at position q are a prefix of by_len
    start, length, kt, kj = start[by_len], length[by_len], kt[by_len], kj[by_len]
    acc = np.zeros((start.size, d.shape[1]), np.float32)
    neg_len = -length
    for q in range(int(length.max()) if length.size else 0):
        live = int(np.searchsorted(neg_len, -q, side="left"))   # runs with length > q
        acc[:live] += d[order[start[:live] + q]]
    out = {}
    for t in np.unique(kt):
        m = kt == t
        out[int(t)] = (kj[m], acc[m])
    return out


def apply_scatter(tables, sums):
    """Copies of `tables` with the rows of typed_scatter_inorder's result overwritten (the kernel stores each run's sum;
    every other row keeps its bits)."""
    out = [None if t is None else np.array(t, copy=True) for t in tables]
    for t, (rows, vals) in sums.items():
        if out[t] is not None:
            out[t][rows] = vals
    return out


def run_heads(node_type, local_idx, order, table_type: int, rows: int):
    """int32 [rows]: position in `order` of the first node of the run with key (table_type, j), -1 for rows outside the
    batch (the scratch embedding_heads_kernel fills before the embedding Adam sweep)."""
    head = np.full(rows, -1, np.int32)
    start, _, kt, kj = _runs(node_type, local_idx, order)
    m = (kt == table_type) & (kj >= 0) & (kj < rows)
    head[kj[m]] = start[m]
    return head
