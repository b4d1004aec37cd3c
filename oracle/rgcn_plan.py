"""numpy restatement of the R-GCN batch plan (efficient_gnns_b200.rgcn.BatchPlan): type grouping, virtual-row forward CSR
for the aggregate-first mean, and its transpose with 1/deg values.  Written from the definition, loop by loop."""
from __future__ import annotations

import numpy as np


class PlanError(ValueError):
    pass


def batch_plan(edge_index, edge_type, node_type, rel_src, rel_dst, n_types):
    src, dst = np.asarray(edge_index[0], np.int64), np.asarray(edge_index[1], np.int64)
    et, nt = np.asarray(edge_type, np.int64).reshape(-1), np.asarray(node_type, np.int64).reshape(-1)
    R, N = len(rel_src), len(nt)
    for e in range(len(et)):
        r = et[e]
        if r < 0 or r >= R or nt[src[e]] != rel_src[r] or nt[dst[e]] != rel_dst[r]:
            raise PlanError(f"edge {e}: type {r} does not match its relation's (source type, destination type)")
    rels_of = [[r for r in range(R) if rel_dst[r] == t] for t in range(n_types)]
    width = [1 + len(x) for x in rels_of]
    # stable grouping by node type
    perm = np.array([i for t in range(n_types) for i in range(N) if nt[i] == t], dtype=np.int64)
    pos = np.empty(N, np.int64)
    pos[perm] = np.arange(N)
    cnt = [int((nt == t).sum()) for t in range(n_types)]
    off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
    vbase = np.concatenate([[0], np.cumsum([cnt[t] * width[t] for t in range(n_types)])]).astype(np.int64)
    V = int(vbase[-1])
    rows = [[] for _ in range(V)]                       # virtual row -> list of internal columns, in insertion order
    for r_int in range(N):
        t = nt[perm[r_int]]
        rows[vbase[t] + (r_int - off[t]) * width[t]].append(r_int)
    for e in range(len(et)):
        t = nt[dst[e]]
        slot = 1 + rels_of[t].index(et[e])
        rows[vbase[t] + (pos[dst[e]] - off[t]) * width[t] + slot].append(pos[src[e]])
    f_rowptr = np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64)
    f_col = np.array([c for x in rows for c in x], dtype=np.int64)
    trows = [[] for _ in range(N)]
    for v in range(V):
        for c in rows[v]:
            trows[c].append(v)
    b_rowptr = np.concatenate([[0], np.cumsum([len(x) for x in trows])]).astype(np.int64)
    b_col = np.array([v for x in trows for v in sorted(x)], dtype=np.int64)
    deg = np.array([len(x) for x in rows], dtype=np.float32)
    b_val = (np.float32(1.0) / deg[b_col]).astype(np.float32) if len(b_col) else np.zeros(0, np.float32)
    return dict(perm=perm, pos=pos, cnt=cnt, off=off, vbase=vbase, V=V, width=width, rels_of=rels_of, f_rowptr=f_rowptr,
                f_col=f_col, b_rowptr=b_rowptr, b_col=b_col, b_val=b_val)


def aggregate(plan, x):
    """Acat arena [V, F] (float64): the mean of each virtual row's columns of x (internal order), 0 for empty rows."""
    V, F = plan["V"], x.shape[1]
    out = np.zeros((V, F))
    rp, col = plan["f_rowptr"], plan["f_col"]
    for v in range(V):
        if rp[v + 1] > rp[v]:
            out[v] = x[col[rp[v]:rp[v + 1]]].mean(0)
    return out
