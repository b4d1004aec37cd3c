"""R-GCN batch plan (efficient_gnns_b200.rgcn.BatchPlan) against its numpy restatement (oracle/rgcn_plan.py), on the CPU:
type grouping, the virtual-row forward CSR of the aggregate-first mean and its 1/deg transpose."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib
from efficient_gnns_b200.rgcn import BatchPlan
from oracle import rgcn_plan as orp

# 3 node types; relations (src type, dst type): 0: 0->0, 1: 1->0, 2: 0->1, 3: 2->1, 4: 1->2, 5: 0->2 (no edges in some cases)
RELS = [(0, 0), (1, 0), (0, 1), (2, 1), (1, 2), (0, 2)]
RS = torch.tensor([s for s, _ in RELS])
RD = torch.tensor([d for _, d in RELS])


def random_batch(seed, n=60, e=300, types=(0, 1, 2), drop_rels=(), dup=True):
    g = np.random.default_rng(seed)
    nt = g.choice(np.array(types), size=n)
    src, dst, et = [], [], []
    for _ in range(e):
        r = int(g.integers(0, len(RELS)))
        s_t, d_t = RELS[r]
        if r in drop_rels or not (nt == s_t).any() or not (nt == d_t).any():
            continue
        src.append(int(g.choice(np.nonzero(nt == s_t)[0]))); dst.append(int(g.choice(np.nonzero(nt == d_t)[0]))); et.append(r)
    if dup and src:                                    # repeat some edges verbatim: the mean counts duplicates
        k = len(src) // 5
        src += src[:k]; dst += dst[:k]; et += et[:k]
    return np.array([src, dst], dtype=np.int64).reshape(2, -1), np.array(et, dtype=np.int64), nt.astype(np.int64)


def check(ei, et, nt):
    got = BatchPlan(torch.from_numpy(ei), torch.from_numpy(et), torch.from_numpy(nt), RS, RD, 3)
    want = orp.batch_plan(ei, et, nt, RS.numpy(), RD.numpy(), 3)
    assert np.array_equal(got.perm.numpy(), want["perm"]) and np.array_equal(got.pos.numpy(), want["pos"])
    assert got.cnt == want["cnt"] and got.off == want["off"].tolist() and got.vbase == want["vbase"].tolist()
    assert got.V == want["V"]
    for k in ("f_rowptr", "f_col", "b_rowptr", "b_col"):
        assert np.array_equal(getattr(got, k).numpy(), want[k]), k
    assert np.array_equal(got.b_val.numpy().view(np.uint32), want["b_val"].view(np.uint32))
    return got, want


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_plan_matches_oracle_with_duplicate_edges(seed):
    ei, et, nt = random_batch(seed)
    _, want = check(ei, et, nt)
    # every slot-0 row is the node itself, so Acat_t starts with X_t; duplicates are counted in the degree
    x = np.random.default_rng(seed).standard_normal((len(nt), 4))
    a = orp.aggregate(want, x[want["perm"]])
    for t in range(3):
        w, n = want["width"][t], want["cnt"][t]
        acat = a[want["vbase"][t]:want["vbase"][t + 1]].reshape(n, w * 4)
        assert np.array_equal(acat[:, :4], x[want["perm"]][want["off"][t]:want["off"][t + 1]])


def test_node_type_missing_from_the_batch():
    ei, et, nt = random_batch(3, types=(0, 2))
    got, want = check(ei, et, nt)
    assert got.cnt[1] == 0 and got.vbase[1] == got.vbase[2]


def test_relation_without_edges_and_destinations_without_in_edges():
    ei, et, nt = random_batch(4, e=40, drop_rels=(3, 5), dup=False)
    got, want = check(ei, et, nt)
    deg = np.diff(want["f_rowptr"])
    for t in range(3):
        w = want["width"][t]
        d = deg[want["vbase"][t]:want["vbase"][t + 1]].reshape(-1, w)
        assert (d[:, 0] == 1).all()                       # slot 0: the node itself
    assert (deg == 0).any()                               # empty slots aggregate to 0 (scatter-mean of nothing)
    t1 = deg[want["vbase"][1]:want["vbase"][2]].reshape(-1, want["width"][1])
    assert (t1[:, 1 + want["rels_of"][1].index(3)] == 0).all()


def test_duplicate_edges_are_not_coalesced():
    nt = np.array([0, 0, 1], dtype=np.int64)
    ei = np.array([[0, 0, 1], [1, 1, 1]], dtype=np.int64)             # relation 0 edge 0->1 twice, plus 1->1
    et = np.array([0, 0, 0], dtype=np.int64)
    got, want = check(ei, et, nt)
    v = want["vbase"][0] + 1 * want["width"][0] + 1                     # node 1, slot of relation 0
    assert want["f_rowptr"][v + 1] - want["f_rowptr"][v] == 3
    x = np.array([[1.0], [2.0], [0.0]])
    assert orp.aggregate(want, x)[v, 0] == pytest.approx((1 + 1 + 2) / 3)


def test_edge_type_with_a_second_type_pair_is_rejected():
    nt = np.array([0, 1, 2], dtype=np.int64)
    ei = np.array([[0, 2], [0, 0]], dtype=np.int64)                     # relation 1 is 1->0, but this edge is 2->0
    et = np.array([0, 1], dtype=np.int64)
    with pytest.raises(lib.B200GnnError, match="fixed"):
        BatchPlan(torch.from_numpy(ei), torch.from_numpy(et), torch.from_numpy(nt), RS, RD, 3)
    with pytest.raises(orp.PlanError):
        orp.batch_plan(ei, et, nt, RS.numpy(), RD.numpy(), 3)
