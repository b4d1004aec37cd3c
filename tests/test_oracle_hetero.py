"""The CPU restatement of the heterogeneous input kernels (oracle/hetero.py) against plain loops: the in-order sum that
tests/test_hetero_kernels_gpu.py holds the typed scatter and the embedding Adam to, the run heads, the typed gather."""
import numpy as np

from oracle import hetero as oh


def _keys(rng, n, n_types, rows):
    nt = rng.integers(0, n_types, n)
    li = rng.integers(0, rows, n)
    return nt, li


def _order(nt, li):
    return np.lexsort((li, nt))                 # stable: ties keep their position, like torch.argsort(stable=True)


def test_in_order_sum_is_the_left_to_right_loop_bit_for_bit():
    rng = np.random.default_rng(0)
    n, F = 3000, 7
    nt, li = _keys(rng, n, 3, 40)
    nt[:400], li[:400] = 1, 5                   # one 400-term run
    d = (rng.standard_normal((n, F)) * np.exp(rng.uniform(-8, 8, (n, 1)))).astype(np.float32)
    order = _order(nt, li)
    got = oh.typed_scatter_inorder(d, nt, li, order, [40, 40, 40])
    want = {}
    for p in order:
        k = (int(nt[p]), int(li[p]))
        acc = want.get(k, np.zeros(F, np.float32))
        want[k] = np.float32(acc + d[p])        # one fp32 rounding per term, in order
    assert sum(len(r) for r, _ in got.values()) == len(want)
    for t, (rows, sums) in got.items():
        for j, s in zip(rows, sums):
            assert np.array_equal(s.view(np.uint32), want[(t, int(j))].view(np.uint32)), (t, j)
    # the order matters: summing the 400-term run backwards gives other bits for this data
    rev = np.zeros(F, np.float32)
    for p in order[::-1]:
        if nt[p] == 1 and li[p] == 5:
            rev = np.float32(rev + d[p])
    rows, sums = got[1]
    assert not np.array_equal(sums[list(rows).index(5)], rev)


def test_small_integer_sums_equal_add_at_in_fp64():
    rng = np.random.default_rng(1)
    n, F = 5000, 5
    nt, li = _keys(rng, n, 4, 60)
    d = rng.integers(-20, 21, (n, F)).astype(np.float32)
    table_rows = [60, None, 60, 30]              # type 1 has no table; type 3's rows past 30 do not exist
    got = oh.apply_scatter([np.zeros((r, F), np.float32) if r else None for r in table_rows],
                           oh.typed_scatter_inorder(d, nt, li, _order(nt, li), table_rows))
    for t, r in enumerate(table_rows):
        if r is None:
            assert got[t] is None
            continue
        m = (nt == t) & (li < r)
        want = np.zeros((r, F))
        np.add.at(want, li[m], d[m].astype(np.float64))
        assert np.array_equal(got[t], want), t


def test_same_index_under_two_types_stays_two_runs():
    nt = np.array([0, 1, 0, 1, 2])
    li = np.array([3, 3, 3, 3, 3])
    d = np.arange(10, dtype=np.float32).reshape(5, 2)
    got = oh.typed_scatter_inorder(d, nt, li, _order(nt, li), [4, 4, 4])
    assert np.array_equal(got[0][0], [3]) and np.array_equal(got[0][1], [[0 + 4, 1 + 5]])
    assert np.array_equal(got[1][0], [3]) and np.array_equal(got[1][1], [[2 + 6, 3 + 7]])
    assert np.array_equal(got[2][1], [[8, 9]])
    heads = [oh.run_heads(nt, li, _order(nt, li), t, 4) for t in range(3)]
    assert [h.tolist() for h in heads] == [[-1, -1, -1, 0], [-1, -1, -1, 2], [-1, -1, -1, 4]]


def test_run_heads_are_the_first_position_of_each_run():
    rng = np.random.default_rng(2)
    nt, li = _keys(rng, 2000, 3, 300)
    li[nt == 2] -= 50                            # negative indices belong to no row
    order = _order(nt, li)
    for t, rows in ((0, 300), (1, 200), (2, 300)):
        want = np.full(rows, -1, np.int32)
        for p in range(len(order) - 1, -1, -1):  # the lowest position of each key wins
            i = order[p]
            if nt[i] == t and 0 <= li[i] < rows:
                want[li[i]] = p
        assert np.array_equal(oh.run_heads(nt, li, order, t, rows), want), t


def test_typed_gather_copies_rows_and_reports_bad_indices():
    rng = np.random.default_rng(3)
    F = 6
    tables = [rng.standard_normal((10, F)).astype(np.float32), None, rng.standard_normal((4, F)).astype(np.float32),
              np.zeros((0, F), np.float32)]
    nt = np.array([0, 1, 2, 5, -1, 0, 2, 3, 0])
    li = np.array([9, 7, 0, 1, 1, 10, -1, 0, 0])
    out, bad = oh.typed_gather(tables, nt, li, F)
    assert bad.tolist() == [5, 6, 7]
    for i in range(len(nt)):
        t, j = nt[i], li[i]
        ok = 0 <= t < len(tables) and tables[t] is not None and 0 <= j < len(tables[t])
        assert np.array_equal(out[i], tables[t][j] if ok else np.zeros(F, np.float32)), i
