"""Contract of the heterogeneous input kernels of the R-GCN step (csrc/hetero.cu, ops.typed_gather / typed_scatter /
embedding_adam, nn.group_input), the ReLU/dropout backward it runs between layers, and the batch plan's aggregation.

* The typed gather is a copy: every row must equal oracle/hetero.py's bit for bit, at widths on both sides of the 32-lane
  chunks, with an output pitch wider than F inside a buffer of NaN canaries, with 1, 4 and 16 tables (null tables,
  zero-row tables, node types past the last table) and at the ogbn-mag table sizes.  An index outside its table gives a
  zero row and sets the error flag; the wrappers turn the flag into B200GnnError.
* The typed scatter adds each run of equal (type, idx) keys one term at a time in ``order``.  On random non-dyadic data
  another order gives other bits, so comparing bit for bit with the in-order oracle (``typed_scatter_inorder``) is what
  pins the order.  Gradient tables start as canaries: rows outside the batch must keep their bits.
* The embedding Adam must be bit-identical to that scatter into a zeroed dense gradient followed by ``ops.adam_step``
  (pinned against torch.optim elsewhere).  The Adam arithmetic itself is not restated here; what is checked is which
  rows update, with which gradient, and that the ``head`` scratch and the step counter are left as the docstring says.
  The moments start non-zero, so a row that is skipped instead of taking its zero-gradient update is visible.
* The batch plan's layer-0 arena must equal, bit for bit, the per-relation scatter-mean of the batch computed in fp64
  from its edge list (small-integer rows make every sum exact, the argument at the top of test_sparse_exact_gpu.py), and
  the transposed SpMM must stay within a derived elementwise bound of the fp64 adjoint of that mean.
* The wrappers refuse tables and index vectors that the kernels would misread.  Every refused case is built so that the
  launch an unchecked wrapper would make still reads and writes only allocated memory."""
import ctypes as C
import zlib

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, nn as bnn, ops, sampling, synthetic
from efficient_gnns_b200.graphdata import Data
from efficient_gnns_b200.rgcn import RGCNTrainer
from efficient_gnns_b200.sparse import device_argsort
from oracle import hetero as oh
from test_rgcn_train_gpu import NODES, batches, small_mag
from test_sparse_exact_gpu import CANARY, NAN_BITS, U, Boxed, _assert_exact, _gamma

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

DEV = "cuda"
MAG = synthetic.MAG_NODES


def _seed(*key) -> int:
    return zlib.crc32(repr(key).encode())


def _rng(*key) -> np.random.Generator:
    return np.random.default_rng(_seed(*key))


def _bits(x: torch.Tensor) -> np.ndarray:
    return x.detach().contiguous().cpu().numpy().view(np.uint32)


def _nonuniform(rng, n, F) -> np.ndarray:
    """Random fp32 rows whose magnitudes span 2^±12: sums of them round differently in another order."""
    return (rng.standard_normal((n, F)) * np.exp2(rng.integers(-12, 13, (n, 1)))).astype(np.float32)


class Padded:
    """A contiguous [rows, F] table inside a flat buffer of `fill` bits (NaN canaries by default), so that a read of row -1
    or row `rows` returns NaN and a stray write is visible."""

    PAD = 64

    def __init__(self, rows: int, F: int, fill: int = CANARY):
        self.flat = torch.full((rows * F + 2 * self.PAD,), fill, dtype=torch.int32, device=DEV).view(torch.float32)
        self.t = self.flat[self.PAD:self.PAD + rows * F].view(rows, F)


def _table_arrays(tables, rows):
    """Host arrays for the C ABI: a null pointer for None; `rows` is passed as given (also for null tables)."""
    ptrs = (C.c_void_p * len(tables))(*[None if t is None else t.data_ptr() for t in tables])
    return ptrs, (C.c_int64 * len(rows))(*rows)


def _gather_abi(tables, rows, nt, li, F, out, ldo):
    err = torch.zeros(1, dtype=torch.int32, device=DEV)
    ptrs, rws = _table_arrays(tables, rows)
    rc = lib.load().b200gnn_typed_gather_f32(ptrs, rws, len(tables), nt.data_ptr(), li.data_ptr(), nt.numel(), F,
                                             out.data_ptr(), ldo, err.data_ptr(), lib.stream_ptr())
    assert rc == lib.OK, rc
    return int(err.item())


def _scatter_abi(d, ldd, nt, li, order, F, tables, rows):
    ptrs, rws = _table_arrays(tables, rows)
    rc = lib.load().b200gnn_typed_scatter_f32(d.data_ptr(), ldd, nt.data_ptr(), li.data_ptr(), order.data_ptr(), nt.numel(),
                                              F, ptrs, rws, len(tables), lib.stream_ptr())
    assert rc == lib.OK, rc


def _cuda(a, dtype=torch.int64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV, dtype)


# ================================================================================================================ gather
GATHER_F = [1, 4, 31, 32, 33, 128, 129]
# rows per node type; None = no table (null pointer), 0 = a zero-row table (a real pointer)
LAYOUTS = {1: [300], 4: [300, None, 7, 1000],
           16: [50, None, 1, 2000, 0, 33, None, 32, 31, 700, 5, None, 129, 64, 3, 900]}


def _gather_case(F, n_tables, n=3000):
    """Tables (inside NaN pads), their host rows, and (node_type, local_idx) with every index inside its table: node types
    in [-2, n_tables + 3), rows 0 and rows - 1 of every table hit, arbitrary indices for the types without rows."""
    rng = _rng("gather", F, n_tables)
    layout = LAYOUTS[n_tables]
    pads, tables, rows, host = [], [], [], []
    for r in layout:
        if r is None:
            tables.append(None); rows.append(1000); host.append(None)          # rows of a null table are ignored
            continue
        p = Padded(r, F)
        p.t.copy_(_cuda(_nonuniform(rng, r, F), torch.float32))
        pads.append(p); tables.append(p.t); rows.append(r); host.append(p.t.cpu().numpy())
    nt = rng.integers(-2, n_tables + 3, n)
    li = rng.integers(-10 ** 9, 10 ** 9, n)
    for i in range(n):
        t = nt[i]
        if 0 <= t < n_tables and layout[t] == 0:
            nt[i] = n_tables + 1                                                 # a zero-row table has no valid index
        elif 0 <= t < n_tables and layout[t]:
            li[i] = rng.integers(0, layout[t])
    k = 0
    for t, r in enumerate(layout):
        if r:
            nt[k:k + 2], li[k:k + 2] = t, (0, r - 1)
            k += 2
    return pads, tables, rows, host, nt, li


@pytest.mark.parametrize("n_tables", [1, 4, 16])
@pytest.mark.parametrize("F", GATHER_F)
def test_typed_gather_is_a_bit_exact_copy(F, n_tables):
    pads, tables, rows, host, nt, li = _gather_case(F, n_tables)
    want, bad = oh.typed_gather(host, nt, li, F)
    assert bad.size == 0
    ldo = F + 3
    box = Boxed(nt.size, F, ldo, c0=5, r0=2)
    box.reset()
    assert _gather_abi(tables, rows, _cuda(nt), _cuda(li), F, box.view, ldo) == 0
    assert np.array_equal(_bits(box.view), want.view(np.uint32))
    assert box.outside_intact()
    assert all(bool((p.flat.view(torch.int32)[:Padded.PAD] == CANARY).all()) for p in pads)
    # the wrapper: contiguous output, same bits, no error
    out = ops.typed_gather({t: tab for t, tab in enumerate(tables) if tab is not None}, n_tables, _cuda(nt), _cuda(li),
                           torch.full((nt.size, F), float("nan"), device=DEV))
    assert np.array_equal(_bits(out), want.view(np.uint32))


@pytest.mark.parametrize("F", [1, 33, 128])
def test_typed_gather_out_of_range_index_gives_a_zero_row_and_the_flag(F):
    pads, tables, rows, host, nt, li = _gather_case(F, 16, n=2000)
    assert LAYOUTS[16][4] == 0                                               # (4, 0): any index of a zero-row table
    poison = {101: (3, 2000), 202: (0, -1), 303: (9, 2 ** 40), 404: (4, 0), 1999: (15, -(2 ** 40))}
    for i, (t, j) in poison.items():
        nt[i], li[i] = t, j
    want, bad = oh.typed_gather(host, nt, li, F)
    assert bad.tolist() == sorted(poison)
    ldo = F + 1
    box = Boxed(nt.size, F, ldo)
    box.reset()
    assert _gather_abi(tables, rows, _cuda(nt), _cuda(li), F, box.view, ldo) == 1
    assert np.array_equal(_bits(box.view), want.view(np.uint32))           # zero rows at the bad positions
    assert box.outside_intact()
    tdict = {t: tab for t, tab in enumerate(tables) if tab is not None}
    with pytest.raises(lib.B200GnnError, match="position 101"):
        ops.typed_gather(tdict, 16, _cuda(nt), _cuda(li), torch.empty(nt.size, F, device=DEV))
    # the module surface (RGCN.group_input) fails on such an index, as the reference's indexing does
    with pytest.raises(lib.B200GnnError, match="position 101"):
        bnn.group_input({}, {str(t): tab for t, tab in tdict.items()}, _cuda(nt), _cuda(li), F)


def test_typed_gather_of_no_rows_launches_nothing_and_writes_nothing():
    t = Padded(10, 8)
    t.t.normal_()
    box = Boxed(0, 8, 9)
    box.reset()
    empty = torch.empty(0, dtype=torch.int64, device=DEV)
    assert _gather_abi([t.t], [10], empty, empty, 8, box.view, 9) == 0
    assert box.outside_intact()
    out = ops.typed_gather({0: t.t}, 1, empty, empty, torch.empty(0, 8, device=DEV))
    assert out.shape == (0, 8)


def test_typed_gather_at_the_ogbn_mag_table_sizes():
    """Full-size paper, author, institution and field-of-study tables at F = 128, a 200,000-node batch hitting row 0 and
    row rows - 1 of every table."""
    F, n = 128, 200_000
    names = ["paper", "author", "institution", "field_of_study"]
    g = torch.Generator(device=DEV).manual_seed(7)
    tables = {t: torch.randn(MAG[k], F, generator=g, device=DEV) for t, k in enumerate(names)}
    rng = _rng("mag-gather")
    nt = rng.integers(0, 4, n)
    li = np.array([rng.integers(0, MAG[names[t]]) for t in nt])
    for t, k in enumerate(names):
        nt[2 * t:2 * t + 2], li[2 * t:2 * t + 2] = t, (0, MAG[k] - 1)
    out = ops.typed_gather(tables, 4, _cuda(nt), _cuda(li), torch.empty(n, F, device=DEV))
    want, bad = oh.typed_gather([tables[t].cpu().numpy() for t in range(4)], nt, li, F)
    assert bad.size == 0 and np.array_equal(_bits(out), want.view(np.uint32))


# ================================================================================================================ scatter
SCATTER_F = [1, 31, 33, 128, 129]
RUNS = [1, 2, 31, 32, 33, 1000, 20_000]          # 20,000: one node of a small table (an institution) in a whole batch
SC_ROWS = [2000, 500, 300, 25_000]                # type 2 gets a null pointer


def _scatter_case(key, n_fill=6000):
    """(node_type, local_idx) with designed runs: for every length in RUNS a run of type 0 and one of type 1 at the same j,
    runs of the null type 2, a type past the tables (5) and indices past their table, random filler; positions shuffled."""
    rng = _rng("scatter", key)
    nt, li = [], []
    for k, L in enumerate(RUNS):
        for t in (0, 1, 2) if L <= 1000 else (3,):
            nt += [t] * L
            li += [10 + k] * L
    for t, j in ((5, 3), (0, 2000), (1, 500), (1, 499), (0, 1999), (0, 0)):
        nt += [t] * 3
        li += [j] * 3
    ft = rng.integers(0, 4, n_fill)
    nt += ft.tolist()
    li += [int(rng.integers(0, min(SC_ROWS[t], 600))) for t in ft]
    p = rng.permutation(len(nt))
    return np.asarray(nt)[p], np.asarray(li)[p], rng


def _want_scatter(d_host, nt, li, order, F, canary_tables):
    sums = oh.typed_scatter_inorder(d_host, nt, li, order, [SC_ROWS[0], SC_ROWS[1], None, SC_ROWS[3]])
    return oh.apply_scatter(canary_tables, sums)


@pytest.mark.parametrize("F", SCATTER_F)
def test_typed_scatter_adds_each_run_in_order(F):
    nt, li, rng = _scatter_case(F)
    n = nt.size
    d_host = _nonuniform(rng, n, F)
    ldd = F + 5
    dbox = Boxed(n, F, ldd, c0=3)
    dbox.reset(_cuda(d_host, torch.float32))
    ntd, lid = _cuda(nt), _cuda(li)
    order = device_argsort(ntd, lid, 6, 25_001)
    grads = [Padded(r, F) for r in SC_ROWS]
    tables = [grads[0].t, grads[1].t, None, grads[3].t]
    _scatter_abi(dbox.view, ldd, ntd, lid, order, F, tables, SC_ROWS)
    canary = np.full((1,), CANARY, np.int32).view(np.float32)[0]
    want = _want_scatter(d_host, nt, li, order.cpu().numpy(), F,
                         [np.full((r, F), canary, np.float32) if t != 2 else None for t, r in enumerate(SC_ROWS)])
    for t in (0, 1, 3):
        assert np.array_equal(_bits(tables[t]), want[t].view(np.uint32)), t
        assert bool((grads[t].flat.view(torch.int32)[:Padded.PAD] == CANARY).all())
        assert bool((grads[t].flat.view(torch.int32)[-Padded.PAD:] == CANARY).all())
    assert dbox.outside_intact()
    # the rows the designed runs hit really are sums of every term (and the two types' j = 10 + k stay apart)
    assert not np.array_equal(want[0][10 + 5], want[1][10 + 5])


def test_typed_scatter_orders_from_both_sorts_and_repeats_bit_for_bit():
    F = 33
    nt, li, rng = _scatter_case("sorts")
    d = _cuda(_nonuniform(rng, nt.size, F), torch.float32)
    ntd, lid = _cuda(nt), _cuda(li)
    o_dev = device_argsort(ntd, lid, 6, 25_001)
    o_torch = torch.argsort(ntd * 25_001 + lid, stable=True)
    assert torch.equal(o_dev, o_torch)
    outs = []
    for order in (o_dev, o_torch, o_dev):
        g = {t: torch.zeros(r, F, device=DEV) for t, r in enumerate(SC_ROWS) if t != 2}
        ops.typed_scatter(d, ntd, lid, order, g, 4)
        outs.append(g)
    for g in outs[1:]:
        assert all(torch.equal(g[t].view(torch.int32), outs[0][t].view(torch.int32)) for t in g)
    want = _want_scatter(d.cpu().numpy(), nt, li, o_dev.cpu().numpy(), F,
                         [np.zeros((r, F), np.float32) if t != 2 else None for t, r in enumerate(SC_ROWS)])
    assert all(np.array_equal(_bits(outs[0][t]), want[t].view(np.uint32)) for t in (0, 1, 3))


def test_equal_indices_of_adjacent_types_stay_separate_runs():
    """In (type, idx) order the last key of one type meets the first key of the next: (0, 7) | (1, 7) and (1, 9) | (3, 9)
    are neighbours with equal indices, and each is its own run, in the scatter and in the embedding Adam's heads."""
    F = 33
    rng = _rng("adjacent")
    nt = np.array([0] * 5 + [0] * 40 + [1] * 30 + [1] * 20 + [3] * 25 + [3] * 10)
    li = np.array([7] * 5 + list(rng.integers(0, 8, 40)) + [7] * 30 + list(rng.integers(7, 10, 20)) + [9] * 25 +
                  list(rng.integers(9, 12, 10)))
    p = rng.permutation(nt.size)
    nt, li = nt[p], li[p]
    ntd, lid = _cuda(nt), _cuda(li)
    order = device_argsort(ntd, lid, 4, 12)
    d_host = _nonuniform(rng, nt.size, F)
    d = _cuda(d_host, torch.float32)
    rows = [12, 12, 12, 12]
    grads = [Padded(12, F) for _ in rows]
    _scatter_abi(d, F, ntd, lid, order, F, [grads[0].t, grads[1].t, None, grads[3].t], rows)
    canary = np.full((1,), CANARY, np.int32).view(np.float32)[0]
    want = oh.apply_scatter([np.full((12, F), canary, np.float32) if t != 2 else None for t in range(4)],
                            oh.typed_scatter_inorder(d_host, nt, li, order.cpu().numpy(), [12, 12, None, 12]))
    for t in (0, 1, 3):
        assert np.array_equal(_bits(grads[t].t), want[t].view(np.uint32)), t
    for t in (0, 1, 3):
        table = torch.zeros(12, F, device=DEV)
        m, v = torch.zeros_like(table), torch.zeros_like(table)
        head = torch.full((12,), -1, dtype=torch.int32, device=DEV)
        ops.embedding_adam(torch.ones_like(d), ntd, lid, order, t, table, m, v, head,
                           torch.zeros(1, dtype=torch.int32, device=DEV), 0.01)
        marked = oh.run_heads(nt, li, order.cpu().numpy(), t, 12) >= 0
        assert np.array_equal((m != 0).all(1).cpu().numpy(), marked), t


def test_group_input_backward_keeps_runs_whole_next_to_types_without_a_table():
    """nn.group_input sorts by type·(rows + 1) + idx; an index of a type without a table is arbitrary and must not land
    inside a table type's run (it would split the run in two, and two warps would store the same row)."""
    F = 32
    rng = _rng("group-input")
    emb = {"0": torch.nn.Parameter(torch.randn(10, F, device=DEV)), "2": torch.nn.Parameter(torch.randn(10, F, device=DEV))}
    # type 1 has no table: (1, 14) sorts as 1·11 + 14 = 2·11 + 3 without clamping, inside the run of (2, 3)
    nt = np.array([2, 1, 2, 0, 2, 1, 0])
    li = np.array([3, 14, 3, 9, 3, 25, 9])
    w = _cuda(_nonuniform(rng, nt.size, F), torch.float32)
    h = bnn.group_input({}, emb, _cuda(nt), _cuda(li), F)
    (h * w).sum().backward()
    order = np.lexsort((li, nt))
    sums = oh.typed_scatter_inorder(w.cpu().numpy(), nt, li, order, [10, None, 10])
    want = oh.apply_scatter([np.zeros((10, F), np.float32), None, np.zeros((10, F), np.float32)], sums)
    for t in (0, 2):
        assert np.array_equal(_bits(emb[str(t)].grad), want[t].view(np.uint32)), t


# ================================================================================================================ embedding Adam
EMB_ROWS = {1: 3000, 2: 50, 3: 700}              # type 3 never appears in the batches


def _emb_batch(key, n=8000):
    rng = _rng("emb", key)
    nt = rng.integers(0, 3, n)                   # type 0: a feature type (no embedding)
    li = np.array([rng.integers(0, EMB_ROWS.get(t, 900)) for t in nt])
    nt[:5000], li[:5000] = 1, 17                 # one 5,000-node run
    nt[5000:5040], li[5000:5040] = 2, 49         # the last row of a small table
    p = rng.permutation(n)
    return nt[p], li[p], rng


def _state(rng, rows, F):
    table = _nonuniform(rng, rows, F)
    m = (rng.standard_normal((rows, F)) * 1e-2).astype(np.float32)        # non-zero moments: a skipped row is visible
    v = (rng.random((rows, F)) * 1e-3).astype(np.float32)
    return [_cuda(a, torch.float32) for a in (table, m, v)]


@pytest.mark.parametrize("F", [4, 33, 128])
def test_embedding_adam_is_the_scatter_then_adam_step(F):
    """Three tables share one head and one step counter, in sequence, as RGCNTrainer.train_step runs them; three steps."""
    rng = _rng("emb-state", F)
    eng = {t: _state(rng, r, F) for t, r in EMB_ROWS.items()}
    ref = {t: [a.clone() for a in s] for t, s in eng.items()}
    absent_m = eng[3][1].clone()
    head = torch.full((3000,), -1, dtype=torch.int32, device=DEV)
    step = torch.full((1,), 4, dtype=torch.int32, device=DEV)
    for s in range(3):
        nt, li, rng2 = _emb_batch((F, s))
        d = _cuda(_nonuniform(rng2, nt.size, F), torch.float32)
        ntd, lid = _cuda(nt), _cuda(li)
        order = device_argsort(ntd, lid, 4, 3000)
        for t in EMB_ROWS:
            ops.embedding_adam(d, ntd, lid, order, t, *eng[t], head, step, 0.01)
            assert bool((head == -1).all()), (s, t)
            assert int(step) == 4 + s, (s, t)
        grads = {t: torch.zeros_like(ref[t][0]) for t in EMB_ROWS}
        ops.typed_scatter(d, ntd, lid, order, grads, 4)
        for t in EMB_ROWS:
            ops.adam_step(*ref[t][:1], grads[t], *ref[t][1:], step.clone(), 0.01)
        for t in EMB_ROWS:
            for a, b, what in zip(eng[t], ref[t], ("table", "exp_avg", "exp_avg_sq")):
                assert torch.equal(a.view(torch.int32), b.view(torch.int32)), (s, t, what)
        step += 1
    # the table absent from every batch still took its zero-gradient updates: every first moment decayed
    assert bool((eng[3][1] != absent_m).all())


def test_embedding_adam_updates_exactly_the_oracle_run_heads():
    """The heads pass is visible as the rows that receive a gradient: from zero moments and an all-ones d_out, a row's
    exp_avg becomes non-zero iff oracle.run_heads marks it (its gradient is its run length)."""
    F = 8
    nt, li, rng = _emb_batch("heads", n=3000)
    ntd, lid = _cuda(nt), _cuda(li)
    order = device_argsort(ntd, lid, 4, 3000)
    d = _cuda(np.ones((nt.size, F), np.float32), torch.float32)
    for t, rows in EMB_ROWS.items():
        table = torch.zeros(rows, F, device=DEV)
        m, v = torch.zeros_like(table), torch.zeros_like(table)
        head = torch.full((rows,), -1, dtype=torch.int32, device=DEV)
        ops.embedding_adam(d, ntd, lid, order, t, table, m, v, head, torch.zeros(1, dtype=torch.int32, device=DEV), 0.01)
        marked = oh.run_heads(nt, li, order.cpu().numpy(), t, rows) >= 0
        moved = (m != 0).all(1).cpu().numpy()                 # exp_avg = 0.1·g with g = run length > 0
        assert np.array_equal(moved, marked), t
        assert bool((m[~torch.from_numpy(marked).to(DEV)] == 0).all())


def test_embedding_adam_empty_batch_and_empty_table():
    F = 33
    rng = _rng("emb-empty")
    tab, m, v = _state(rng, 700, F)
    ref = [a.clone() for a in (tab, m, v)]
    head = torch.full((700,), -1, dtype=torch.int32, device=DEV)
    step = torch.full((1,), 2, dtype=torch.int32, device=DEV)
    e = torch.empty(0, dtype=torch.int64, device=DEV)
    ops.embedding_adam(torch.empty(0, F, device=DEV), e, e, e, 1, tab, m, v, head, step, 0.01)
    ops.adam_step(ref[0], torch.zeros_like(ref[0]), ref[1], ref[2], step.clone(), 0.01)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip((tab, m, v), ref))
    assert bool((head == -1).all()) and int(step) == 2
    # rows == 0: nothing to sweep, nothing written
    nt, li, rng2 = _emb_batch("empty-table", n=500)
    ntd, lid = _cuda(nt), _cuda(li)
    buf = Padded(0, F)
    head2 = torch.full((8,), 7, dtype=torch.int32, device=DEV)
    ops.embedding_adam(_cuda(_nonuniform(rng2, 500, F), torch.float32), ntd, lid, device_argsort(ntd, lid, 4, 3000), 1,
                       buf.t, buf.t, buf.t, head2, step, 0.01)
    assert bool((buf.flat.view(torch.int32) == CANARY).all()) and bool((head2 == 7).all()) and int(step) == 2


def test_embedding_adam_on_the_full_size_author_table():
    F, rows, n = 128, MAG["author"], 150_000
    rng = _rng("emb-author")
    nt = rng.integers(0, 4, n)
    li = np.where(nt == 1, rng.integers(0, rows, n), rng.integers(0, 8000, n))
    nt[:3], li[:3] = 1, (0, rows - 1, rows - 1)
    ntd, lid = _cuda(nt), _cuda(li)
    order = device_argsort(ntd, lid, 4, rows)
    d = _cuda(_nonuniform(rng, n, F), torch.float32)
    g = torch.Generator(device=DEV).manual_seed(3)
    tab = torch.randn(rows, F, generator=g, device=DEV)
    m = torch.randn(rows, F, generator=g, device=DEV) * 1e-2
    v = torch.rand(rows, F, generator=g, device=DEV) * 1e-3
    ref = [tab.clone(), m.clone(), v.clone()]
    head = torch.full((rows,), -1, dtype=torch.int32, device=DEV)
    step = torch.full((1,), 9, dtype=torch.int32, device=DEV)
    ops.embedding_adam(d, ntd, lid, order, 1, tab, m, v, head, step, 0.01)
    grad = torch.zeros(rows, F, device=DEV)
    ops.typed_scatter(d, ntd, lid, order, {1: grad}, 4)
    ops.adam_step(ref[0], grad, ref[1], ref[2], step.clone(), 0.01)
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip((tab, m, v), ref))
    assert bool((head == -1).all()) and int(step) == 9


# ================================================================================================================ ReLU/dropout backward
@pytest.mark.parametrize("p", [0.0, 0.5, 0.3])
@pytest.mark.parametrize("K", [4, 32, 352, 512])
def test_relu_dropout_backward_bits(K, p):
    """d_y = d_out · fl(1 / fl(1 - p)) where x_out > 0, else +0 (x_out = 0, -0, negative or NaN), rounded once."""
    rng = _rng("relu-bwd", K, p)
    n = 1037
    x = rng.standard_normal((n, K)).astype(np.float32)
    x[rng.random((n, K)) < 0.2] = 0.0
    x[rng.random((n, K)) < 0.05] = -0.0
    x[0, 0] = np.nan
    d = _nonuniform(rng, n, K)
    inv = np.float32(1) / (np.float32(1) - np.float32(p)) if p > 0 else np.float32(1)
    want = np.where(x > 0, d * inv, np.float32(0)).astype(np.float32)
    xd, dd = _cuda(x, torch.float32), _cuda(d, torch.float32)
    out = ops.relu_dropout_bwd(dd, xd, p)
    assert np.array_equal(_bits(out), want.view(np.uint32))
    assert np.array_equal(_bits(dd), d.view(np.uint32))                   # out of place: d_out untouched
    same = ops.relu_dropout_bwd(dd, xd, p, out=dd)                         # in place, as RGCNTrainer.backward calls it
    assert same.data_ptr() == dd.data_ptr() and np.array_equal(_bits(dd), want.view(np.uint32))


def test_relu_dropout_backward_refuses_an_output_of_another_shape():
    x, d = torch.rand(100, 32, device=DEV), torch.randn(100, 32, device=DEV)
    with pytest.raises(lib.B200GnnError):
        ops.relu_dropout_bwd(d, x, 0.5, out=torch.empty(102, 32, device=DEV))   # larger: an unchecked launch stays inside


# ================================================================================================================ batch plan
def _rels_of(relations, T):
    return [sorted(r for r, (_, dst) in relations.items() if dst == t) for t in range(T)]


def _layout(nt: torch.Tensor, rels_of, T):
    """Internal row of every batch node (types grouped, stable) and the first virtual row of each type, from the
    definition: type t's block holds cnt_t nodes of (1 + R_t) slots."""
    cnt = [int((nt == t).sum()) for t in range(T)]
    vbase = [0]
    for t in range(T):
        vbase.append(vbase[-1] + cnt[t] * (1 + len(rels_of[t])))
    rank = torch.empty_like(nt)
    for t in range(T):
        m = (nt == t).nonzero().view(-1)
        rank[m] = torch.arange(m.numel(), device=nt.device)
    return cnt, vbase, rank


def _acat_fp64(b, tables, rels_of, T, F):
    """{t: Acat_t = [X_t | mean_r1 | ...] in fp64}, the reference's per-relation scatter-mean over the batch's edge list
    (duplicate edges counted, self-loops kept, empty neighbourhoods 0), and every sum's sum of magnitudes."""
    nt, li = b.node_type.view(-1).long(), b.local_node_idx.view(-1).long()
    n = nt.numel()
    h = torch.zeros(n, F, dtype=torch.float64, device=DEV)
    for t, tab in tables.items():
        m = nt == t
        h[m] = tab.double()[li[m]]
    src, dst = b.edge_index[0].long(), b.edge_index[1].long()
    et = b.edge_attr.view(-1).long()
    out, mags = {}, []
    for t in range(T):
        nodes = (nt == t).nonzero().view(-1)
        if nodes.numel() == 0:
            continue
        blocks = [h[nodes]]
        for r in rels_of[t]:
            m = et == r
            s = torch.zeros(n, F, dtype=torch.float64, device=DEV).index_add_(0, dst[m], h[src[m]])
            a = torch.zeros(n, F, dtype=torch.float64, device=DEV).index_add_(0, dst[m], h[src[m]].abs())
            c = torch.zeros(n, dtype=torch.float64, device=DEV).index_add_(0, dst[m], torch.ones_like(src[m], dtype=torch.float64))
            blocks.append((s / c.clamp(min=1)[:, None])[nodes])
            mags.append(a)
        out[t] = torch.cat(blocks, 1)
    return out, (torch.cat(mags) if mags else torch.zeros(1, device=DEV))


def _integer_model(tr: RGCNTrainer, x_types, F, key):
    """Load small-integer embedding rows (|v| <= 8) into the trainer; small-integer features for the feature types."""
    g = torch.Generator().manual_seed(_seed(key))
    sd = tr.state_dict()
    for k in sd:
        if k.startswith("emb_dict."):
            sd[k] = torch.randint(-8, 9, tuple(sd[k].shape), generator=g).float()
    tr.load_state_dict(sd)
    x = {t: torch.randint(-8, 9, (tr.num_nodes[t], F), generator=g).float().to(DEV) for t in x_types}
    tables = dict(x)
    tables.update(tr.emb)
    return x, tables


def _designed_batch():
    """A batch of small_mag's graph: papers, authors and institutions but no field of study (so relations 3 and 6 have no
    edge), no paper -> author edge (relation 5 empty while authors are present), institutions whose only relation is
    affiliated_with, duplicate edges in every relation present and self-loops in cites; nodes and edges shuffled."""
    rng = _rng("designed-batch")
    cnt = {0: 40, 1: 30, 2: 5}
    nt = np.concatenate([np.full(c, t) for t, c in cnt.items()])
    li = np.concatenate([np.concatenate([[0, NODES[t] - 1], rng.choice(np.arange(1, NODES[t] - 1), c - 2, replace=False)])
                         for t, c in cnt.items()])
    p = rng.permutation(nt.size)
    nt, li = nt[p], li[p]
    ids = {t: np.flatnonzero(nt == t) for t in cnt}
    edges = []
    for r, (s, d, e) in {0: (1, 2, 60), 1: (1, 0, 150), 2: (0, 0, 200), 4: (2, 1, 40)}.items():
        src, dst = rng.choice(ids[s], e), rng.choice(ids[d][:-3], e)           # leaves nodes without in-edges
        src[1::7], dst[1::7] = src[0::7][:len(src[1::7])], dst[0::7][:len(dst[1::7])]   # duplicates
        if r == 2:
            dst[2::9] = src[2::9]                                                       # self-loops
        edges += [(a, b, r) for a, b in zip(src, dst)]
    edges = [edges[i] for i in rng.permutation(len(edges))]
    ei = torch.tensor([[a for a, _, _ in edges], [b for _, b, _ in edges]])
    et = torch.tensor([r for _, _, r in edges])
    return Data(edge_index=ei, edge_attr=et, node_type=torch.from_numpy(nt), local_node_idx=torch.from_numpy(li)).to(DEV)


def _mag_batches(n):
    from tools.bench_rgcn import mag_graph
    data, x_dict, num_nodes, relations, C_ = mag_graph(0.002)
    loader = sampling.GraphSAINTRandomWalkSampler(data, batch_size=300, walk_length=2, num_steps=n, seed=4)
    return list(loader), list(x_dict), num_nodes, relations, C_


def _plan_cases():
    data, _, rel = small_mag(3)
    small = [("designed", _designed_batch())] + [(f"small_mag{i}", b) for i, b in enumerate(batches(data, 3, seed=9))]
    mag, x_types, num_nodes, mrel, C_ = _mag_batches(2)
    mk_small = lambda: RGCNTrainer(16, 24, 7, 2, 0.0, NODES, [0], len(rel), rel, seed=1)
    mk_mag = lambda: RGCNTrainer(128, 32, C_, 2, 0.0, num_nodes, x_types, len(mrel), mrel, seed=1)
    return [(name, b, mk_small, [0], rel, 16) for name, b in small] + \
           [(f"mag{i}", b, mk_mag, x_types, mrel, 128) for i, b in enumerate(mag)]


def test_designed_batch_reaches_the_edge_cases():
    b = _designed_batch()
    _, _, rel = small_mag(3)
    nt, et = b.node_type, b.edge_attr
    assert int((nt == 3).sum()) == 0 and int((et == 5).sum()) == 0 and int((nt == 1).sum()) > 0
    assert _rels_of(rel, 4)[2] == [0] and int((et == 0).sum()) > 0
    key = b.edge_index[0] * 1000 + b.edge_index[1] + et * 10 ** 6
    assert torch.unique(key).numel() < key.numel()
    assert bool(((b.edge_index[0] == b.edge_index[1]) & (et == 2)).any())


def test_batch_plan_arena_is_the_per_relation_scatter_mean():
    for name, b, make, x_types, rel, F in _plan_cases():
        tr = make()
        T = tr.T
        x, tables = _integer_model(tr, x_types, F, name)
        tr.forward(b, x, training=False)
        arena = tr._fwd["arenas"][0]
        rels_of = _rels_of(rel, T)
        nt = b.node_type.view(-1).long()
        cnt, vbase, _ = _layout(nt, rels_of, T)
        assert arena.shape == (vbase[-1], F), name
        want, mags = _acat_fp64(b, tables, rels_of, T, F)
        _assert_exact(mags, 0, name)
        assert sorted(want) == [t for t in range(T) if cnt[t]], name
        for t, w in want.items():
            got = arena[vbase[t]:vbase[t + 1]].view(cnt[t], -1)
            assert torch.equal(got, w.float()), (name, t)


def test_batch_plan_transposed_spmm_is_within_the_adjoint_bound():
    """dX = Gtᵀ-SpMM(dArena) is the adjoint of the mean: dX[i] = dA[v_self(i)] + Σ_{e: src(e) = i} dA[v(e)] / deg(v(e)),
    v(e) the virtual row (destination, relation slot) of edge e and deg(v) its edge count.

    The kernel multiplies by the stored value w_v = fl(1/deg_v) = (1/deg_v)(1 + δ), |δ| <= u (w = 1 exactly for slot 0),
    and adds the m_i = 1 + outdeg(i) products in some order, products rounded or fused: computed = Σ_v dA_v·w_v·(1 + θ_v),
    |θ_v| <= γ(m_i) (Higham §3.1).  So |computed - exact| <= Σ_v |dA_v|/deg_v · |(1 + δ)(1 + θ_v) - 1|
    <= (γ(m_i) + u·(1 + γ(m_i))) · Σ_v |dA_v| / deg_v.  The fp64 reference errs by ~m_i·2^-53 of the same sum, far below."""
    for name, b, make, x_types, rel, F in _plan_cases():
        tr = make()
        T = tr.T
        P = tr.plan(b)
        _, Gt = P.graphs()
        rels_of = _rels_of(rel, T)
        nt = b.node_type.view(-1).long()
        cnt, vbase, rank = _layout(nt, rels_of, T)
        off = np.concatenate([[0], np.cumsum(cnt)])
        width = torch.tensor([1 + len(r) for r in rels_of], device=DEV)
        vb = torch.tensor(vbase[:-1], device=DEV)
        slot = torch.zeros(len(rel), dtype=torch.long, device=DEV)
        for t in range(T):
            for k, r in enumerate(rels_of[t]):
                slot[r] = k + 1
        V = vbase[-1]
        g = torch.Generator(device=DEV).manual_seed(_seed(name, "dA"))
        dA = torch.randn(V, F, generator=g, device=DEV) * torch.exp2(torch.randint(-10, 11, (V, 1), generator=g, device=DEV)).float()
        dx = ops.spmm_csr(Gt, dA, "sum")
        src, dst = b.edge_index[0].long(), b.edge_index[1].long()
        et = b.edge_attr.view(-1).long()
        v_self = vb[nt] + rank * width[nt]
        v_edge = vb[nt[dst]] + rank[dst] * width[nt[dst]] + slot[et]
        deg = torch.bincount(v_edge, minlength=V).double()
        d64 = dA.double()
        term = d64[v_edge] / deg[v_edge][:, None]
        exact = d64[v_self].clone().index_add_(0, src, term)
        mag = d64[v_self].abs().index_add_(0, src, term.abs())
        m = 1 + torch.bincount(src, minlength=nt.numel()).double()
        bound = (_gamma(m) + U * (1 + _gamma(m)))[:, None].to(DEV) * mag
        internal = torch.tensor(off[:-1], device=DEV)[nt] + rank
        got = dx.double()[internal]
        err = (got - exact).abs()
        assert bool((err <= bound).all()), (name, float((err / bound.clamp(min=1e-300)).max()))


# ================================================================================================================ refusals
F0 = 16


def _good(n=50, rows=20):
    g = torch.Generator(device=DEV).manual_seed(1)
    tab = torch.randn(rows, F0, generator=g, device=DEV)
    nt = torch.zeros(n, dtype=torch.int64, device=DEV)
    li = torch.randint(0, rows, (n,), generator=g, device=DEV)
    return tab, nt, li


def _bad_tables(tab):
    """Tables the kernels would misread, each readable at pitch F0 for rows < tab.shape[0] (no stray access)."""
    rows = tab.shape[0]
    return {"float64": tab.double(), "column slice": torch.randn(rows, 2 * F0, device=DEV)[:, :F0],
            "wider": torch.randn(rows, F0 + 4, device=DEV), "flat": torch.randn(rows * F0, device=DEV)}


def test_typed_gather_refuses_what_it_would_misread():
    tab, nt, li = _good()
    out = torch.empty(nt.numel(), F0, device=DEV)
    for what, bad in _bad_tables(tab).items():
        with pytest.raises(lib.B200GnnError, match="table of type 0"):
            ops.typed_gather({0: bad}, 1, nt, li, out)
    with pytest.raises(lib.B200GnnError):
        ops.typed_gather({1: tab}, 1, nt, li, out)                       # key past n_tables
    with pytest.raises(lib.B200GnnError):
        ops.typed_gather({0: tab}, 17, nt, li, out)                      # more node types than the kernels take
    long_nt = torch.zeros(nt.numel() + 8, dtype=torch.int64, device=DEV)
    with pytest.raises(lib.B200GnnError):
        ops.typed_gather({0: tab}, 1, long_nt[:nt.numel() - 3], li, out)  # shorter than out (a prefix of a longer buffer)
    with pytest.raises(lib.B200GnnError):
        ops.typed_gather({0: tab}, 1, nt, li.view(-1, 1), out)           # not 1-D
    e = torch.empty(0, dtype=torch.int64, device=DEV)
    with pytest.raises(lib.B200GnnError):
        ops.typed_gather({0: tab.cpu()}, 1, e, e, torch.empty(0, F0, device=DEV))   # a host table (empty batch)


def test_typed_scatter_refuses_what_it_would_misread():
    tab, nt, li = _good()
    d = torch.randn(nt.numel(), F0, device=DEV)
    order = torch.argsort(li, stable=True)
    for what, bad in _bad_tables(tab).items():
        if what == "float64":
            bad = torch.zeros_like(bad)
        with pytest.raises(lib.B200GnnError):
            ops.typed_scatter(d, nt, li, order, {0: bad}, 1)
    longer = torch.zeros(order.numel() + 8, dtype=torch.int64, device=DEV)
    longer[:order.numel()] = order
    with pytest.raises(lib.B200GnnError):
        ops.typed_scatter(d, nt, li, longer[:order.numel() - 5], {0: torch.zeros_like(tab)}, 1)
    with pytest.raises(lib.B200GnnError):
        ops.typed_scatter(d, nt, li, order, {3: torch.zeros_like(tab)}, 2)   # key past n_tables


def test_embedding_adam_refuses_what_it_would_misread():
    tab, nt, li = _good()
    d = torch.randn(nt.numel(), F0, device=DEV)
    order = torch.argsort(li, stable=True)
    m, v = torch.zeros_like(tab), torch.zeros_like(tab)
    head = torch.full((tab.shape[0],), -1, dtype=torch.int32, device=DEV)
    step = torch.zeros(1, dtype=torch.int32, device=DEV)
    with pytest.raises(lib.B200GnnError):
        ops.embedding_adam(d, nt, li, order, 0, tab, torch.zeros(tab.shape[0] + 1, F0, device=DEV), v, head, step, 0.01)
    with pytest.raises(lib.B200GnnError):
        ops.embedding_adam(d, nt, li, order, 0, tab, m, v, head[:-1], step, 0.01)
    with pytest.raises(lib.B200GnnError):
        ops.embedding_adam(torch.randn(nt.numel(), F0 + 4, device=DEV), nt, li, order, 0, tab, m, v, head, step, 0.01)
    longer = torch.zeros(order.numel() + 8, dtype=torch.int64, device=DEV)
    with pytest.raises(lib.B200GnnError):
        ops.embedding_adam(d, nt, li, longer[:order.numel() - 5], 0, tab, m, v, head, step, 0.01)
    for what, bad in _bad_tables(tab).items():
        if what in ("float64",):
            continue                                                    # refused by the fp32 pointer check before
        with pytest.raises(lib.B200GnnError):
            ops.embedding_adam(d, nt, li, order, 0, bad, m, v, head, step, 0.01)
    assert bool((head == -1).all()) and int(step) == 0


def test_group_input_takes_int32_indices_as_the_reference_does():
    tab, nt, li = _good(n=64)
    emb = {"0": torch.nn.Parameter(tab.clone())}
    want = bnn.group_input({}, emb, nt, li, F0)
    # int32 vectors that are prefixes of buffers twice as long, so that an int64 read of them stays inside
    nt32 = torch.zeros(2 * nt.numel(), dtype=torch.int32, device=DEV)[:nt.numel()]
    li32 = torch.zeros(2 * li.numel(), dtype=torch.int32, device=DEV)
    li32[:li.numel()] = li.int()
    got = bnn.group_input({}, emb, nt32, li32[:li.numel()], F0)
    assert torch.equal(got, want)
