"""The integer graph kernels, element for element against plain CPU references: the stable LSD radix argsort, coalesce and
row pointers (csrc/graph_prep.cu), random walks, the GraphSAINT induced sub-graph and the induced edge list
(csrc/sampling.cu).  Everything downstream takes their output as exact: a wrong permutation or a dropped edge is a different
graph, not a rounding error.  So every check here is equality, at the digit-pass counts, tile edges, grid-stride sizes and
MAG-scale shapes where these kernels can go wrong:

* argsort: ``np.lexsort((minor, major))``, which is stable and cannot overflow;
* coalesce, row pointers and the SparseTensor views built on them: oracle/graph.py;
* random walks and the induced sub-graph: oracle/sampling.py;
* induced edges: torch_geometric.utils.subgraph(mask.nonzero(), edge_index, relabel_nodes=True), restated in oracle/graph.py;
* the refusals: the error code, and no launch.
"""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, rgcn, sampling
from efficient_gnns_b200.sparse import SparseTensor, device_argsort, device_coalesce
from oracle import graph as og
from oracle import sampling as osamp

ROOT = Path(__file__).resolve().parents[1]
BAD_ARG, UNSUPPORTED = -1, -2
SORT_TILE = 2048                   # keys per CTA of the radix sort; also the tile of the coalesce scan
GRID_STRIDE = 132 * 16 * 256       # above this many items the 1-D kernels of graph_prep.cu grid-stride
U64 = 2 ** 64 - 1


def rng(seed):
    return np.random.default_rng(seed)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


# ================================================================================================= 1. radix argsort
def sizes_for_bits(bits):
    """(major_size, minor_size), neither a power of two where it can be avoided, whose product - 1 has ``bits`` bits and
    lies in the top half of that range, so that the top digit pass decides the order of about half the keys."""
    if bits == 1:
        return 1, 2
    if bits == 2:
        return 1, 3
    if bits == 64:
        return 3, 5_000_000_000_000_000_000                  # 1.5e19: 8 digit passes
    target = (3 << (bits - 2)) + 1                             # 1.5 * 2^(bits-1)
    major = max(1, int(round(target ** 0.5)) | 1)
    minor = -(-target // major)
    assert (major * minor - 1).bit_length() == bits
    return major, minor


def keys(n, major_size, minor_size, seed, dup=True):
    """Uniform keys over the whole range, both extremes present, and (``dup``) runs of equal keys and of equal majors."""
    r = rng(seed)
    major = r.integers(0, major_size, n, dtype=np.int64)
    minor = r.integers(0, minor_size, n, dtype=np.int64)
    major[0], minor[0] = major_size - 1, minor_size - 1
    if n > 1:
        major[1] = minor[1] = 0
    if dup and n > 8:
        h = n // 2
        major[h:] = major[:n - h]                             # equal majors ...
        minor[n // 3: n // 3 + n // 5] = minor[:n // 5]       # ... and equal keys, far apart in the input
    return major, minor


def check_argsort(major, minor, major_size, minor_size):
    got = device_argsort(cuda(major), cuda(minor), major_size, minor_size)
    assert got.dtype == torch.int64 and got.is_cuda
    want = np.lexsort((minor, major))
    g = host(got)
    if not np.array_equal(g, want):
        bad = int(np.argmax(g != want))
        raise AssertionError(f"n={len(major)} range {major_size}x{minor_size}: first difference at {bad}: {g[bad]} != {want[bad]}")


BITS = [1, 2, 7, 8, 9, 16, 17, 24, 25, 32, 33, 40, 41, 56, 57, 64]


def test_sizes_for_bits_cover_the_digit_boundaries():
    for b in BITS:
        ma, mi = sizes_for_bits(b)
        assert (ma * mi - 1).bit_length() == b and ma * mi < 1.8e19, b


def test_host_argsort_is_stable_and_exact_for_wide_keys():
    """The CPU path of device_argsort (host-side logic) sorts key ranges of 2^63 and above without overflowing."""
    for ma, mi in [(3, 5_000_000_000_000_000_000), (9, 1_999_999_999_000_000_000), (7, 3), (2, 1)]:
        major, minor = keys(5000, ma, mi, seed=ma)
        got = device_argsort(torch.from_numpy(major), torch.from_numpy(minor), ma, mi)
        assert np.array_equal(got.numpy(), np.lexsort((minor, major))), (ma, mi)


@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
def test_argsort_every_key_bit_length(bits):
    """ceil(bits / 8) digit passes: bit lengths 8k and 8k+1 on both sides of a pass boundary, 64 bits (8 passes)."""
    ma, mi = sizes_for_bits(bits)
    for n, seed in ((20_011, bits), (SORT_TILE * 3 + 5, bits + 100)):
        check_argsort(*keys(n, ma, mi, seed), ma, mi)


@pytest.mark.gpu
def test_argsort_key_range_just_below_the_limit():
    """A key range of 1.8e19 - 9e9, past 2^63, where an int64 key major * minor_size + minor would overflow."""
    ma, mi = 9, 1_999_999_999_000_000_000
    assert 2 ** 63 < ma * mi < 1.8e19
    check_argsort(*keys(70_001, ma, mi, 7), ma, mi)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 31, 32, 33, 255, 256, 257, 2047, 2048, 2049, 4095, 4097, 300 * SORT_TILE - 1,
                               300 * SORT_TILE + 1])
def test_argsort_tile_edges(n):
    ma = mi = 1_939_743                                       # MAG node ids: 42-bit keys, 6 passes
    check_argsort(*keys(n, ma, mi, n), ma, mi)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_argsort_grid_stride_and_a_long_histogram_scan():
    """n above the 1-D kernels' grid (grid-stride loops of make_keys), and n = 5.3 M: 2,588 tiles, so the single-CTA scan of
    the 256 x 2,588 digit histogram carries across 647 rounds."""
    check_argsort(*keys(GRID_STRIDE + 12_345, 169_343, 169_343, 1), 169_343, 169_343)
    n = 5_300_000
    assert 256 * (-(-n // SORT_TILE)) > 600 * 1024
    check_argsort(*keys(n, 736_389, 1_134_649, 2), 736_389, 1_134_649)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_argsort_stability_alone():
    """Every key equal (the identity), and minor_size = 1 with 2 to 4 types over millions of entries: the R-GCN plan's
    node-type sort, where the order inside a type is decided by stability alone."""
    n = 3_000_017
    got = device_argsort(torch.full((n,), 4, device="cuda"), torch.full((n,), 6, device="cuda"), 5, 7)
    assert torch.equal(got, torch.arange(n, device="cuda"))
    for types, n in ((2, 2_000_003), (3, 4_194_305), (4, 3_333_333)):
        nt = rng(types).integers(0, types, n, dtype=np.int64)
        nt[: n // 3] = np.sort(nt[: n // 3])[::-1]          # long descending runs too
        check_argsort(nt, np.zeros(n, dtype=np.int64), types, 1)


@pytest.mark.gpu
def test_argsort_accepts_int32_indices():
    """The kernel reads int64; the wrapper widens int32 inputs instead of reading them as int64."""
    major, minor = keys(10_007, 1000, 3000, 3)
    got = device_argsort(cuda(major.astype(np.int32)), cuda(minor.astype(np.int32)), 1000, 3000)
    assert np.array_equal(host(got), np.lexsort((minor, major)))


@pytest.mark.gpu
def test_argsort_beyond_the_kernel_raises_instead_of_overflowing():
    x = torch.zeros(4, dtype=torch.long, device="cuda")
    with pytest.raises(lib.B200GnnError, match="1.8e19"):
        device_argsort(x, x, 2, 2 ** 63 - 1)


# --------------------------------------------------------------------------------- the MAG synthetic at scale 1
@pytest.fixture(scope="module")
def mag():
    """The reference's homogeneous view of ogbn-mag at full size (mag_pyg/gnn.py:320-347): 1,939,743 nodes, about 42 M
    directed edges once the relations are made undirected."""
    sys.path.insert(0, str(ROOT / "tools"))
    from bench_rgcn import mag_graph
    data, _, num_nodes, relations, _ = mag_graph(1.0)
    return data, num_nodes, relations


def loader_roots(loader, step):
    g = torch.Generator(device="cuda")
    g.manual_seed(loader.seed * 1_000_003 + step)
    return host(torch.randint(0, loader.N, (loader.batch_size,), generator=g, device="cuda"))


@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_argsort_the_rgcn_plan_call_shapes(mag, monkeypatch):
    """The four argsorts of an R-GCN step, recorded from BatchPlan on a GraphSAINT batch of the MAG synthetic (20,000 roots,
    walk_length 2) and checked one by one: node types and virtual rows (minor_size = 1: stability alone), the transpose
    (f_col, f_row) with a key of more than 32 bits, and the embedding order (type, local id) of embedding Adam."""
    data, num_nodes, relations = mag
    b = next(iter(sampling.GraphSAINTRandomWalkSampler(data, batch_size=20_000, walk_length=2, num_steps=1, seed=3)))
    R, T = len(relations), len(num_nodes)
    rel_src = torch.tensor([relations[r][0] for r in range(R)], device="cuda")
    rel_dst = torch.tensor([relations[r][1] for r in range(R)], device="cuda")
    calls = []

    def recording(major, minor, major_size, minor_size):
        out = device_argsort(major, minor, major_size, minor_size)
        calls.append((host(major), host(minor), major_size, minor_size, host(out)))
        return out
    monkeypatch.setattr(rgcn, "device_argsort", recording)
    P = rgcn.BatchPlan(b.edge_index, b.edge_attr, b.node_type, rel_src, rel_dst, T)
    li = b.local_node_idx.view(-1).long()[P.perm].contiguous()
    recording(P.node_type_int, li, T, max(num_nodes.values()))      # RGCNTrainer.train_step's embedding order
    assert len(calls) == 4
    (nt, z0, s0, m0, _), (vrow, z1, s1, m1, _), (fc, fr, s2, m2, _), (nti, lii, s3, m3, _) = calls
    assert (s0, m0) == (T, 1) and not z0.any() and (s1, m1) == (P.V, 1) and not z1.any()
    assert len(vrow) > SORT_TILE * 50 and len(nt) > 10_000
    assert (s2, m2) == (P.N, P.V) and (s2 * m2 - 1).bit_length() >= 32
    assert (s3, m3) == (T, 1_134_649)
    for major, minor, _, _, got in calls:
        assert np.array_equal(got, np.lexsort((minor, major)))


# ================================================================================================= 2. coalesce
def raw_coalesce(row, col, n_rows, n_cols, with_src=True):
    """b200gnn_graph_coalesce_i64 with canary-filled outputs; returns (rc, row, col, src or None, rowptr, nnz)."""
    L = lib.load()
    n = int(row.numel())
    ws = torch.empty(int(L.b200gnn_graph_sort_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
    o_r, o_c = torch.full((n,), -7, dtype=torch.long, device="cuda"), torch.full((n,), -7, dtype=torch.long, device="cuda")
    src = torch.full((n,), -7, dtype=torch.int32, device="cuda") if with_src else None
    ptr = torch.full((n_rows + 1,), -7, dtype=torch.long, device="cuda")
    nnz = torch.full((1,), -7, dtype=torch.long, device="cuda")
    rc = L.b200gnn_graph_coalesce_i64(row.data_ptr(), col.data_ptr(), n, n_rows, n_cols, o_r.data_ptr(), o_c.data_ptr(),
                                      None if src is None else src.data_ptr(), ptr.data_ptr(), nnz.data_ptr(), ws.data_ptr(),
                                      lib.stream_ptr())
    k = int(nnz.item())
    return rc, o_r[:k], o_c[:k], None if src is None else src[:k], ptr, k


def want_coalesce(row, col, n_rows, n_cols):
    """oracle/graph.py's coalesce and row pointers, and the input index of the first duplicate of every kept entry."""
    r, c, _ = og.coalesce(row, col, n_cols)
    order = np.lexsort((col, row))
    rs, cs = row[order], col[order]
    head = np.ones(len(rs), dtype=bool)
    head[1:] = (rs[1:] != rs[:-1]) | (cs[1:] != cs[:-1])
    return r, c, og.ind2ptr(r, n_rows), order[head]


def check_coalesce(row, col, n_rows, n_cols):
    rc, o_r, o_c, src, ptr, k = raw_coalesce(cuda(row), cuda(col), n_rows, n_cols)
    assert rc == 0
    r, c, p, s = want_coalesce(row, col, n_rows, n_cols)
    assert k == len(r)
    assert np.array_equal(host(o_r), r) and np.array_equal(host(o_c), c)
    assert np.array_equal(host(ptr), p)
    assert np.array_equal(host(src), s)
    ro, co, rowptr, src_l = device_coalesce(cuda(row), cuda(col), n_rows, n_cols)      # the wrapper: same arrays
    assert torch.equal(ro, o_r) and torch.equal(co, o_c) and torch.equal(rowptr, ptr) and torch.equal(src_l, src.long())
    return r, c


def relation(n_src, n_dst, e, seed, empty_tail=777):
    """A MAG-like relation with duplicates: sources uniform (the last ``empty_tail`` rows empty), destinations skewed, 15 %
    of the entries repeated at random later positions."""
    r = rng(seed)
    src = r.integers(0, n_src - empty_tail, e, dtype=np.int64)
    dst = np.minimum((r.random(e) ** 3 * n_dst).astype(np.int64), n_dst - 1)
    dup = r.integers(0, e, e // 7)
    src, dst = np.concatenate([src, src[dup]]), np.concatenate([dst, dst[dup]])
    p = r.permutation(len(src))
    return src[p], dst[p]


MAG_RECT = [("author", "paper", 1_134_649, 736_389), ("paper", "author", 736_389, 1_134_649),
            ("paper", "field", 736_389, 59_965), ("field", "paper", 59_965, 736_389)]


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("src_t,dst_t,n_rows,n_cols", MAG_RECT, ids=[f"{a}-{b}" for a, b, _, _ in MAG_RECT])
def test_coalesce_rectangular_mag_relations(src_t, dst_t, n_rows, n_cols):
    """Rectangular matrices of MAG relation sizes in both orientations, with duplicates and trailing empty rows; the
    author rows (n_rows + 1 > 540,672) make the row-pointer kernel grid-stride."""
    row, col = relation(n_rows, n_cols, 2_500_000, n_rows % 1000)
    r, _ = check_coalesce(row, col, n_rows, n_cols)
    assert len(r) < len(row) and r[-1] < n_rows - 777


@pytest.mark.gpu
def test_coalesce_duplicate_runs_across_tiles():
    """Duplicate runs that straddle every sorted index 2048*k (the radix tile and the scan tile), runs longer than a tile,
    on a 37 x 45,001 matrix; each kept entry's source must be the first of its duplicates in input order."""
    r = rng(5)
    U = 9000
    key = np.sort(r.choice(37 * 45_001, U, replace=False)).astype(np.int64)
    lens = r.integers(2, 12, U)
    lens[::997] = (SORT_TILE + 1, 2 * SORT_TILE + 3, SORT_TILE - 1, 5000, 2, 7, 3, 4, 9, 11)[: len(lens[::997])]
    sk = np.repeat(key, lens)
    straddle = sk[SORT_TILE - 1::SORT_TILE][: len(sk[SORT_TILE::SORT_TILE])] == sk[SORT_TILE::SORT_TILE]
    assert straddle.sum() > 0.7 * len(straddle)
    p = r.permutation(len(sk))
    row, col = sk[p] // 45_001, sk[p] % 45_001
    c_r, _ = check_coalesce(row, col, 37, 45_001)
    assert len(c_r) == U


@pytest.mark.gpu
def test_coalesce_all_duplicates_no_duplicates_and_one_entry():
    n = 100_003
    r, c = check_coalesce(np.full(n, 3, dtype=np.int64), np.full(n, 5, dtype=np.int64), 7, 9)
    assert (r.tolist(), c.tolist()) == ([3], [5])
    key = rng(6).choice(1000 * 1_000_003, 300_000, replace=False).astype(np.int64)
    r, _ = check_coalesce(key // 1_000_003, key % 1_000_003, 1000, 1_000_003)
    assert len(r) == len(key)
    check_coalesce(np.array([4], dtype=np.int64), np.array([0], dtype=np.int64), 5, 1)


@pytest.mark.gpu
def test_coalesce_without_source_indices():
    """src_out = NULL: the same rows, columns, row pointers and count as with it."""
    row, col = relation(1_134_649, 736_389, 700_000, 9)
    rr, cc = cuda(row), cuda(col)
    full = raw_coalesce(rr, cc, 1_134_649, 736_389)
    none = raw_coalesce(rr, cc, 1_134_649, 736_389, with_src=False)
    assert full[0] == none[0] == 0 and full[5] == none[5]
    for a, b in zip(full[1:3] + full[4:5], none[1:3] + none[4:5]):
        assert torch.equal(a, b)
    r, c, p, _ = want_coalesce(row, col, 1_134_649, 736_389)
    assert np.array_equal(host(none[1]), r) and np.array_equal(host(none[2]), c) and np.array_equal(host(none[4]), p)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_sparse_tensor_views_of_a_rectangular_relation():
    """The SparseTensor views engines build on these kernels, on author->paper (1,134,649 x 736,389), unsorted with
    duplicates: construction (argsort), csr2csc, colptr, t() and to_symmetric against oracle/graph.py."""
    M, N = 1_134_649, 736_389
    row, col = relation(M, N, 1_500_000, 11)
    adj = SparseTensor(row=cuda(row), col=cuda(col), sparse_sizes=(M, N))
    order = np.lexsort((col, row))
    r0, c0 = row[order], col[order]
    r, c, _ = adj.coo()
    assert np.array_equal(host(r), r0) and np.array_equal(host(c), c0)
    assert np.array_equal(host(adj.storage.rowptr()), og.ind2ptr(r0, M))
    perm = og.csr2csc(r0, c0)
    assert np.array_equal(host(adj.storage.csr2csc()), perm)
    colptr = og.ind2ptr(c0[perm], N)
    assert np.array_equal(host(adj.storage.colptr()), colptr)
    t = adj.t()
    rt, ct, _ = t.coo()
    assert t.sparse_sizes() == (N, M)
    assert np.array_equal(host(rt), c0[perm]) and np.array_equal(host(ct), r0[perm])
    assert np.array_equal(host(t.storage.rowptr()), colptr)
    sym = adj.to_symmetric()
    r1, c1 = og.to_symmetric(r0, c0, M)
    rs, cs, _ = sym.coo()
    assert sym.sparse_sizes() == (M, M)
    assert np.array_equal(host(rs), r1) and np.array_equal(host(cs), c1)
    assert np.array_equal(host(sym.storage.rowptr()), og.ind2ptr(r1, M))


# ================================================================================================= 3. random walks
@pytest.fixture(scope="module")
def walk_graph():
    """20,000 nodes, skewed in-degrees; the 600 lowest ids (the most visited ones) have no out-edges, so walkers land on
    them and must hold."""
    from efficient_gnns_b200.synthetic import skewed_edges
    n = 20_000
    ei = skewed_edges(n, 200_000, 21).numpy()
    ei = ei[:, ei[0] >= 600]
    rowptr, col, _ = osamp.csr_by_source(ei, n)
    g = sampling.SaintGraph(cuda(ei), n)
    assert np.array_equal(host(g.rowptr), rowptr) and np.array_equal(host(g.col), col)
    return g, rowptr, col


def check_walks(g, rowptr, col, start, L, seed, offset):
    got = host(sampling.random_walk(g.rowptr, g.col, cuda(start), L, seed=seed, offset=offset))
    want = osamp.random_walk(rowptr, col, start, L, seed, offset)
    assert got.shape == (len(start), L + 1)
    if not np.array_equal(got, want):
        w, s = np.argwhere(got != want)[0]
        raise AssertionError(f"L={L} seed={seed} offset={offset}: walker {w} step {s}: {got[w, s]} != {want[w, s]}")
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("L", [0, 1, 3, 4, 5, 8])
def test_random_walk_lengths_counts_seeds_and_offsets(walk_graph, L):
    """Walker counts around the 256-thread block, seeds 0 and 2^64 - 1, offsets past 2^32; walkers that reach a node
    without out-edges hold."""
    g, rowptr, col = walk_graph
    held = 0
    for k, (nw, seed, offset) in enumerate(((1, 0, 0), (255, U64, 2 ** 32 + 7), (257, 0, 2 ** 40 + 3), (9_999, U64, 0),
                                            (12_345, 987_654_321_987, 2 ** 63 + 5))):
        start = rng(L * 10 + k).integers(0, 20_000, nw)
        start[: nw // 10] = rng(k).integers(0, 600, nw // 10)    # some start on a node without out-edges
        w = check_walks(g, rowptr, col, start, L, seed, offset)
        held += int(((w[:, 1:] == w[:, :-1]) & (w[:, :-1] < 600)).sum())
    assert L == 0 or held > 0


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_random_walk_a_million_walkers(walk_graph):
    g, rowptr, col = walk_graph
    nw = 2 ** 20 + 7
    check_walks(g, rowptr, col, rng(1).integers(0, 20_000, nw), 4, U64, 2 ** 33 + 1)


@pytest.mark.gpu
def test_random_walk_of_the_longest_length(walk_graph):
    """walk_length 4096, the largest the kernel takes: 1,024 Philox blocks per walker."""
    g, rowptr, col = walk_graph
    start = rng(2).integers(0, 20_000, 301)
    check_walks(g, rowptr, col, start, 4096, 0, 2 ** 32)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_random_walk_from_a_hub_of_three_million():
    """A star whose centre has 3,000,017 out-edges (each leaf points back): every second step picks (u * deg) >> 32 over a
    degree far above 2^16, from walkers that all start at the centre."""
    D = 3_000_017
    rowptr = np.concatenate([[0], D + np.arange(D + 1)]).astype(np.int64)
    col = np.concatenate([np.arange(1, D + 1), np.zeros(D)]).astype(np.int64)
    g = SimpleNamespace(rowptr=cuda(rowptr.astype(np.int32)), col=cuda(col.astype(np.int32)))
    w = check_walks(g, rowptr, col, np.zeros(100_003, dtype=np.int64), 5, 0x9E3779B97F4A7C15, 2 ** 36 + 11)
    assert len(np.unique(w[:, 1])) > 95_000 and w[:, 1].max() > D - 1000   # picks spread over the whole row


# ================================================================================================= 4. induced sub-graph
LOOPED = 2_000_050                 # outside the hub's targets: a self-loop and an edge into the hub, nothing else


@pytest.fixture(scope="module")
def designed_graph():
    """A hub (node 0) with 2,000,000 out-edges; four rows each of degree 31, 32, 33, 64 and 65 into a 5,000-node core;
    edges into node 0 (local id 0 whenever the hub is selected); self-loops; a random core; parent edge order shuffled."""
    r = rng(31)
    N, H = 2_000_100, 2_000_000
    src = [np.zeros(H, dtype=np.int64)]
    dst = [np.arange(1, H + 1, dtype=np.int64)]
    rows = {}
    for d in (31, 32, 33, 64, 65):
        for k in range(4):
            v = int(r.integers(1, 5000))
            while v in rows:
                v = int(r.integers(1, 5000))
            rows[v] = d
            t = r.choice(5000, d, replace=False)
            t[0] = 0
            if k == 1:
                t[1] = v                                    # a self-loop
            src.append(np.full(d, v))
            dst.append(t)
    core = r.integers(1, 5000, (2, 120_000))
    core = core[:, ~np.isin(core[0], list(rows))]
    src += [core[0], np.array([LOOPED, LOOPED])]
    dst += [core[1], np.array([LOOPED, 0])]
    ei = np.stack([np.concatenate(src), np.concatenate(dst)]).astype(np.int64)
    ei = ei[:, r.permutation(ei.shape[1])]
    rowptr, col, eid = osamp.csr_by_source(ei, N)
    g = sampling.SaintGraph(cuda(ei), N)
    assert np.array_equal(host(g.eid), eid) and np.array_equal(host(g.rowptr), rowptr) and np.array_equal(host(g.col), col)
    deg = np.diff(rowptr)
    assert deg[0] == H and all(deg[v] == d for v, d in rows.items())
    return g, rowptr, col, eid, rows


def check_subgraph(g, rowptr, col, eid, nodes):
    ei_loc, e_id = g.subgraph(cuda(nodes))
    r, c, e = osamp.saint_subgraph(rowptr, col, eid, nodes)
    assert np.array_equal(host(ei_loc[0]), r) and np.array_equal(host(ei_loc[1]), c) and np.array_equal(host(e_id), e)
    assert int((g.node_map != -1).sum()) == 0
    return r


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_subgraph_rows_of_every_ballot_shape(designed_graph):
    """Selected rows of degree 31, 32, 33, 64, 65 (partial and several ballot rounds per warp) and the 2 M hub, with a
    partial selection of the hub's targets."""
    g, rowptr, col, eid, rows = designed_graph
    r = rng(4)
    base = np.concatenate([[0], list(rows), r.choice(np.arange(1, 5000), 2000, replace=False),
                           r.choice(np.arange(5000, 2_000_100), 30_000, replace=False)])
    nodes = np.unique(base)
    got = check_subgraph(g, rowptr, col, eid, nodes)
    assert (got == 0).sum() > 20_000                         # the hub row's kept edges
    without_hub = nodes[1:]
    check_subgraph(g, rowptr, col, eid, without_hub)


@pytest.mark.gpu
@pytest.mark.timeout(300)
def test_subgraph_of_every_node_is_the_graph_in_csr_order(designed_graph):
    g, rowptr, col, eid, _ = designed_graph
    N = len(rowptr) - 1
    ei_loc, e_id = g.subgraph(torch.arange(N, device="cuda"))
    assert np.array_equal(host(ei_loc[0]), np.repeat(np.arange(N), np.diff(rowptr)))
    assert np.array_equal(host(ei_loc[1]), col) and np.array_equal(host(e_id), eid)
    assert int((g.node_map != -1).sum()) == 0


@pytest.mark.gpu
def test_subgraph_of_a_single_node(designed_graph):
    g, rowptr, col, eid, rows = designed_graph
    loop = next(v for v in rows if v in col[rowptr[v]:rowptr[v + 1]])
    assert len(check_subgraph(g, rowptr, col, eid, np.array([loop]))) == 1       # its self-loop, as (0, 0)
    assert len(check_subgraph(g, rowptr, col, eid, np.array([0]))) == 0
    assert len(check_subgraph(g, rowptr, col, eid, np.array([2_000_099]))) == 0  # no edges at all


@pytest.mark.gpu
def test_subgraph_without_edge_ids_reports_csr_positions(designed_graph):
    """eid = NULL through the raw ABI: the third output is the CSR position of every kept edge."""
    g, rowptr, col, _, rows = designed_graph
    L = lib.load()
    nodes = np.unique(np.concatenate([[0, LOOPED], list(rows), rng(8).choice(np.arange(1, 5000), 1500, replace=False)]))
    nd = cuda(nodes)
    n_sel = len(nodes)
    counts = torch.full((n_sel,), -7, dtype=torch.long, device="cuda")
    st = lib.stream_ptr()
    assert L.b200gnn_saint_subgraph_count_i64(g.rowptr.data_ptr(), g.col.data_ptr(), nd.data_ptr(), n_sel, g.node_map.data_ptr(),
                                              counts.data_ptr(), st) == 0
    ptr = torch.cumsum(counts, 0) - counts
    e = int(counts.sum())
    out = torch.full((3, e), -7, dtype=torch.long, device="cuda")
    assert L.b200gnn_saint_subgraph_fill_i64(g.rowptr.data_ptr(), g.col.data_ptr(), None, nd.data_ptr(), n_sel,
                                             g.node_map.data_ptr(), ptr.data_ptr(), out[0].data_ptr(), out[1].data_ptr(),
                                             out[2].data_ptr(), st) == 0
    g.node_map[nd] = -1
    r, c, p = osamp.saint_subgraph(rowptr, col, np.arange(len(col), dtype=np.int64), nodes)
    assert np.array_equal(host(out[0]), r) and np.array_equal(host(out[1]), c) and np.array_equal(host(out[2]), p)
    assert int((g.node_map != -1).sum()) == 0


# ================================================================================================= 5. induced edges
def want_induced(ei, mask):
    return og.subgraph(np.nonzero(mask)[0], ei, relabel_nodes=True)[0].reshape(2, -1)


def masks(n, seed):
    r = rng(seed)
    return {"random": r.random(n) < 0.45, "all": np.ones(n, dtype=bool), "none": np.zeros(n, dtype=bool)}


@pytest.mark.gpu
@pytest.mark.timeout(300)
@pytest.mark.parametrize("E", [1023, 1024, 1025, 1_050_001, 4_200_000])
def test_induced_edges_tile_counts_masks_and_column_slices(E):
    """E around the 1,024-edge tile and past 1,024 tiles (each scan thread then owns several tiles); masks of 1,025 and
    2 M nodes, all true, all false; the edge list a [:, :E] slice of a wider tensor (row pitch > E)."""
    for n in (1025, 2_000_000):
        wide = rng(E + n).integers(0, n, (2, E + 333))
        ei = cuda(wide)[:, :E]
        assert ei.stride(0) == E + 333
        for name, m in masks(n, E % 97 + n).items():
            got = sampling.induced_edges(ei, cuda(m))
            want = want_induced(wide[:, :E], m)
            assert np.array_equal(host(got), want), (n, name)
            if name == "all":
                assert np.array_equal(host(got), wide[:, :E])


@pytest.mark.gpu
def test_induced_edges_count_out_of_range_endpoints():
    """Edges with a negative or >= n endpoint are counted in totals[1], never read; the kept count and the fill cover the
    valid edges only; the wrapper raises."""
    L = lib.load()
    n, E = 3000, 5000
    r = rng(12)
    ei = r.integers(0, n, (2, E))
    bad_at = r.choice(E, 41, replace=False)
    ei[0, bad_at[:10]] = -1
    ei[1, bad_at[10:20]] = n
    ei[0, bad_at[20:30]] = -(2 ** 40)
    ei[1, bad_at[30:]] = n + 10 ** 12
    m = r.random(n) < 0.5
    good = np.ones(E, dtype=bool)
    good[bad_at] = False
    want = want_induced(ei[:, good], m)
    d_ei, d_m = cuda(ei), cuda(m)
    rank = torch.empty(n + 1, dtype=torch.long, device="cuda")
    tiles = torch.empty(2 * int(L.b200gnn_induced_edges_tiles(E)), dtype=torch.long, device="cuda")
    totals = torch.full((2,), -7, dtype=torch.long, device="cuda")
    st = lib.stream_ptr()
    assert L.b200gnn_induced_edges_count_i64(d_ei.data_ptr(), E, E, d_m.data_ptr(), n, rank.data_ptr(), tiles.data_ptr(),
                                             totals.data_ptr(), st) == 0
    assert totals.tolist() == [want.shape[1], 41]
    assert np.array_equal(host(rank), np.concatenate([[0], np.cumsum(m)]))
    out = torch.full((2, want.shape[1]), -7, dtype=torch.long, device="cuda")
    assert L.b200gnn_induced_edges_fill_i64(d_ei.data_ptr(), E, E, d_m.data_ptr(), n, rank.data_ptr(), tiles.data_ptr(),
                                            out.data_ptr(), out.stride(0), st) == 0
    assert np.array_equal(host(out), want)
    with pytest.raises(lib.B200GnnError, match="41 edges refer to a node outside"):
        sampling.induced_edges(d_ei, d_m)


# ================================================================================================= 6. the sampler at MAG scale
@pytest.mark.gpu
@pytest.mark.timeout(900)
def test_sampler_at_the_reference_settings_on_a_mag_sized_graph(mag):
    """GraphSAINTRandomWalkSampler(batch_size=20000, walk_length=2, num_steps=30) (mag_pyg/gnn.py:361-366, 504-506) on the
    MAG-sized graph: the first and the last batch of the epoch against the oracle's replay of the walks, its induced
    sub-graph and its attribute slicing."""
    data, _, _ = mag
    loader = sampling.GraphSAINTRandomWalkSampler(data, batch_size=20000, walk_length=2, num_steps=30, sample_coverage=0,
                                                  seed=5)
    assert loader.N == 1_939_743 and loader.E > 40_000_000
    kept = {}
    for step, b in enumerate(loader):
        assert b.num_nodes == b.n_id.numel() and b.edge_index.shape[1] == b.e_id.numel()
        if step in (0, 29):
            kept[step] = b
    assert sorted(kept) == [0, 29]
    ei = data.edge_index.numpy()
    rowptr, col, eid = osamp.csr_by_source(ei, loader.N)
    for step, b in kept.items():
        walks = osamp.random_walk(rowptr, col, loader_roots(loader, step), 2, 5, step)
        nodes = np.unique(walks)
        assert np.array_equal(host(b.n_id), nodes), step
        r, c, e = osamp.saint_subgraph(rowptr, col, eid, nodes)
        assert len(e) > 10_000
        assert np.array_equal(host(b.edge_index), np.stack([r, c])) and np.array_equal(host(b.e_id), e), step
        assert np.array_equal(host(b.edge_attr), data.edge_attr.numpy()[e])
        for k in ("node_type", "local_node_idx", "y", "train_mask"):
            assert np.array_equal(host(getattr(b, k)), getattr(data, k).numpy()[nodes]), (step, k)


# ================================================================================================= 7. refusals
@pytest.mark.gpu
def test_refusals_do_no_device_work():
    """Bad sizes and ranges come back as B200GNN_ERR_BAD_ARG / _UNSUPPORTED before any launch, outputs untouched."""
    L = lib.load()
    st = lib.stream_ptr()
    a = torch.arange(64, dtype=torch.long, device="cuda")
    ws = torch.empty(int(L.b200gnn_graph_sort_workspace_bytes(64)), dtype=torch.uint8, device="cuda")
    perm = torch.full((64,), -7, dtype=torch.int32, device="cuda")
    o64 = torch.full((200,), -7, dtype=torch.long, device="cuda")
    i32 = torch.zeros(8, dtype=torch.int32, device="cuda")
    P, W, O = a.data_ptr(), ws.data_ptr(), o64.data_ptr()
    torch.cuda.synchronize()
    before = lib.launch_count()
    cases = {
        "workspace n < 0": (L.b200gnn_graph_sort_workspace_bytes(-1), BAD_ARG),
        "argsort n < 0": (L.b200gnn_graph_argsort_i64(P, P, -1, 4, 4, perm.data_ptr(), W, st), BAD_ARG),
        "argsort major_size 0": (L.b200gnn_graph_argsort_i64(P, P, 64, 0, 4, perm.data_ptr(), W, st), BAD_ARG),
        "argsort minor_size < 0": (L.b200gnn_graph_argsort_i64(P, P, 64, 4, -3, perm.data_ptr(), W, st), BAD_ARG),
        "argsort range 1.8e19": (L.b200gnn_graph_argsort_i64(P, P, 64, 2, 9_000_000_000_000_000_000, perm.data_ptr(), W, st),
                                 UNSUPPORTED),
        "argsort range 2^64 - 2": (L.b200gnn_graph_argsort_i64(P, P, 64, 2, 2 ** 63 - 1, perm.data_ptr(), W, st), UNSUPPORTED),
        "coalesce n < 0": (L.b200gnn_graph_coalesce_i64(P, P, -1, 4, 4, O, O, None, O, O, W, st), BAD_ARG),
        "coalesce n_rows 0": (L.b200gnn_graph_coalesce_i64(P, P, 64, 0, 4, O, O, None, O, O, W, st), BAD_ARG),
        "coalesce n_cols < 0": (L.b200gnn_graph_coalesce_i64(P, P, 64, 4, -1, O, O, None, O, O, W, st), BAD_ARG),
        "coalesce range 1.8e19": (L.b200gnn_graph_coalesce_i64(P, P, 64, 3, 6_000_000_000_000_000_000, O, O, None, O, O, W, st),
                                  UNSUPPORTED),
        "walk length 4097": (L.b200gnn_random_walk_i64(i32.data_ptr(), i32.data_ptr(), 7, P, 64, 4097, 0, 0, O, st), BAD_ARG),
        "walk length < 0": (L.b200gnn_random_walk_i64(i32.data_ptr(), i32.data_ptr(), 7, P, 64, -1, 0, 0, O, st), BAD_ARG),
        "walk n_nodes 0": (L.b200gnn_random_walk_i64(i32.data_ptr(), i32.data_ptr(), 0, P, 64, 2, 0, 0, O, st), BAD_ARG),
        "walk n_walks < 0": (L.b200gnn_random_walk_i64(i32.data_ptr(), i32.data_ptr(), 7, P, -1, 2, 0, 0, O, st), BAD_ARG),
        "subgraph count n_sel < 0": (L.b200gnn_saint_subgraph_count_i64(i32.data_ptr(), i32.data_ptr(), P, -1, i32.data_ptr(), O,
                                                                         st), BAD_ARG),
        "subgraph fill n_sel < 0": (L.b200gnn_saint_subgraph_fill_i64(i32.data_ptr(), i32.data_ptr(), None, P, -1,
                                                                      i32.data_ptr(), O, O, O, O, st), BAD_ARG),
        "induced count ld < E": (L.b200gnn_induced_edges_count_i64(P, 31, 32, P, 64, O, O, O, st), BAD_ARG),
        "induced fill ld < E": (L.b200gnn_induced_edges_fill_i64(P, 31, 32, P, 64, O, O, O, 32, st), BAD_ARG),
        "induced count n < 0": (L.b200gnn_induced_edges_count_i64(P, 32, 32, P, -1, O, O, O, st), BAD_ARG),
        "induced count E < 0": (L.b200gnn_induced_edges_count_i64(P, 32, -1, P, 64, O, O, O, st), BAD_ARG),
        "induced fill ld_out < 0": (L.b200gnn_induced_edges_fill_i64(P, 32, 32, P, 64, O, O, O, -1, st), BAD_ARG),
    }
    torch.cuda.synchronize()
    assert lib.launch_count() == before
    for what, (rc, want) in cases.items():
        assert rc == want, (what, rc)
    assert bool((perm == -7).all()) and bool((o64 == -7).all())
    with pytest.raises(lib.B200GnnError, match="random_walk_i64 failed: bad argument"):
        sampling.random_walk(i32, i32, a, 4097)
    aliased = torch.zeros(1, 40, dtype=torch.long, device="cuda").expand(2, 40)      # both rows one row: ld = 0 < E
    with pytest.raises(lib.B200GnnError, match="induced_edges_count_i64 failed: bad argument"):
        sampling.induced_edges(aliased, torch.ones(3, dtype=torch.bool, device="cuda"))
    assert lib.launch_count() == before
