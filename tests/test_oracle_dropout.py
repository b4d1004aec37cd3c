"""The CPU restatement of the dropout keep decisions (oracle/dropout.py) against the contract it restates: the threshold rule
on both paths, the exact 24-bit comparison on grid points, a word-use audit (no random unit decides two elements) and the
engines' stream layouts.  CPU only; tests/test_dropout_draws_gpu.py holds every kernel to this restatement."""
import numpy as np
import pytest

from oracle import dropout as od
from oracle.sampling import philox4x32

P16_CASES = [(2.0 ** -16, 1), (0.25, 16384), (0.5, 32768), (0.75, 49152), (1 - 2.0 ** -16, 65535)]
P24_CASES = [0.1, 0.2, 0.3]
SEED, OFFSET = 0x9E3779B97F4A7C15, (1 << 32) + 5           # both 32-bit halves of key and counter in use


def scalar_keep(g: int, c: int, p: float, seed: int, offset: int) -> bool:
    """The contract for one element, written out once more without arrays."""
    p = float(np.float32(p))
    t = p * 65536.0
    if p > 0 and t == int(t):
        r = philox4x32(seed, offset, np.array([g >> 1], dtype=np.uint64))[0]
        word = int(r[2 * (g & 1) + c // 2])
        u16 = (word >> 16) if c % 2 else (word & 0xFFFF)
        return u16 >= int(t)
    word = int(philox4x32(seed, offset, np.array([g], dtype=np.uint64))[0][c])
    return (word >> 8) * 2.0 ** -24 >= p


@pytest.mark.parametrize("p,thr", P16_CASES)
def test_p16_threshold_and_decisions(p, thr):
    assert od.p16_threshold(p) == thr
    g = np.arange(37, 37 + 41, dtype=np.uint64)                 # odd start: both halves of straddling blocks
    keep = od.keep_float4(g, p, SEED, OFFSET)
    want = np.array([[scalar_keep(int(x), c, p, SEED, OFFSET) for c in range(4)] for x in g])
    assert np.array_equal(keep, want)
    assert od.expected_keep_rate(p) == 1 - thr / 65536


@pytest.mark.parametrize("p", P24_CASES)
def test_24bit_path_and_its_exact_rate(p):
    assert od.p16_threshold(p) is None
    g = np.arange(11, 11 + 41, dtype=np.uint64)
    keep = od.keep_float4(g, p, SEED, OFFSET)
    want = np.array([[scalar_keep(int(x), c, p, SEED, OFFSET) for c in range(4)] for x in g])
    assert np.array_equal(keep, want)
    # u * 2^-24 >= p is u >= ceil(p * 2^24): the exact rate of the fp32 threshold
    assert od.expected_keep_rate(p) == 1 - np.ceil(np.float32(p) * 2.0 ** 24) / 2.0 ** 24
    assert od.expected_keep_rate(p) != 1 - p                    # the fp32 p is not the decimal one


@pytest.mark.parametrize("p16", [True, False])
def test_rate_of_the_restatement(p16):
    p = 0.25 if p16 else 0.3
    keep = od.keep_float4(np.arange(1 << 18, dtype=np.uint64), p, 7, 3)
    q = od.expected_keep_rate(p)
    n = keep.size
    assert abs(keep.mean() - q) <= 5 * np.sqrt(q * (1 - q) / n)
    col = keep.mean(axis=0)                                     # the four components, each on its own units
    assert np.all(np.abs(col - q) <= 5 * np.sqrt(q * (1 - q) / keep.shape[0]))


def test_zero_rate_keeps_everything_and_p16_needs_p_above_zero():
    assert od.p16_threshold(0.0) is None
    assert od.keep_float4(np.arange(100, dtype=np.uint64), 0.0, 1, 2).all()


def test_24bit_comparison_on_grid_points():
    """p = k·2⁻²⁴ exactly: an element whose uniform is k is kept at p = k·2⁻²⁴ (>=) and dropped at p = (k + 1)·2⁻²⁴."""
    g = np.arange(64, dtype=np.uint64)
    u24 = philox4x32(SEED, OFFSET, g) >> 8
    picked = 0
    for x in range(64):
        for c in range(4):
            k = int(u24[x, c])
            if k % 256 == 0 or (k + 1) % 256 == 0:              # a multiple of 2⁸·2⁻²⁴ would take the P16 path
                continue
            p = k * 2.0 ** -24
            assert float(np.float32(p)) == p and od.p16_threshold(p) is None
            assert od.keep_float4(g[x:x + 1], p, SEED, OFFSET)[0, c]
            assert not od.keep_float4(g[x:x + 1], (k + 1) * 2.0 ** -24, SEED, OFFSET)[0, c]
            picked += 1
    assert picked > 200


@pytest.mark.parametrize("p16", [True, False])
@pytest.mark.parametrize("start,n", [(0, 1), (1, 1), (0, 64), (3, 61), ((1 << 32) - 3, 9)])
def test_word_use_audit_passes_on_the_contract(p16, start, n):
    assert od.audit_word_use(np.arange(start, start + n, dtype=np.uint64), p16)


def _reuse_x(g, p16):
    """A restatement with the bug `half ? r.x : r.x`: odd float4s read the even one's words."""
    block, word, half = od.sources(g, p16)
    return block, word % 2, half


def _one_half(g, p16):
    """... and one that reads the low 16-bit half for both components of a word."""
    block, word, half = od.sources(g, p16)
    return block, word, np.zeros_like(half) if p16 else half


def _block_per_float4(g, p16):
    """... and one that gives P16 float4 g block g instead of g >> 1, reading words x, y only."""
    block, word, half = od.sources(g, p16)
    return (np.asarray(g, dtype=np.uint64) if p16 else block), word % 2 if p16 else word, half


@pytest.mark.parametrize("bug", [_reuse_x, _one_half])
def test_word_use_audit_fails_a_restatement_that_reuses_words(bug):
    g = np.arange(5, 69, dtype=np.uint64)
    assert not od.audit_word_use(g, True, src=bug)
    # the decisions of such a restatement differ from the contract's
    assert not np.array_equal(od.keep_float4(g, 0.5, SEED, OFFSET, src=bug), od.keep_float4(g, 0.5, SEED, OFFSET))


def test_block_per_float4_passes_the_audit_but_not_the_decisions():
    """Block g instead of g >> 1 uses no word twice, so only the comparison with the contract's decisions catches it."""
    g = np.arange(5, 69, dtype=np.uint64)
    assert od.audit_word_use(g, True, src=_block_per_float4)
    assert not np.array_equal(od.keep_float4(g, 0.5, SEED, OFFSET, src=_block_per_float4), od.keep_float4(g, 0.5, SEED, OFFSET))


def test_derived_layouts_agree_with_the_flat_rule():
    n, K, p = 7, 36, 0.5                                        # nvec_row = 9: P16 blocks straddle rows
    full = od.mask(n + 5, K, p, SEED, OFFSET)
    assert np.array_equal(od.mask(n, K, p, SEED, OFFSET, row_offset=5), full[5:])
    gid = np.array([11, 0, 3, 3, 8], dtype=np.int64)
    assert np.array_equal(od.mask_mapped(gid, 12, K, 8, p, SEED, OFFSET), full[gid][:, 8:20])
    b = od.bits(2, n, K, p, SEED, OFFSET)
    assert b.shape == (2, n, 2)
    for l in range(2):
        m = od.mask(n, K, p, SEED, OFFSET + l)
        unpacked = ((b[l][:, :, None] >> np.arange(32, dtype=np.uint32)) & 1).reshape(n, 64).astype(bool)
        assert np.array_equal(unpacked[:, :K], m) and not unpacked[:, K:].any()
    hops = od.sign_hops(3, n, K, p, SEED, OFFSET)
    assert all(np.array_equal(hops[h], od.mask(n, K, p, SEED, OFFSET + h)) for h in range(3))
    d = od.label_drop(23, p, SEED, OFFSET)
    assert all(d[j] == (not od.keep_float4(np.array([j // 4], dtype=np.uint64), p, SEED, OFFSET)[0, j % 4]) for j in range(23))


def _offsets_over_steps(layout, steps=6):
    return [o for s in range(steps) for o in layout(s).values()]


@pytest.mark.parametrize("name,layout", [
    *[(f"gcn L={L}", lambda s, L=L: od.gcn_streams(L, s)) for L in (2, 3, 4)],
    *[(f"gat L={L}", lambda s, L=L: od.gat_streams(L, s)) for L in (2, 3)],
    *[(f"gat_teacher L={L} it={it}", lambda s, L=L, it=it: od.gat_teacher_streams(L, it, s)) for L in (2, 3) for it in (0, 1, 2)],
    *[(f"sign H={H} ff={ff}", lambda s, H=H, ff=ff: od.sign_streams(H, ff, s)) for H in (1, 3, 5) for ff in (1, 2, 3)],
])
def test_stream_layouts_give_every_stream_of_every_step_its_own_offset(name, layout):
    offs = _offsets_over_steps(layout)
    assert len(offs) == len(set(offs)), name
    assert max(offs) < od.gcrd_sample_stream(0)                 # far below the sampler's stream


def test_layout_off_by_one_clashes_with_the_next_step():
    """What the audit on the GPU guards against: one offset too few per step reuses the next step's first stream."""
    L, it = 3, 1
    short = (it + 1) * 2 * L                                    # step_streams without the label mask's + 1
    label = [(it + 1) * 2 * L + s * short for s in range(4)]
    first = [s * short for s in range(4)]
    assert set(label) & set(first)
    H, ff = 3, 2
    D = od.sign_step_streams(H, ff) - 1
    assert {H + (H + 1) * (ff - 1) + s * D for s in range(4)} & {s * D for s in range(4)}


def test_disjoint_reports_shared_blocks_only_at_equal_seed_and_offset():
    a = (1, 5, np.arange(0, 10, dtype=np.uint64))
    b = (1, 5, np.arange(10, 20, dtype=np.uint64))
    c = (1, 5, np.arange(19, 21, dtype=np.uint64))
    d = (2, 5, np.arange(0, 10, dtype=np.uint64))
    assert od.disjoint([a, b, d]) == []
    assert od.disjoint([a, b, c, d]) == [(1, 2, 1, 5)]
