"""The geometry tables of tests/test_gemm_fused_gpu.py (no GPU needed): each fused-operand GEMM entry point's table keeps
reaching the shapes where its fused code paths run — CTAs with two or more tiles on a 132-SM H100 (with random keep bits,
so a wrong next-tile prefetch changes the result), both tile shapes, K off the 32-column grid, ragged N, misaligned and
ldc % 4 != 0 outputs, p in {0, 0.1, 0.5}, slopes of both signs, 0 and 1, the weight gradient's node-range clamp and the
PReLU weight gradient on column blocks with a wider keep-bit pitch."""
import test_gemm_fused_gpu as T

RAGGED_N = {1, 40, 49, 100, 349}
P_ALL = {0.0, 0.1, 0.5}
SLOPES = ("negative", "zero", "positive", "one")


def _slope_kinds(slopes):
    return {"negative" if s < 0 else "zero" if s == 0 else "one" if s == 1 else "positive" for s in slopes}


def _multi(M, N, narrow_ok=True):
    return T.gemm_tiles(M, N, narrow_ok) > T.SMS


def _prologue_table(cases, k_big):
    """Properties shared by the ACT and PReLU prologue tables: rows (M, N, K, p, ..., view, bias)."""
    # >= 2 tiles per CTA on both tile shapes, with random keep bits and with K off the 32-grid
    for narrow in (True, False):
        assert any(_multi(M, N) and (N <= 48) == narrow and p > 0 and K % 32 for M, N, K, p, *_ in cases), narrow
    assert any(K % 32 for _, _, K, *_ in cases)
    assert {4, 36, 100, 1000} <= {c[2] for c in cases}
    assert k_big in {c[2] for c in cases}
    assert RAGGED_N <= {c[1] for c in cases}
    assert {"shift", "odd", "vec"} <= {c[-2] for c in cases}
    assert P_ALL <= {c[3] for c in cases}
    assert {True, False} <= {c[-1] for c in cases}
    # the scalar epilogue on a multi-tile launch
    assert any(_multi(c[0], c[1]) and c[-2] != "vec" for c in cases)


def test_act_table():
    _prologue_table(T.ACT_CASES, 2048)
    assert all(c[2] <= 2048 and c[2] % 4 == 0 for c in T.ACT_CASES)


def test_prelu_table():
    _prologue_table(T.PRELU_CASES, 4100)
    assert _slope_kinds(c[4] for c in T.PRELU_CASES) == set(SLOPES)
    assert all(c[2] % 4 == 0 for c in T.PRELU_CASES)


def test_bnbwd_bits_table():
    cases = T.BNBWD_CASES
    assert all(N % 32 == 0 and 48 < N <= 256 for _, N, *_ in cases)
    # both epilogue paths (the TMA path needs N % 128 == 0) over >= 2 tiles per CTA
    tma = [c for c in cases if c[4] == 1 and c[1] % 128 == 0]
    reg = [c for c in cases if c[4] == 2]
    assert any(_multi(M, N, False) and p > 0 for M, N, _, p, *_ in tma)
    assert any(_multi(M, N, False) and p > 0 for M, N, _, p, *_ in reg)
    assert {0, 1, 2} <= {c[4] for c in cases}
    assert any(K % 32 for _, _, K, *_ in cases)
    assert P_ALL <= {c[3] for c in cases}
    assert {True, False} <= {c[5] for c in cases}


def test_prelu_bwd_table():
    cases = T.PRELU_BWD_CASES
    assert all(N % 32 == 0 for _, N, *_ in cases)
    assert any(_multi(M, N, False) and p > 0 for M, N, _, p, *_ in cases)
    assert any(N <= 48 for _, N, *_ in cases) and any(N > 256 for _, N, *_ in cases)
    assert any(K % 32 for _, _, K, *_ in cases) and 4100 in {c[2] for c in cases}
    assert P_ALL <= {c[3] for c in cases}
    assert _slope_kinds(c[4] for c in cases) == set(SLOPES)
    assert {True, False} <= {c[5] for c in cases} and {True, False} <= {c[6] for c in cases}


def test_rowidx_table():
    cases = T.ROWIDX_CASES
    for narrow in (True, False):
        assert any(_multi(M, N) and (N <= 48) == narrow for M, N, *_ in cases), narrow
    assert RAGGED_N <= {c[1] for c in cases}
    assert {"shift", "odd", "vec"} <= {c[3] for c in cases}
    assert any(_multi(M, N) and v != "vec" for M, N, _, v in cases)
    assert any(K % 32 for _, _, K, _ in cases)


def _wgrad_table(cases):
    assert {4, 36, 100, 132, 520, 2048} <= {c[1] for c in cases}
    assert {4, 40, 132, 512} <= {c[2] for c in cases}
    assert {1, 31, 33, 40_001} <= {c[0] for c in cases}
    assert all(c[1] % 4 == 0 and c[1] <= 2048 and c[2] % 4 == 0 and c[2] <= 512 for c in cases)
    assert P_ALL <= {c[3] for c in cases}
    # more node ranges fit than there are node blocks: the ranges > num_kb clamp
    assert any(r > kb for r, kb in (T.wgrad_ranges(*c[:3]) for c in cases))
    # several node ranges, each over several blocks: the keep words prefetched one block ahead
    assert any(1 < r and 2 * r <= kb for r, kb in (T.wgrad_ranges(*c[:3]) for c in cases if c[3] > 0))


def test_wgrad_act_table():
    _wgrad_table(T.WGRAD_ACT_CASES)


def test_wgrad_prelu_table():
    cases = T.WGRAD_PRELU_CASES
    _wgrad_table(cases)
    assert _slope_kinds(c[4] for c in cases) == set(SLOPES)
    assert all(c0 % 32 == 0 for *_, c0, _ in cases)
    # column blocks: a bits base offset of c0 / 32 words and a row pitch wider than ceil(Kin / 32)
    blocks = [(Kin, c0, spare) for _, Kin, _, _, _, c0, spare in cases if c0 > 0]
    assert any(spare > 0 for *_, spare in blocks) and any(c0 + Kin > 2048 for Kin, c0, _ in blocks)
    assert any(c0 > 0 and Kin % 32 for Kin, c0, _ in blocks)
    assert {2052, 3000} <= set(T.WGRAD_PRELU_WIDE_KIN)


def test_refusal_entries_cover_the_table():
    assert set(T.REFUSAL_ENTRIES) == {"act", "prelu", "prelu_bwd", "bnbwd_bits", "rowidx", "wgrad_act", "wgrad_prelu"}
