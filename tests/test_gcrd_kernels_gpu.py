"""Contract of the G-CRD kernels (csrc/gcrd.cu, the row gather of dense_rows.cu and the row-indexed store of
gemm_tf32x3.cu), checked through the C ABI against exact or float64 restatements computed from the same fp32 inputs the
kernels read (DESIGN.md §2, §4.13):

* the sampler equals oracle/gcrd.sample_perm, a CPU Philox restatement, element for element, ties included, eagerly and
  replayed from a CUDA graph with the device step counter advanced between replays;
* the row gather is bit-identical to X[idx] and to affine_relu_bits(Y, bits, scale, shift, p)[idx];
* the row-indexed GEMM stores exactly the plain GEMM's rows, on the vector and on the scalar epilogue, and leaves every
  other row alone;
* the operands and the backward obey elementwise bounds derived below from u = 2^-24, correctly rounded sqrtf, division
  and fmaf, and the length of each fp32 chain; the ReLU masks are exact; rows with norms on both sides of eps reach the
  clamped (clamp_min) branch, and the unclamped formula on those rows must violate the bound;
* every output and advertised buffer sits among NaN canaries that survive bit for bit, refusals launch nothing, and
  repeated calls are bit-identical;
* one engine step runs the clamped branch end to end and matches the fp64 oracle.

Worst observed ratio (error / bound) of each family on an H100 80GB HBM3 at a 700 W power limit (printed at the end of the
run): operands 0.54, backward 0.84, BatchNorm-backward slots 0.49, loss 0.60.  Every threshold is derived in a comment."""
import math

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.gcrd import GCRD, SAMPLE_STREAM
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import gcrd as og_gcrd, graph as og
from oracle.sampling import philox4x32

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# ----------------------------------------------------------------------------------------------------------- error model
U = 2.0 ** -24          # unit roundoff of fp32 round to nearest
TIGHT = 1e-5            # a well-conditioned random input must get a relative bound below this
EPS = float(torch.tensor(1e-12, dtype=torch.float32))     # the fp32 eps the kernels compare with (F.normalize)
INV_T = float(torch.tensor(1.0 / 0.075, dtype=torch.float32))
CANARY = 0x7FC0DEAD     # a quiet NaN with a payload: outside an output it must survive bit for bit
OK, ERR_BAD_ARG, ERR_UNSUPPORTED = 0, -1, -2

WORST = {}


def _g(k: float) -> float:
    """gamma(k) = k u / (1 - k u): k fp32 roundings in a product of (1 + delta) factors."""
    return k * U / (1 - k * U)


def _record(family: str, r: float) -> None:
    assert r <= 1.0, (family, r)
    WORST[family] = max(WORST.get(family, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    print("\nworst bound ratio per family: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))


def _gen(seed: int) -> torch.Generator:
    return torch.Generator(device="cuda").manual_seed(seed)


def _pow2(n: int, g: torch.Generator, span: int) -> torch.Tensor:
    """n powers of two 2^e, e uniform in [-span, span]."""
    return torch.exp2(torch.randint(-span, span + 1, (n,), generator=g, device="cuda").double()).float()


def _canary(*shape) -> torch.Tensor:
    return torch.full(shape, CANARY, dtype=torch.int32, device="cuda").view(torch.float32)


def _canary_i32(*shape) -> torch.Tensor:
    return torch.full(shape, CANARY, dtype=torch.int32, device="cuda")


def _is_canary(t: torch.Tensor) -> bool:
    return bool((t.contiguous().view(torch.int32) == CANARY).all())


def _bits_equal(a: torch.Tensor, b: torch.Tensor) -> bool:
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _bound_ratio(out: torch.Tensor, ref: torch.Tensor, bound: torch.Tensor) -> float:
    """max |out - ref| / bound (<= 1 passes); a zero bound demands an exact result."""
    assert bool(torch.isfinite(out).all()), "non-finite output"
    err = (out.double() - ref).abs()
    r = torch.where(bound > 0, err / bound, torch.where(err > 0, math.inf, 0.0))
    return float(r.max()) if r.numel() else 0.0


def _tight(bound: torch.Tensor, mag: torch.Tensor) -> None:
    m = mag > 0
    assert float((bound[m] / mag[m]).max()) < TIGHT


def _ceil(a, b):
    return -(-a // b)


def _L():
    return lib.load()


def _st():
    return lib.stream_ptr()


def _p(t):
    return None if t is None else t.data_ptr()


def _refused(call, code=ERR_BAD_ARG):
    """The call returns `code` and launches nothing."""
    torch.cuda.synchronize()
    before = lib.launch_count()
    assert call() == code
    assert lib.launch_count() == before


# ============================================================================================ 1. the row sampler
SAMPLE_N = [1, 2, 3, 4, 5, 255, 256, 257, 4097, 90_941, (1 << 20) + 3]


def _sample(n, seed, offset, step=None):
    """b200gnn_gcrd_sample_i32 into a canary-tailed perm; the workspace tail past its advertised size is checked too."""
    L = _L()
    wsb = int(L.b200gnn_gcrd_sample_workspace_bytes(n))
    ws_words = _ceil(wsb, 4)
    ws = _canary_i32(ws_words + 64)
    perm = _canary_i32(n + 8)
    st = None if step is None else torch.tensor([step], dtype=torch.int32, device="cuda")
    lib.check(L.b200gnn_gcrd_sample_i32(n, seed, offset, _p(st), perm.data_ptr(), ws.data_ptr(), _st()), "sample")
    torch.cuda.synchronize()
    assert _is_canary(perm[n:]) and _is_canary(ws[ws_words:])
    return perm[:n].long().cpu().numpy()


@pytest.mark.parametrize("n", SAMPLE_N)
def test_sampler_equals_cpu_restatement(n):
    """Every position of the permutation, at the G-CRD stream and a small offset, with no counter and with a device counter
    at several steps (the key offset is offset + *step_dev)."""
    seed = 0x9E3779B97F4A7C15 ^ n                          # both 32-bit halves of the Philox key in use
    for offset, step in ((SAMPLE_STREAM, None), (SAMPLE_STREAM, 0), (SAMPLE_STREAM, 1), (SAMPLE_STREAM, 977),
                         (5, None), (5, 3)):
        got = _sample(n, seed, offset, step)
        ref = og_gcrd.sample_perm(n, seed, offset + (step or 0))
        assert np.array_equal(got, ref), (n, offset, step)
    assert np.array_equal(_sample(n, seed, 5, 3), got)                   # repeated calls: the same permutation
    _refused(lambda: _L().b200gnn_gcrd_sample_i32(0, seed, 5, None, got.ctypes.data, got.ctypes.data, _st()))


def _seed_with_tie(n, offset):
    for seed in range(64):
        key = philox4x32(seed, offset, np.arange(_ceil(n, 4), dtype=np.uint64)).reshape(-1)[:n]
        if np.unique(key).size < n:
            return seed
    raise AssertionError("no tied keys in 64 seeds")


def test_sampler_ties_go_to_the_lower_row():
    """A seed whose 90,941 keys contain an equal pair (found on the CPU): the GPU order is the restatement's, and a restatement
    that orders ties toward the higher row differs on it, so the tie is really exercised."""
    n = 90_941
    seed = _seed_with_tie(n, SAMPLE_STREAM)
    got = _sample(n, seed, SAMPLE_STREAM, 0)
    assert np.array_equal(got, og_gcrd.sample_perm(n, seed, SAMPLE_STREAM))
    assert not np.array_equal(got, og_gcrd.sample_perm(n, seed, SAMPLE_STREAM, tie_to_higher=True))


def test_sampler_in_a_cuda_graph_reads_the_counter_at_replay():
    """The sample launch alone captured in a CUDA graph; the device counter advanced between replays: replay k draws
    sample_perm(n, seed, offset + k)."""
    n, seed = 90_941, 12345
    L = _L()
    wsb = int(L.b200gnn_gcrd_sample_workspace_bytes(n))
    ws = _canary_i32(_ceil(wsb, 4) + 64)
    perm = _canary_i32(n + 8)
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        rc = L.b200gnn_gcrd_sample_i32(n, seed, SAMPLE_STREAM, step.data_ptr(), perm.data_ptr(), ws.data_ptr(), _st())
    assert rc == OK
    for k in range(4):
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(perm[:n].long().cpu().numpy(), og_gcrd.sample_perm(n, seed, SAMPLE_STREAM + k)), k
        assert _is_canary(perm[n:]) and _is_canary(ws[_ceil(wsb, 4):])
        step.add_(1)


# ====================================================================================== 2. gather_rows_act (exact)
GATHER_K = [4, 28, 32, 36, 100, 256, 512]


def _gather(X, ldx, idx, K, bits=None, scale=None, shift=None, p=0.0):
    n_idx = idx.numel()
    out = _canary(n_idx * K + 8)
    lib.check(_L().b200gnn_gather_rows_act_f32(X.data_ptr(), ldx, idx.data_ptr(), n_idx, K, _p(bits), _p(scale), _p(shift), p,
                                              out.data_ptr(), _st()), "gather")
    torch.cuda.synchronize()
    assert _is_canary(out[n_idx * K:])
    return out[:n_idx * K].view(n_idx, K)


@pytest.mark.parametrize("K", GATHER_K)
@pytest.mark.parametrize("p", [0.0, 0.5])
def test_gather_rows_act_bit_exact(K, p):
    """out == X[idx] without bits, == affine_relu_bits(Y, bits, scale, shift, p)[idx] with them: K with a partial last keep
    word and K % 32 != 0, a pitched X whose trailing NaN columns must not leak, idx unsorted with duplicates naming the
    first and last row."""
    g = _gen(31 * K + int(4 * p))
    n_rows, n_idx = 777, 1500
    words = _ceil(K, 32)
    idx = torch.randint(0, n_rows, (n_idx,), generator=g, device="cuda")
    idx[0], idx[1], idx[n_idx - 1] = n_rows - 1, 0, n_rows - 1
    bits = torch.randint(-2 ** 31, 2 ** 31, (n_rows * words,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    scale = torch.randn(K, generator=g, device="cuda")
    shift = torch.randn(K, generator=g, device="cuda")
    for ldx in (K, K + 8):
        X = torch.full((n_rows, ldx), float("nan"), device="cuda")
        X[:, :K] = torch.randn(n_rows, K, generator=g, device="cuda") * _pow2(n_rows, g, 10)[:, None]
        Y = X[:, :K].contiguous()
        assert _bits_equal(_gather(X, ldx, idx, K), Y[idx])
        ref = _canary(n_rows * K + 8)
        lib.check(_L().b200gnn_affine_relu_bits_f32(Y.data_ptr(), bits.data_ptr(), scale.data_ptr(), shift.data_ptr(), p,
                                                   ref.data_ptr(), n_rows, K, _st()), "affine_relu_bits")
        act = _gather(X, ldx, idx, K, bits, scale, shift, p)
        assert _bits_equal(act, ref[:n_rows * K].view(n_rows, K)[idx])
        assert _bits_equal(_gather(X, ldx, idx, K, bits, scale, shift, p), act)          # repeated call
        assert bool((act == 0).any()) and bool((act > 0).any())


def test_gather_rows_act_refusals_and_empty():
    K, n = 32, 16
    X = torch.randn(n + 1, K, device="cuda")
    idx = torch.arange(n, device="cuda")
    bits = torch.full((n,), -1, dtype=torch.int32, device="cuda")
    sc, sh = torch.ones(K + 4, device="cuda"), torch.zeros(K + 4, device="cuda")
    out = _canary(n * K + 8)
    L, o = _L(), out.data_ptr()

    def call(Xp=X.data_ptr(), ldx=K, b=None, s=None, h=None, p=0.0, op=o, n_idx=n):
        return L.b200gnn_gather_rows_act_f32(Xp, ldx, idx.data_ptr(), n_idx, K, b, s, h, p, op, _st())
    _refused(lambda: call(ldx=K - 4))                                           # ldx < K
    _refused(lambda: call(ldx=K + 2))                                           # ldx % 4
    _refused(lambda: call(Xp=X.data_ptr() + 4))                                 # misaligned X
    _refused(lambda: call(op=o + 4))                                            # misaligned out
    _refused(lambda: call(b=bits.data_ptr(), s=sc.data_ptr() + 4, h=sh.data_ptr()))
    _refused(lambda: call(b=bits.data_ptr(), s=sc.data_ptr(), h=sh.data_ptr() + 4))
    _refused(lambda: call(p=1.0))
    _refused(lambda: call(p=1.5))
    _refused(lambda: call(b=bits.data_ptr(), h=sh.data_ptr()))                  # bits without scale
    _refused(lambda: call(b=bits.data_ptr(), s=sc.data_ptr()))                  # bits without shift
    _refused(lambda: call(n_idx=0), OK)                                         # nothing to gather: OK, no launch
    torch.cuda.synchronize()
    assert _is_canary(out)


# ============================================================================= 3. gemm_tf32x3_rowidx (exact vs plain)
# The row-indexed entry dispatches the same Cfg as b200gnn_gemm_tf32x3_f32 (Cfg<48,6> for N <= 48, else Cfg<128,4>) and
# has no split-K; only the row a tile row is stored to differs.  So C[row_idx] must equal the plain GEMM bit for bit, whose
# own accuracy test_gemm_numerics_gpu.py bounds.
GEMM_N = [4, 36, 48, 49, 64, 100, 128, 129, 256, 512]
GEMM_M = [1, 127, 128, 129, 45_471, 90_941]


def _split(W):
    N, K = W.shape
    hi, lo = torch.empty_like(W), torch.empty_like(W)
    lib.check(_L().b200gnn_split_tf32_f32(W.data_ptr(), N, K, 0, hi.data_ptr(), lo.data_ptr(), _st()), "split")
    return hi, lo


def _gemm_pair(A, hi, lo, M, N, K, ldc, off, row_idx, rows_C):
    """(plain GEMM into [M, ldc] at float offset off, row-indexed GEMM into [rows_C, ldc] at the same offset), both
    buffers canary-filled around and between the stored elements."""
    L = _L()
    plain = _canary(M * ldc + off + 8)
    lib.check(L.b200gnn_gemm_tf32x3_f32(A.data_ptr(), K, hi.data_ptr(), lo.data_ptr(), K, plain.data_ptr() + 4 * off, ldc, M, N,
                                        K, None, _st()), "gemm")
    C = _canary(rows_C * ldc + off + 8)
    lib.check(L.b200gnn_gemm_tf32x3_rowidx_f32(A.data_ptr(), K, hi.data_ptr(), lo.data_ptr(), K, C.data_ptr() + 4 * off, ldc,
                                               M, N, K, row_idx.data_ptr(), _st()), "gemm_rowidx")
    torch.cuda.synchronize()
    assert _is_canary(plain[:off]) and _is_canary(plain[off + M * ldc:]) and _is_canary(plain[off:off + M * ldc].view(M, ldc)[:, N:])
    assert _is_canary(C[:off]) and _is_canary(C[off + rows_C * ldc:])
    return plain[off:off + M * ldc].view(M, ldc), C, C[off:off + rows_C * ldc].view(rows_C, ldc)


def _check_rowidx(plain, Cv, row_idx, rows_C):
    assert _bits_equal(Cv[row_idx], plain)                       # columns [N, ldc) of both are canaries too
    untouched = torch.ones(rows_C, dtype=torch.bool, device="cuda")
    untouched[row_idx] = False
    assert _is_canary(Cv[untouched])


@pytest.mark.parametrize("M", GEMM_M)
@pytest.mark.parametrize("N", GEMM_N)
def test_gemm_rowidx_equals_plain_gemm(N, M):
    """ldc > N (columns past N stay canaries), row_idx a random permutation of distinct rows and a sorted train_idx-like
    subset of a larger C; rows not named keep their canaries; repeated calls are bit-identical."""
    g = _gen(N * 100_003 + M)
    rows_C = M + M // 2 + 3
    ldc = _ceil(N, 4) * 4 + 4
    for K in (64, 256):
        A = torch.randn(M, K, generator=g, device="cuda") * _pow2(M, g, 10)[:, None]
        hi, lo = _split(torch.randn(N, K, generator=g, device="cuda"))
        pick = torch.randperm(rows_C, generator=g, device="cuda")[:M]
        for row_idx in (pick, pick.sort().values):
            plain, C, Cv = _gemm_pair(A, hi, lo, M, N, K, ldc, 0, row_idx, rows_C)
            _check_rowidx(plain, Cv, row_idx, rows_C)
        _, C2, _ = _gemm_pair(A, hi, lo, M, N, K, ldc, 0, row_idx, rows_C)
        assert _bits_equal(C2, C)


@pytest.mark.parametrize("N", GEMM_N)
@pytest.mark.parametrize("M", [129, 45_471])
def test_gemm_rowidx_scalar_epilogue(N, M):
    """ldc odd, and C one float off 16-byte alignment: the ragged scalar epilogue stores every element, and the result
    equals the plain GEMM stored the same way."""
    g = _gen(7 * N + M)
    rows_C = M + 77
    K = 64
    A = torch.randn(M, K, generator=g, device="cuda")
    hi, lo = _split(torch.randn(N, K, generator=g, device="cuda"))
    row_idx = torch.randperm(rows_C, generator=g, device="cuda")[:M]
    odd = N + 1 + N % 2
    for ldc, off in ((odd, 0), (odd, 1), (_ceil(N, 4) * 4 + 4, 1)):
        plain, _, Cv = _gemm_pair(A, hi, lo, M, N, K, ldc, off, row_idx, rows_C)
        _check_rowidx(plain, Cv, row_idx, rows_C)


def test_gemm_rowidx_refusals():
    M, N, K = 64, 64, 64
    A = torch.randn(M + 1, K, device="cuda")
    hi, lo = _split(torch.randn(N + 1, K, device="cuda")[:N].contiguous())
    hi = torch.cat([hi.view(-1), torch.zeros(4, device="cuda")])
    lo = torch.cat([lo.view(-1), torch.zeros(4, device="cuda")])
    row_idx = torch.arange(M, device="cuda")
    C = _canary(M * N + 8)
    L = _L()

    def call(a=A.data_ptr(), h=hi.data_ptr(), l_=lo.data_ptr(), ldc=N, ri=row_idx.data_ptr()):
        return L.b200gnn_gemm_tf32x3_rowidx_f32(a, K, h, l_, K, C.data_ptr(), ldc, M, N, K, ri, _st())
    _refused(lambda: call(ri=None))
    _refused(lambda: call(ldc=N - 4))
    _refused(lambda: call(a=A.data_ptr() + 4), ERR_UNSUPPORTED)
    _refused(lambda: call(h=hi.data_ptr() + 4), ERR_UNSUPPORTED)
    _refused(lambda: call(l_=lo.data_ptr() + 4), ERR_UNSUPPORTED)
    torch.cuda.synchronize()
    assert _is_canary(C)


# ============================================================================================ 4. gcrd_operands
# operand_row, one warp per sampled row, lane c owning float4 chunks c and c + 32 (m = 4 terms per lane for P <= 128,
# 8 above), from the fp32 (pre, scale, shift) it reads:
#   a = max(fmaf(y, s, h), 0): one rounding of the exact y s + h (u relative), and fmaf's sign is the exact sign, so the
#     ReLU mask is exactly the fp64 one;
#   ss = sum a^2 by an m-long fma chain and a 5-level xor tree: positive terms, gamma(m + 5) relative, plus 2u from a's own
#     rounding: gamma(m + 7);
#   nrm = sqrtf(ss): half of that plus u:                  norm bound gamma(0.5 (m + 7) + 1) |nrm|;
#   inv = sc / max(nrm, eps): the norm's error (max is 1-Lipschitz, so rows on either side of eps obey it) plus u;
#   x = a inv: a's u, inv's, and the product's u:          x bound gamma(0.5 (m + 7) + 4) |x|.
# sc is the fp32 1/nce_T for the student, 1 for the teacher; the reference uses the same fp32 value.
P_LIST = [4, 12, 60, 64, 96, 100, 132, 252, 256]
S_LIST = [1, 7, 8, 9, 8447, 8448, 8449, 16384]
DESIGNED = [("zero", 0.0), ("tiny", 1e-14), ("under", 0.9e-12), ("over", 1.1e-12), ("on", 1e-12)]


def _lane_terms(P: int) -> int:
    return 4 if P <= 128 else 8


def _zero_shift_cols(P):
    return sorted({0, P // 3, P // 2, P - 1})


def _head_inputs(P, n_train, inds, g, designed_at):
    """pre [n_train, P], bn [4, P] = (mean, invstd, scale, shift) for one head.  Columns _zero_shift_cols have shift 0, so a
    designed row reaches any target norm there exactly: every other column is driven below zero."""
    pre = torch.randn(n_train, P, generator=g, device="cuda") * _pow2(n_train, g, 8)[:, None]
    s = torch.randn(P, generator=g, device="cuda") * _pow2(P, g, 4)
    h = torch.randn(P, generator=g, device="cuda") * _pow2(P, g, 4)
    zc = torch.tensor(_zero_shift_cols(P), device="cuda")
    h[zc] = 0
    mean = torch.randn(P, generator=g, device="cuda")
    invstd = torch.rand(P, generator=g, device="cuda") + 0.5
    for j, (_, target) in zip(designed_at, DESIGNED):
        y = -torch.sign(s) * (h.abs() + 1) / s.abs()                            # y s + h <= -1: ReLU closed
        if target > 0:
            y[zc] = target / math.sqrt(zc.numel()) / s[zc]
        pre[int(inds[j])] = y
    return pre, torch.stack([mean, invstd, s, h]).contiguous()


def _gcrd_problem(P, S, seed):
    g = _gen(seed)
    n_train = S + S // 3 + 5
    rest = torch.randperm(n_train - 2, generator=g, device="cuda")[:max(S - 2, 0)] + 1
    inds = torch.cat([torch.tensor([n_train - 1, 0], device="cuda")[:S], rest])
    inds = inds[torch.randperm(S, generator=g, device="cuda")].to(torch.int32).contiguous()
    # designed rows: the student's at sampled positions 1..5, the teacher's at 6..2 (other kinds on the same rows)
    ds = list(range(1, 6)) if S >= 7 else []
    dt = list(range(6, 1, -1)) if S >= 7 else []
    pre_s, bn_s = _head_inputs(P, n_train, inds, g, ds)
    pre_t, bn_t = _head_inputs(P, n_train, inds, g, dt)
    return dict(P=P, S=S, n_train=n_train, inds=inds, pre_s=pre_s, bn_s=bn_s, pre_t=pre_t, bn_t=bn_t, ds=ds, dt=dt, g=g)


def _operands(pb, reps=1):
    P, S = pb["P"], pb["S"]
    outs = []
    for _ in range(reps):
        x_s, x_t, n_s, n_t = _canary(S + 2, P), _canary(S + 2, P), _canary(S + 4), _canary(S + 4)
        lib.check(_L().b200gnn_gcrd_operands_f32(pb["inds"].data_ptr(), S, P, pb["pre_s"].data_ptr(), pb["bn_s"].data_ptr(),
                                                pb["pre_t"].data_ptr(), pb["bn_t"].data_ptr(), INV_T, EPS, x_s.data_ptr(),
                                                x_t.data_ptr(), n_s.data_ptr(), n_t.data_ptr(), _st()), "operands")
        torch.cuda.synchronize()
        # padding: rows of x past S are never written (GCRD relies on its zero padding rows staying zero)
        assert _is_canary(x_s[S:]) and _is_canary(x_t[S:]) and _is_canary(n_s[S:]) and _is_canary(n_t[S:])
        outs.append((x_s[:S], x_t[:S], n_s[:S], n_t[:S]))
    for o in outs[1:]:
        assert all(_bits_equal(a, b) for a, b in zip(o, outs[0]))
    return outs[0]


def _act64(pre, bn, inds):
    return (pre[inds.long()].double() * bn[2].double() + bn[3].double()).clamp_min(0)


def _operand_ref(pre, bn, inds, sc, P):
    a = _act64(pre, bn, inds)
    nrm = a.norm(dim=1)
    x = a * sc / nrm.clamp_min(EPS)[:, None]
    m = _lane_terms(P)
    return a, x, _g(0.5 * (m + 7) + 4) * x.abs(), nrm, _g(0.5 * (m + 7) + 1) * nrm


@pytest.mark.parametrize("S", S_LIST)
@pytest.mark.parametrize("P", P_LIST)
def test_operands_elementwise(P, S):
    """Partial lane chunk sets (P = 12, 60, 96, 100, 132, 252), the grid-stride loop past 1056 x 8 rows, designed rows
    around eps, distinct heads (swapping them fails: different inputs and scales)."""
    pb = _gcrd_problem(P, S, 1000 * P + S)
    x_s, x_t, n_s, n_t = _operands(pb, reps=2)
    r = 0.0
    for x, nrm, pre, bn, sc, designed in ((x_s, n_s, pb["pre_s"], pb["bn_s"], INV_T, pb["ds"]),
                                          (x_t, n_t, pb["pre_t"], pb["bn_t"], 1.0, pb["dt"])):
        a, xr, xb, nr, nb = _operand_ref(pre, bn, pb["inds"], sc, P)
        assert torch.equal(x == 0, a == 0)                                     # the ReLU mask is exact
        r = max(r, _bound_ratio(x, xr, xb), _bound_ratio(nrm, nr, nb))
        if designed:                                                           # the designed rows land where intended
            kinds = dict(zip((d[0] for d in DESIGNED), designed))
            assert float(nrm[kinds["zero"]]) == 0 and 0 < float(nrm[kinds["tiny"]]) < EPS
            assert float(nrm[kinds["under"]]) < EPS < float(nrm[kinds["over"]])
        keep = torch.ones(S, dtype=torch.bool, device="cuda")
        keep[designed] = False
        _tight(xb[keep], xr.abs()[keep])
    _record("operands", r)


def test_operands_refusals():
    pb = _gcrd_problem(64, 9, 5)
    S = pb["S"]
    x_s, x_t, n_s, n_t = _canary(S + 2, 260), _canary(S + 2, 260), _canary(S + 4), _canary(S + 4)
    L = _L()
    ptr = dict(pre_s=pb["pre_s"].data_ptr(), bn_s=pb["bn_s"].data_ptr(), pre_t=pb["pre_t"].data_ptr(), bn_t=pb["bn_t"].data_ptr(),
               x_s=x_s.data_ptr(), x_t=x_t.data_ptr())

    def call(P=64, inv_T=INV_T, S_=S, **over):
        q = dict(ptr, **over)
        return L.b200gnn_gcrd_operands_f32(pb["inds"].data_ptr(), S_, P, q["pre_s"], q["bn_s"], q["pre_t"], q["bn_t"], inv_T,
                                           EPS, q["x_s"], q["x_t"], n_s.data_ptr(), n_t.data_ptr(), _st())
    for P in (0, 2, 6, 66, 258, 260):
        _refused(lambda: call(P=P))
    for inv_T in (0.0, -1.0, float("nan")):
        _refused(lambda: call(inv_T=inv_T))
    _refused(lambda: call(S_=0))
    for k in ptr:
        _refused(lambda: call(**{k: ptr[k] + 4}))
    torch.cuda.synchronize()
    assert _is_canary(x_s) and _is_canary(x_t) and _is_canary(n_s) and _is_canary(n_t)


# ============================================================================================ 5. gcrd_backward
# head_bwd, from the fp32 (x, norm, g) it reads, per sampled row j (row r = inds[j]) and the same m terms per lane:
#   u_k = x_k (1/sc): the fp32 reciprocal and the product, 2u relative to uu = x / sc;
#   dot = sum u g by an m-long fma chain and a 5-level tree: dot_err = gamma(m + 7) sum |uu g|;
#   inv = sc / max(norm, eps): u;
#   unclamped (norm >= eps): v = inv (g - u_k dot): the product u_k dot carries |uu| dot_err + gamma(3) |uu dot|, the
#     difference and the product with inv one rounding each and inv one more:  vb = inv (|uu| dot_err + gamma(3)|uu dot|)
#     + gamma(3) |v|   (the _norm_bwd_ref form of test_loss_kernels_gpu.py, with u = x / sc);
#   clamped (norm < eps, the clamp_min gradient): v = g inv: gamma(2) |v|;
#   dz = mask ? v beta : 0, mask = fmaf(y, s, h) > 0 (exactly the fp64 sign): |beta| vb (1 + u) + u |beta v|.
# Slots (pass 1 of the BatchNorm backward), warp gw of 512 taking rows j = gw, gw + 512, ...: c = ceil(S / 512) additions
# of the stored fp32 dz per slot: gamma(c) sum |dz|; the dz xhat column with xhat = (y - mean) invstd in two fp32
# roundings (restated in fp32, so exactly the kernel's) and one more for the product: gamma(c + 1) sum |dz xhat|.
# Loss: loss_total + beta loss_aux in two roundings, or one if the compiler contracts it to an fma: gamma(1) |beta la|
# + gamma(1) |result|.
BETA = float(torch.tensor(0.3, dtype=torch.float32))


def _bwd_ref(x, nrm, gg, sc, P):
    o, nr, gd = x.double(), nrm.double()[:, None], gg.double()
    m = _lane_terms(P)
    uu = o / sc
    dot = (uu * gd).sum(1, keepdim=True)
    dot_err = _g(m + 7) * (uu * gd).abs().sum(1, keepdim=True)
    inv = sc / nr.clamp_min(EPS)
    clamped = nr < EPS
    v_un = inv * (gd - uu * dot)
    vb_un = inv * (uu.abs() * dot_err + _g(3) * (uu * dot).abs()) + _g(3) * v_un.abs()
    v = torch.where(clamped, gd * inv, v_un)
    vb = torch.where(clamped, _g(2) * v.abs(), vb_un)
    mag = torch.where(clamped, v.abs(), inv * (gd.abs() + uu.abs() * (uu * gd).abs().sum(1, keepdim=True)))
    return v, vb, mag, v_un, clamped[:, 0]


def _backward(pb, ops_out, g_s, g_t, with_loss=True):
    P, S, n = pb["P"], pb["S"], pb["n_train"]
    x_s, x_t, n_s, n_t = ops_out
    slots = int(_L().b200gnn_gcrd_bwd_slots())
    dz_s, dz_t = _canary(n + 1, P), _canary(n + 1, P)
    part_s, part_t = _canary(slots * 2 * P + 8), _canary(slots * 2 * P + 8)
    loss_aux = torch.tensor([2.7], device="cuda")
    loss = _canary(4)
    loss[0] = 1.3
    lib.check(_L().b200gnn_gcrd_backward_f32(pb["inds"].data_ptr(), S, P, g_s.data_ptr(), g_t.data_ptr(), x_s.data_ptr(),
                                            x_t.data_ptr(), n_s.data_ptr(), n_t.data_ptr(), INV_T, EPS, pb["pre_s"].data_ptr(),
                                            pb["bn_s"].data_ptr(), pb["pre_t"].data_ptr(), pb["bn_t"].data_ptr(), BETA,
                                            dz_s.data_ptr(), dz_t.data_ptr(), part_s.data_ptr(), part_t.data_ptr(),
                                            loss_aux.data_ptr(), loss.data_ptr() if with_loss else None, _st()), "backward")
    torch.cuda.synchronize()
    assert _is_canary(part_s[slots * 2 * P:]) and _is_canary(part_t[slots * 2 * P:]) and _is_canary(loss[1:])
    assert float(loss_aux[0]) == float(torch.tensor(2.7))
    return dz_s, dz_t, part_s[:slots * 2 * P].view(slots, 2, P), part_t[:slots * 2 * P].view(slots, 2, P), loss


@pytest.mark.parametrize("S", S_LIST)
@pytest.mark.parametrize("P", P_LIST)
def test_backward_elementwise(P, S):
    pb = _gcrd_problem(P, S, 1000 * P + S)
    g = pb["g"]
    ops_out = _operands(pb)
    g_s = torch.randn(S, P, generator=g, device="cuda") * _pow2(S, g, 6)[:, None]
    g_t = torch.randn(S, P, generator=g, device="cuda") * _pow2(S, g, 6)[:, None]
    dz_s, dz_t, part_s, part_t, loss = _backward(pb, ops_out, g_s, g_t)
    inds = pb["inds"].long()
    n = pb["n_train"]
    sampled = torch.zeros(n + 1, dtype=torch.bool, device="cuda")
    sampled[inds] = True
    slots = part_s.shape[0]
    c = _ceil(S, slots)
    slot_of = torch.arange(S, device="cuda") % slots
    r = rs = 0.0
    for dz, part, x, nrm, gg, pre, bn, sc, designed in (
            (dz_s, part_s, ops_out[0], ops_out[2], g_s, pb["pre_s"], pb["bn_s"], INV_T, pb["ds"]),
            (dz_t, part_t, ops_out[1], ops_out[3], g_t, pb["pre_t"], pb["bn_t"], 1.0, pb["dt"])):
        assert _is_canary(dz[~sampled])                                        # rows not sampled are never stored
        got = dz[inds]
        v, vb, mag, v_un, clamped = _bwd_ref(x, nrm, gg, sc, P)
        mask = _act64(pre, bn, pb["inds"]) > 0
        ref = torch.where(mask, v * BETA, 0.0)
        bound = torch.where(mask, abs(BETA) * vb * (1 + U) + U * (BETA * v).abs(), 0.0)
        # the ReLU mask is exact: closed elements are exact zeros (open ones may cancel to 0 in fp32: a row with one open
        # element has u_k = 1 and g - u_k dot = 0, where fp64 keeps a rounding-sized remainder inside the bound)
        assert not bool(got[~mask].any())
        r = max(r, _bound_ratio(got, ref, bound))
        keep = torch.ones(S, dtype=torch.bool, device="cuda")
        keep[designed] = False
        _tight(bound[keep][mask[keep]], (abs(BETA) * mag)[keep][mask[keep]])
        if designed:
            # negative control: on the clamped rows with a nonzero norm, the unclamped formula violates the bound, so the
            # clamped branch is what the kernel ran
            probe = clamped & (nrm > 0)
            assert int(probe.sum()) >= 2
            un = torch.where(mask, v_un * BETA, 0.0)
            assert _bound_ratio(got[probe], un[probe], bound[probe]) > 1
        # the 512 slots against fp64 column sums of the stored dz and dz xhat
        y = pre[inds]
        xhat = (y - bn[0]) * bn[1]
        s64 = torch.zeros(slots, P, dtype=torch.float64, device="cuda").index_add_(0, slot_of, got.double())
        sa = torch.zeros_like(s64).index_add_(0, slot_of, got.double().abs())
        q = got.double() * xhat.double()
        q64 = torch.zeros_like(s64).index_add_(0, slot_of, q)
        qa = torch.zeros_like(s64).index_add_(0, slot_of, q.abs())
        rs = max(rs, _bound_ratio(part[:, 0], s64, _g(c) * sa), _bound_ratio(part[:, 1], q64, _g(c + 1) * qa))
        if S < slots:                                                          # warps with no rows store exact zeros
            assert not bool(part[S:].any())
    la, lt = float(torch.tensor(2.7)), 1.3
    lt32 = float(torch.tensor(lt))
    ref_l = lt32 + BETA * la
    _record("loss", _bound_ratio(loss[:1], torch.tensor([ref_l], dtype=torch.float64, device="cuda"),
                                 torch.tensor([_g(1) * abs(BETA * la) + _g(1) * abs(ref_l)], dtype=torch.float64, device="cuda")))
    # repeated call with loss_total = NULL: every output bit-identical, the loss left as it was
    again = _backward(pb, ops_out, g_s, g_t, with_loss=False)
    assert all(_bits_equal(a, b) for a, b in zip(again[:4], (dz_s, dz_t, part_s, part_t)))
    assert float(again[4][0]) == float(torch.tensor(lt))
    _record("backward", r)
    _record("bn_slots", rs)


def test_backward_refusals():
    pb = _gcrd_problem(64, 9, 6)
    P, S, n = 64, 9, pb["n_train"]
    x_s, x_t, n_s, n_t = _operands(pb)
    g_s, g_t = torch.randn(S, P, device="cuda"), torch.randn(S, P, device="cuda")
    slots = int(_L().b200gnn_gcrd_bwd_slots())
    dz_s, dz_t = _canary(n + 1, P), _canary(n + 1, P)
    part_s, part_t = _canary(slots * 2 * P + 8), _canary(slots * 2 * P + 8)
    loss_aux, loss = torch.ones(1, device="cuda"), torch.ones(1, device="cuda")
    names = ["g_s", "g_t", "x_s", "x_t", "pre_s", "pre_t", "bn_s", "bn_t", "dz_s", "dz_t", "part_s", "part_t"]
    ptr = dict(g_s=g_s, g_t=g_t, x_s=x_s, x_t=x_t, pre_s=pb["pre_s"], pre_t=pb["pre_t"], bn_s=pb["bn_s"], bn_t=pb["bn_t"],
               dz_s=dz_s, dz_t=dz_t, part_s=part_s, part_t=part_t)
    ptr = {k: v.data_ptr() for k, v in ptr.items()}
    L = _L()

    def call(la=loss_aux.data_ptr(), lt=loss.data_ptr(), **over):
        q = dict(ptr, **over)
        return L.b200gnn_gcrd_backward_f32(pb["inds"].data_ptr(), S, P, q["g_s"], q["g_t"], q["x_s"], q["x_t"], n_s.data_ptr(),
                                           n_t.data_ptr(), INV_T, EPS, q["pre_s"], q["bn_s"], q["pre_t"], q["bn_t"], BETA,
                                           q["dz_s"], q["dz_t"], q["part_s"], q["part_t"], la, lt, _st())
    _refused(lambda: call(la=None))                                             # loss_total without loss_aux
    for k in names:                                                            # each of the twelve 16-byte operands
        _refused(lambda: call(**{k: ptr[k] + 4}))
    torch.cuda.synchronize()
    assert _is_canary(dz_s) and _is_canary(dz_t) and _is_canary(part_s) and _is_canary(part_t) and float(loss[0]) == 1.0


# ============================================================================= 6. one engine step through the clamp
def _rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    d = b.abs().max().item()
    return (a - b).abs().max().item() / (d if d > 0 else 1.0)


def test_engine_step_through_the_clamped_branch():
    """Student head gamma = 0, beta = 1e-14: every projected student row is the same positive vector of norm 8e-14 < eps, so
    the clamped branch runs end to end with its ReLU mask open.  Every gradient matches the fp64 oracle at the whole-step
    tolerance, and the student head's d gamma and d beta, carried only by the clamped formula, are nonzero."""
    dims, p, beta, nce_T, S = (32, 64, 64, 8), 0.5, 0.5, 0.075, 256
    n = 3000
    ei = skewed_edges(n, 20_000, 0)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(n, dims[0], generator=gen)
    y = torch.randint(0, dims[-1], (n,), generator=gen)
    t = torch.randn(n, dims[-1], generator=gen) * 2
    idx = torch.randperm(n, generator=gen)[: n // 2].sort().values
    t_feat = torch.randn(n, 90, generator=gen).relu()
    head = GCRD(t_feat.cuda(), idx.cuda(), dims[-2], proj_dim=64, max_samples=S, nce_T=nce_T, beta=beta, seed=3)
    head.gamma_s.zero_()
    head.beta_s.fill_(1e-14)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    tr = GCNStudentTrainer(adj, list(dims), dropout=p, lr=0.01, seed=0, gcrd=head)
    init = (tr.state_dict(), head.student_proj_state_dict(), head.teacher_proj_state_dict())
    masks = [ops.dropout_mask(n, dims[l + 1], p, tr.seed, tr.dropout_offset(l, 0)).cpu().bool() for l in range(tr.L - 1)]
    sample = torch.as_tensor(np.random.RandomState(4).choice(idx.numel(), S, replace=False))
    loss = tr.train_step(x.cuda(), y.cuda(), idx.cuda(), t.cuda(), sample=sample).cpu()
    assert bool((head.norm_s < EPS).all()) and bool((head.norm_s > 0).all())     # every student row took the clamp
    rr, cc, vv = og.gcn_norm(r, c, n)
    cpu = lambda sd: {k: v.cpu() for k, v in sd.items()}
    ref = og_gcrd.gcrd_step("gcn", x, torch.from_numpy(og.ind2ptr(rr, n)), torch.from_numpy(cc), torch.from_numpy(vv),
                            cpu(init[0]), cpu(init[1]), cpu(init[2]), y, idx, t_feat, t, sample, beta, nce_T, masks=masks, p=p)
    assert abs(float(loss[0]) - ref["loss"]) < 2e-5 * abs(ref["loss"])
    assert abs(float(head.loss_aux) - ref["loss_aux"]) < 2e-5 * abs(ref["loss_aux"])
    got = {"sproj": {"0.weight": head.gW_s, "0.bias": head.gb_s, "1.weight": head.ggamma_s, "1.bias": head.gbeta_s},
           "tproj": {"0.weight": head.gW_t[:, :head.F_t], "0.bias": head.gb_t, "1.weight": head.ggamma_t, "1.bias": head.gbeta_t},
           "model": {}}
    for l in range(tr.L):
        got["model"][f"convs.{l}.weight"], got["model"][f"convs.{l}.bias"] = tr.gW[l], tr.gb[l]
        if l < tr.L - 1:
            got["model"][f"bns.{l}.weight"], got["model"][f"bns.{l}.bias"] = tr.ggamma[l], tr.gbeta[l]
    for group, grads in ref["grads"].items():
        scale = max(g_.abs().max().item() for g_ in grads.values())
        for k, g_ in grads.items():
            a = got[group][k]
            pre_bn = k == "0.bias" if group != "model" else (k.endswith("bias") and k.startswith("convs.")
                                                             and not k.startswith(f"convs.{tr.L - 1}."))
            if pre_bn:                    # in front of a training-mode BatchNorm: exact gradient 0, rounding on both sides
                assert a.abs().max().item() < 1e-5 * scale, (group, k)
            else:
                assert _rel_err(a, g_.float()) < 1e-4, (group, k, _rel_err(a, g_.float()))
    assert float(head.ggamma_s.abs().max()) > 0 and float(head.gbeta_s.abs().max()) > 0
