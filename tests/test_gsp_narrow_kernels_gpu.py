"""The two kernels BatchGSP adds around the shared GSP pair pass: the student-only chunk entry
(b200gnn_gsp_pair_student_chunk_f32) against the student side of b200gnn_gsp_pair_chunk_f32 bit for bit, and the narrow
contraction (b200gnn_gsp_contract_narrow_f32) against an elementwise fp64 bound of dG . x, its chunking invariance, and its
refusals."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SLAB = lib.GSP_CONTRACT_SLAB


def f(t):
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------------ 1. student-only pair pass
@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
def test_student_chunk_equals_the_student_side_of_the_two_sided_pass(kernel):
    L, st = lib.load(), lib.stream_ptr()
    g = torch.Generator(device="cuda").manual_seed(kernel)
    S, ld = 301, 308
    xs, xt = torch.randn(S, 8, generator=g, device="cuda"), torch.randn(S, 12, generator=g, device="cuda")
    if kernel <= 1:
        xs, xt = torch.nn.functional.normalize(xs), torch.nn.functional.normalize(xt)
    Gs_full = torch.zeros(S, ld, device="cuda")
    Gt_full = torch.zeros(S, ld, device="cuda")
    Gs_full[:, :S], Gt_full[:, :S] = xs @ xs.t(), xt @ xt.t()
    Gs_full[:, S:], Gt_full[:, S:] = 7.0, 7.0                      # padding columns: both passes zero them
    ns, nt = xs.pow(2).sum(1).contiguous(), xt.pow(2).sum(1).contiguous()
    raw = kernel >= 2
    for r0, r in ((0, 64), (64, 100), (164, 137), (300, 1)):
        a_s, a_t = Gs_full[r0:r0 + r].clone(), Gt_full[r0:r0 + r].clone()
        b_s, b_t = a_s.clone(), a_t.clone()
        pa, pb = torch.full((S,), -1.0, device="cuda"), torch.full((S,), -1.0, device="cuda")
        ra, rb = torch.full((S,), -1.0, device="cuda"), torch.full((S,), -1.0, device="cuda")
        rt = torch.full((S,), -1.0, device="cuda")
        assert L.b200gnn_gsp_pair_chunk_f32(f(a_s), f(a_t), ld, r, S, r0, f(ns) if raw else None, f(nt) if raw else None,
                                            kernel, f(ra) if raw else None, f(rt) if raw else None, f(pa), st) == 0
        t_before = b_t.clone()
        assert L.b200gnn_gsp_pair_student_chunk_f32(f(b_s), f(b_t), ld, r, S, r0, f(ns) if raw else None,
                                                    f(nt) if raw else None, kernel, f(rb) if raw else None, f(pb), st) == 0
        torch.cuda.synchronize()
        assert torch.equal(a_s, b_s), (kernel, r0)
        assert torch.equal(pa, pb) and torch.equal(ra, rb), (kernel, r0)
        assert torch.equal(b_t, t_before), "the student-only pass must not write Gt"
        assert bool((pb[r0:r0 + r] != -1).all()) and bool((pb[:r0] == -1).all())


# ------------------------------------------------------------------------------------------------ 2. the contraction
def operands(n_rows, S, F, seed, ldg=None, ldx=None):
    """dG [n_rows, ldg] and x [S + 5, ldx] with NaN past column S of dG and past row S / column F of x (never read)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ldg, ldx = ldg or S + 3, ldx or F + 4
    dG = torch.full((n_rows, ldg), float("nan"), device="cuda")
    x = torch.full((S + 5, ldx), float("nan"), device="cuda")
    # non-dyadic values of mixed sign and a spread of magnitudes, so the order of the sums shows in the bits
    dG[:, :S] = torch.randn(n_rows, S, generator=g, device="cuda") * torch.rand(n_rows, 1, generator=g, device="cuda").exp()
    x[:S, :F] = torch.randn(S, F, generator=g, device="cuda") / 3
    return dG, x


def contract(dG, S, x, F, ldo=None, rows=None):
    n_rows = dG.shape[0] if rows is None else rows
    ldo = ldo or F
    out = torch.full((n_rows, ldo), -3.0, device="cuda")
    ws = ops.gsp_contract_workspace(n_rows, S, F, "cuda")
    ops.gsp_contract_narrow(dG[:n_rows], S, x[:, :F], out[:, :F], ws)
    return out


SHAPES = [(4, 100), (8, 255), (8, 256), (8, 257), (32, 1000), (32, 24576), (128, 700), (128, 3 * SLAB)]


@pytest.mark.parametrize("F,S", SHAPES)
def test_contraction_within_the_fp64_bound(F, S):
    """|g - dG . x| <= (S + 2) u sum_j |dG_ij| |x_jf| elementwise: one fp32 rounding per FMA along a slab, one per slab
    added, with the NaN padding (columns of dG past S, rows of x past S, x's columns past F) never read."""
    n_rows = 70
    dG, x = operands(n_rows, S, F, seed=F + S, ldx=F + 8)
    out = contract(dG, S, x, F, ldo=F + 4)
    torch.cuda.synchronize()
    assert bool((out[:, F:] == -3.0).all()), "columns past F of the output must stay untouched"
    got = out[:, :F].double()
    A, X = dG[:, :S].double(), x[:S, :F].double()
    ref, mag = A @ X, A.abs() @ X.abs()
    assert bool(torch.isfinite(got).all())
    ratio = ((got - ref).abs() / ((S + 2) * U * mag)).max().item()
    assert ratio <= 1.0, (F, S, ratio)


@pytest.mark.parametrize("F,S", [(8, 255), (32, 1000), (32, 24576), (128, 3 * SLAB + 1)])
def test_contraction_bits_do_not_depend_on_the_chunking(F, S):
    """The same rows split into chunks in two ways, at other pitches, and a second run: the same bits."""
    n_rows = 200
    dG, x = operands(n_rows, S, F, seed=S)
    whole = contract(dG, S, x, F)
    again = contract(dG, S, x, F)
    dG2 = torch.full((n_rows, S + 11), float("nan"), device="cuda")
    dG2[:, :S] = dG[:, :S]
    pieces = torch.full((n_rows, F), -3.0, device="cuda")
    for r0, r in ((0, 1), (1, 37), (38, 128), (166, 34)):
        ws = ops.gsp_contract_workspace(r, S, F, "cuda")
        ops.gsp_contract_narrow(dG2[r0:r0 + r], S, x[:, :F], pieces[r0:r0 + r], ws)
    torch.cuda.synchronize()
    assert torch.equal(whole, again)
    assert torch.equal(whole, pieces)


def test_contraction_workspace_sizes():
    L = lib.load()
    assert L.b200gnn_gsp_contract_workspace_bytes(128, SLAB, 32) == 0
    assert L.b200gnn_gsp_contract_workspace_bytes(128, SLAB + 1, 32) == 2 * 128 * 32 * 4
    assert L.b200gnn_gsp_contract_workspace_bytes(128, 24576, 32) == 96 * 128 * 32 * 4
    assert L.b200gnn_gsp_contract_workspace_bytes(0, 24576, 32) == 0


def test_contraction_refusals_write_nothing():
    L, st = lib.load(), lib.stream_ptr()
    S, F, n = 600, 32, 40
    dG, x = operands(n, S, F, seed=1)
    out = torch.full((n, F), -3.0, device="cuda")
    need = int(L.b200gnn_gsp_contract_workspace_bytes(n, S, F))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    ok = dict(dG=f(dG), ldg=dG.stride(0), n=n, S=S, x=f(x), ldx=x.stride(0), F=F, g=f(out), ldo=F, ws=f(ws), wsb=need)
    bad = [dict(F=6), dict(F=132), dict(F=0), dict(ldg=S - 1), dict(ldx=F - 4), dict(ldo=F - 4), dict(dG=None), dict(x=None),
           dict(g=None), dict(ws=None), dict(wsb=need - 1), dict(n=0), dict(S=0), dict(g=f(out) + 2)]
    torch.cuda.synchronize()
    launches = lib.launch_count()
    for kw in bad:
        a = dict(ok, **kw)
        rc = L.b200gnn_gsp_contract_narrow_f32(a["dG"], a["ldg"], a["n"], a["S"], a["x"], a["ldx"], a["F"], a["g"], a["ldo"],
                                               a["ws"], a["wsb"], st)
        assert rc == -1, kw
    torch.cuda.synchronize()
    assert lib.launch_count() == launches and bool((out == -3.0).all())
    assert L.b200gnn_gsp_contract_narrow_f32(*ok.values(), st) == 0
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
