"""The fixed-teacher GSP kernels of csrc/loss_pair.cu through the C ABI: the similarity builder, the one-sided pair pass
against a stored teacher similarity matrix, and the plain-row operands and backward.

- The pair pass over a sim_t the builder made equals the student outputs of b200gnn_gsp_pair_chunk_f32 (dG_s, rc_s, the
  per-row partials) bit for bit, for the four kernels, several S and chunk sizes, with every row and with a sample.
- The builder is held to an fp64 bound of the same Gram entries.
- The rows operands and backward equal the eager row kernels (row_normalize / row_sqnorm / row_normalize_bwd / row_axpy)
  followed by the multiply by beta, bit for bit, including a zero row and a row under the eps clamp.
- Padding and unwritten rows are NaN canaries; bad arguments are refused with no launch."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion, lib

pytestmark = pytest.mark.gpu
KERNELS = [0, 1, 2, 3]
EPS = 1e-12
BAD = -1                                   # B200GNN_ERR_BAD_ARG
NAN = float("nan")


def L():
    return lib.load()


def p(t):
    return None if t is None else t.data_ptr()


def st():
    return lib.stream_ptr()


def operands(n, F, kernel, seed):
    """[n, F] rows as the pair passes see them: normalised for cosine / poly, raw (with their squared norms) for l2 / rbf,
    scaled so that rbf similarities stay well above underflow."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, F, generator=g).cuda()
    if kernel <= 1:
        return criterion._normalize(x)[0], None
    x = x * 0.3
    sq = torch.empty(n, device="cuda")
    assert L().b200gnn_row_sqnorm_f32(p(x), n, F, p(sq), st()) == 0
    return x, sq


def gram(x):
    return (x @ x.t()).contiguous()


def pad_cols(a, ld, fill=0.0):
    out = torch.full((a.shape[0], ld), fill, device="cuda")
    out[:, :a.shape[1]] = a
    return out


def both_pass(Gs, Gt, ns, nt, S, kernel):
    """The reference: b200gnn_gsp_pair_chunk_f32 over the whole S x S matrices in one chunk; the student outputs."""
    ld = (S + 3) // 4 * 4
    gs, gt = pad_cols(Gs, ld), pad_cols(Gt, ld)
    rc_s, rc_t, part = (torch.zeros(S, device="cuda") for _ in range(3))
    raw = kernel >= 2
    assert L().b200gnn_gsp_pair_chunk_f32(p(gs), p(gt), ld, S, S, 0, p(ns) if raw else None, p(nt) if raw else None, kernel,
                                          p(rc_s) if raw else None, p(rc_t) if raw else None, p(part), st()) == 0
    return gs[:, :S], rc_s, part


def build_sim(Gt, nt, kernel, R, ld_sim=None):
    n = Gt.shape[0]
    ld_sim = ld_sim or n
    sim = torch.full((n, ld_sim), NAN, device="cuda")
    ldg = (n + 3) // 4 * 4
    G = pad_cols(Gt, ldg, NAN)
    for r0 in range(0, n, R):
        r = min(R, n - r0)
        chunk = G[r0:r0 + r].clone()
        assert L().b200gnn_gsp_sim_chunk_f32(p(chunk), ldg, r, n, r0, p(nt) if kernel >= 2 else None, kernel, p(sim[r0]),
                                             ld_sim, st()) == 0
    return sim


def fixed_pass(Gs, ns, sim, S, kernel, R, inds=None):
    ld = (S + 3) // 4 * 4 + 4                 # a padded pitch wider than Sp: every padding column must come out zero
    out = torch.empty(S, ld, device="cuda")
    rc, part = torch.full((S + 8,), NAN, device="cuda"), torch.full((S + 8,), NAN, device="cuda")
    raw = kernel >= 2
    n_t, ld_t = sim.shape[0], sim.stride(0)
    for r0 in range(0, S, R):
        r = min(R, S - r0)
        chunk = torch.full((r, ld), NAN, device="cuda")
        chunk[:, :S] = Gs[r0:r0 + r]
        assert L().b200gnn_gsp_pair_fixed_chunk_f32(p(chunk), ld, r, S, r0, p(ns) if raw else None, p(sim), ld_t, n_t, p(inds),
                                                    kernel, p(rc) if raw else None, p(part), st()) == 0
        out[r0:r0 + r] = chunk
    assert torch.equal(out[:, S:], torch.zeros_like(out[:, S:]))
    assert torch.isnan(part[S:]).all() and torch.isnan(rc[S:]).all()
    return out[:, :S], rc[:S], part[:S]


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("S", [1, 7, 257, 600])
def test_fixed_pass_equals_the_two_sided_pass_every_row(kernel, S):
    xs, ns = operands(S, 24, kernel, 1)
    xt, nt = operands(S, 40, kernel, 2)
    Gs, Gt = gram(xs), gram(xt)
    ref_g, ref_rc, ref_part = both_pass(Gs, Gt, ns, nt, S, kernel)
    for R_sim in sorted({S, 128, 5}):
        sim = build_sim(Gt, nt, kernel, R_sim, ld_sim=S + 3)
        for R in sorted({S, 256, 64, 3}):
            g, rc, part = fixed_pass(Gs, ns, sim, S, kernel, R)
            assert torch.equal(g, ref_g), (R_sim, R)
            assert torch.equal(part, ref_part), (R_sim, R)
            if kernel >= 2:
                assert torch.equal(rc, ref_rc), (R_sim, R)
        assert torch.isnan(sim[:, S:]).all()                                # the builder writes only n columns


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("S", [1, 7, 257, 600])
def test_fixed_pass_with_a_sample_reads_sim_t_at_the_sampled_nodes(kernel, S):
    n = 700
    xs, ns = operands(S, 24, kernel, 3)                      # the student operands of the S sampled positions
    xt, nt = operands(n, 40, kernel, 4)                      # the teacher over all n nodes
    inds = torch.from_numpy(np.random.RandomState(S).choice(n, S, replace=False)).cuda()
    Gt_full = gram(xt)
    sim = build_sim(Gt_full, nt, kernel, 128)
    il = inds.long()
    ref_g, ref_rc, ref_part = both_pass(gram(xs), Gt_full[il][:, il].contiguous(), ns, None if nt is None else nt[il], S, kernel)
    i32 = inds.to(torch.int32)
    for R in sorted({S, 256, 3}):
        g, rc, part = fixed_pass(gram(xs), ns, sim, S, kernel, R, inds=i32)
        assert torch.equal(g, ref_g) and torch.equal(part, ref_part), R
        if kernel >= 2:
            assert torch.equal(rc, ref_rc), R


@pytest.mark.parametrize("kernel", KERNELS)
def test_builder_within_its_fp64_bound(kernel):
    n = 333
    x, sq = operands(n, 40, kernel, 5)
    G = gram(x)
    sim = build_sim(G, sq, kernel, 100).double()
    u = 2.0 ** -24
    G64 = G.double()
    if kernel == 0:
        assert torch.equal(sim, G64)
        return
    if kernel == 1:
        ref = G64 * G64
        assert ((sim - ref).abs() <= u * ref.abs()).all()
        return
    s64 = sq.double()
    mag = s64.view(-1, 1) + s64.view(1, -1) + 2 * G64.abs()
    d2 = (s64.view(-1, 1) + s64.view(1, -1) - 2 * G64).clamp_min(0)
    d2.fill_diagonal_(0)
    e = 4 * u * mag                                           # the fp32 rounding of n_i + n_j - 2 G
    if kernel == 2:
        ref = d2.sqrt()
        bound = e.sqrt() + 2 * u * ref
    else:
        ref = torch.exp(-0.5 * d2)
        bound = ref * (0.5 * e + 4 * u) + 1e-37
    bound.fill_diagonal_(0 if kernel == 2 else u)
    assert ((sim - ref).abs() <= bound).all()
    if kernel == 3:
        assert torch.equal(sim.diagonal(), torch.ones(n, dtype=torch.float64, device="cuda"))


def rows_problem(n=300, F=136, seed=6):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(n, F, generator=g).cuda()
    feat[3] = 0.0                                            # a zero row
    feat[5] = 1e-15                                          # a row under F.normalize's eps clamp
    return feat


def eager_operands(rows, kernel):
    if kernel <= 1:
        return criterion._normalize(rows)
    sq = torch.empty(rows.shape[0], device="cuda")
    assert L().b200gnn_row_sqnorm_f32(p(rows), rows.shape[0], rows.shape[1], p(sq), st()) == 0
    return rows, sq


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("sampled", [False, True])
def test_rows_operands_and_backward_equal_the_eager_row_kernels(kernel, sampled):
    n, F, beta = 300, 136, 100.0
    feat = rows_problem(n, F)
    ldf = F + 8
    fpad = torch.full((n, ldf), NAN, device="cuda")
    fpad[:, :F] = feat
    if sampled:
        rest = np.random.RandomState(0).permutation([i for i in range(n) if i not in (3, 5)])[:95]
        inds = torch.tensor([3, 5] + rest.tolist(), device="cuda")              # the zero and the clamped row sampled
        rows = feat[inds.long()]
        i32 = inds.to(torch.int32)
    else:
        rows, i32 = feat, None
    S = rows.shape[0]
    Sp = (S + 3) // 4 * 4
    x = torch.full((Sp, F), NAN, device="cuda")
    norm = torch.full((Sp,), NAN, device="cuda")
    assert L().b200gnn_gsp_rows_operands_f32(p(fpad), ldf, p(i32), S, F, kernel, EPS, p(x), F, p(norm), st()) == 0
    ref_x, ref_norm = eager_operands(rows.contiguous(), kernel)
    assert torch.equal(x[:S], ref_x) and torch.equal(norm[:S], ref_norm)
    assert torch.isnan(x[S:]).all() and torch.isnan(norm[S:]).all()
    zero, clamped = (0, 1) if sampled else (3, 5)                          # the sample positions of rows 3 and 5
    if kernel <= 1:
        assert torch.equal(x[zero], torch.zeros(F, device="cuda")) and float(norm[clamped]) < EPS

    # the way back: g = dG . x, the eager d = 2 g -> normalise backward / row_axpy, then * beta (autograd's multiply)
    gen = torch.Generator().manual_seed(9)
    gx = torch.randn(Sp, F, generator=gen).cuda()
    rc = torch.randn(Sp, generator=gen).cuda()
    d = (gx[:S] * 2.0).contiguous()
    if kernel >= 2:
        assert L().b200gnn_row_axpy_f32(p(ref_x), p(rc), S, F, 4.0, p(d), st()) == 0
    else:
        d = criterion._normalize_bwd(ref_x, ref_norm, d)
    d = d * torch.tensor(beta, device="cuda")
    ldd = F + 4
    d_feat = torch.full((n, ldd), NAN, device="cuda")
    loss_aux = torch.tensor([0.37], device="cuda")
    loss_total = torch.tensor([1.25], device="cuda")
    expect_total = loss_total + loss_aux * beta
    assert L().b200gnn_gsp_rows_backward_f32(p(i32), S, F, kernel, p(gx), p(x), F, p(norm), p(rc), EPS, beta, p(d_feat), ldd,
                                             p(loss_aux), p(loss_total), st()) == 0
    rows_idx = inds.long() if sampled else torch.arange(n, device="cuda")
    assert torch.equal(d_feat[rows_idx, :F], d)
    assert torch.isnan(d_feat[:, F:]).all()
    others = torch.ones(n, dtype=torch.bool, device="cuda")
    others[rows_idx] = False
    assert torch.isnan(d_feat[others]).all()                 # rows outside the sample are left alone
    assert torch.equal(loss_total, expect_total)


def test_refusals_launch_nothing():
    x = torch.zeros(64, 16, device="cuda")
    v = torch.zeros(64, device="cuda")
    i = torch.zeros(16, dtype=torch.int32, device="cuda")
    odd = x.data_ptr() + 2                                   # not 4-byte aligned
    lib_ = L()
    calls = [
        # builder: null G, null sim, n out of range, rows past n, unknown kernel, l2 without norms, misaligned
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(None, 16, 4, 16, 0, None, 0, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 16, 4, 16, 0, None, 0, None, 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 16, 4, 0, 0, None, 0, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 16, 4, 16, 14, None, 0, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 16, 4, 16, 0, None, 4, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 16, 4, 16, 0, None, 2, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(odd, 16, 4, 16, 0, None, 0, p(x), 16, st()),
        lambda: lib_.b200gnn_gsp_sim_chunk_f32(p(x), 8, 4, 16, 0, None, 0, p(x), 16, st()),
        # fixed pass: null partial, S past n_t, ld < S, unknown kernel, rbf without rc, misaligned sim_t
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 16, 4, 16, 0, None, p(x), 16, 16, None, 0, None, None, st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 32, 4, 32, 0, None, p(x), 16, 16, None, 0, None, p(v), st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 8, 4, 16, 0, None, p(x), 16, 16, None, 0, None, p(v), st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 16, 4, 16, 0, None, p(x), 16, 16, None, -1, None, p(v), st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 16, 4, 16, 0, p(v), p(x), 16, 16, None, 3, None, p(v), st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 16, 4, 16, 0, None, odd, 16, 16, None, 0, None, p(v), st()),
        lambda: lib_.b200gnn_gsp_pair_fixed_chunk_f32(p(x), 16, 4, 16, 13, None, p(x), 16, 16, p(i), 0, None, p(v), st()),
        # operands: null feat, F above the maximum, ldx < F, unknown kernel, eps 0, misaligned x
        lambda: lib_.b200gnn_gsp_rows_operands_f32(None, 16, None, 16, 16, 0, EPS, p(x), 16, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 4096, None, 1, lib.GSP_ROWS_MAX_F + 4, 0, EPS, p(x), 4096, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 16, None, 16, 16, 0, EPS, p(x), 8, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 16, None, 16, 16, 5, EPS, p(x), 16, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 16, None, 16, 16, 0, 0.0, p(x), 16, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 16, None, 16, 16, 0, EPS, odd, 16, p(v), st()),
        lambda: lib_.b200gnn_gsp_rows_operands_f32(p(x), 16, None, 0, 16, 0, EPS, p(x), 16, p(v), st()),
        # backward: null g, cosine without norm, rbf without rc, loss_total without loss_aux, ldd < F, misaligned d_feat
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 0, None, p(x), 16, p(v), None, EPS, 1.0, p(x), 16, None, None,
                                                   st()),
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 0, p(x), p(x), 16, None, None, EPS, 1.0, p(x), 16, None, None,
                                                   st()),
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 3, p(x), p(x), 16, p(v), None, EPS, 1.0, p(x), 16, None, None,
                                                   st()),
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 0, p(x), p(x), 16, p(v), None, EPS, 1.0, p(x), 16, None, p(v),
                                                   st()),
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 0, p(x), p(x), 16, p(v), None, EPS, 1.0, p(x), 8, None, None,
                                                   st()),
        lambda: lib_.b200gnn_gsp_rows_backward_f32(None, 16, 16, 0, p(x), p(x), 16, p(v), None, EPS, 1.0, odd, 16, None, None,
                                                   st()),
    ]
    torch.cuda.synchronize()
    before = lib.launch_count()
    for k, call in enumerate(calls):
        assert call() == BAD, k
    torch.cuda.synchronize()
    assert lib.launch_count() == before
    assert torch.equal(x, torch.zeros_like(x)) and torch.equal(v, torch.zeros_like(v))
