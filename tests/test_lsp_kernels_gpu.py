"""The captured LSP step's kernels through the C ABI: b200gnn_lsp_student_f32 equals the three-call sequence edge_sim ->
lsp_segment -> lsp_bwd_values bit for bit, and b200gnn_scatter_rows_scaled_f32 writes exactly src[i] * scale at idx[i]
and nothing else.  Every output sits among NaN canaries; every bad argument is refused before any launch."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion as C, lib, ops

pytestmark = pytest.mark.gpu

PAD = 64                 # NaN canary floats on each side of an output
HS = [4, 36, 64, 256, lib.LSP_MAX_F]


def canary(n):
    """(whole buffer, the n-float view an output is written to) with PAD NaNs on each side."""
    buf = torch.full((n + 2 * PAD,), float("nan"), device="cuda")
    return buf, buf[PAD:PAD + n]


def pads_intact(buf):
    return bool(torch.isnan(buf[:PAD]).all() and torch.isnan(buf[-PAD:]).all())


def designed_edges(n=3000, hub=2100, seed=0):
    """A dst-sorted-to-be edge list with empty segments (every node >= n - 300 and every 7th node receives nothing), one-edge
    segments, a hub segment of more than 2048 edges, duplicate edges and self loops."""
    rs = np.random.RandomState(seed)
    dst = [np.zeros(hub, dtype=np.int64)]                                  # node 0: the hub
    src = [rs.randint(0, n, hub)]
    receivers = np.array([i for i in range(1, n - 300) if i % 7])
    deg = rs.randint(1, 12, receivers.size)
    deg[::5] = 1                                                           # one-edge segments
    dst.append(np.repeat(receivers, deg))
    src.append(rs.randint(0, n, deg.sum()))
    src, dst = np.concatenate(src), np.concatenate(dst)
    dup = rs.choice(src.size, 200, replace=False)
    src, dst = np.concatenate([src, src[dup], [5, 6]]), np.concatenate([dst, dst[dup], [5, 6]])   # duplicates, self loops
    return torch.from_numpy(np.stack([src, dst])).cuda()


def designed_feat(n, H, seed=0):
    """Rows of every kind the cosine clamp sees: a zero row, norms in (0, 1e-8), a norm of exactly 1e-8 (sqrtf(x * x) == x),
    and ordinary rows."""
    g = torch.Generator().manual_seed(seed)
    f = torch.randn(n, H, generator=g)
    f[1] = 0.0                                                 # zero row
    f[2] = 0.0
    f[2, 0] = 3e-9                                             # norm in (0, 1e-8): the clamped branch
    f[3] = 0.0
    f[3, -1] = 1e-8                                            # norm exactly COS_EPS: the clamp's boundary
    f[4] *= 1e-3
    return f.cuda()


def hub_sources_hit_special_rows(ei):
    """Make the hub and a few other segments read the designed rows, as sources and as destinations."""
    ei = ei.clone()
    ei[0, :8] = torch.tensor([1, 2, 3, 4, 1, 2, 3, 4])
    return ei


def plan_of(ei, n):
    plan = C.LspPlan(ei)
    Cm, pos_dst, pos_src, diag_pos, _ = plan.backward_matrix(n)
    return plan, Cm, pos_dst, pos_src, diag_pos


def three_calls(feat, plan, Cm, pos_dst, pos_src, diag_pos, sim_t, kernel):
    """The existing sequence: sim_s, val (diagonal included), loss."""
    L, st = lib.load(), lib.stream_ptr()
    E, n = plan.E, Cm.n_rows
    sim_s, g = torch.empty(E, device="cuda"), torch.empty(E, device="cuda")
    loss, part = torch.empty(1, device="cuda"), torch.empty(int(L.b200gnn_lsp_partials(plan.n_seg)), device="cuda")
    val, selfc = torch.full_like(Cm.val, float("nan")), torch.empty_like(Cm.val)
    lib.check(L.b200gnn_edge_sim_f32(feat.data_ptr(), feat.shape[1], plan.src.data_ptr(), plan.dst.data_ptr(), E, kernel,
                                     sim_s.data_ptr(), st), "edge_sim_f32")
    lib.check(L.b200gnn_lsp_segment_f32(sim_s.data_ptr(), sim_t.data_ptr(), plan.rowptr.data_ptr(), plan.n_seg, E, 0,
                                        g.data_ptr(), loss.data_ptr(), part.data_ptr(), st), "lsp_segment_f32")
    lib.check(L.b200gnn_lsp_bwd_values_f32(feat.data_ptr(), feat.shape[1], plan.src.data_ptr(), plan.dst.data_ptr(), E, kernel,
                                           sim_s.data_ptr(), g.data_ptr(), pos_dst.data_ptr(), pos_src.data_ptr(),
                                           Cm.rowptr.data_ptr(), diag_pos.data_ptr(), n, val.data_ptr(), selfc.data_ptr(), st),
              "lsp_bwd_values_f32")
    return sim_s, val, loss


def fused(feat, plan, Cm, pos_dst, pos_src, diag_pos, sim_t, kernel):
    """b200gnn_lsp_student_f32 into canary buffers: (sim_s, val, loss, the three whole buffers)."""
    L = lib.load()
    E, n = plan.E, Cm.n_rows
    bs, sim_s = canary(E)
    bv, val = canary(Cm.val.numel())
    bl, loss = canary(1)
    scratch, selfc = torch.empty(2 * E, device="cuda"), torch.empty_like(Cm.val)
    part = torch.empty(int(L.b200gnn_lsp_partials(plan.n_seg)), device="cuda")
    ops.lsp_student(feat, plan.src, plan.dst, plan.rowptr, sim_t, kernel, pos_dst, pos_src, Cm.rowptr, diag_pos, sim_s,
                    scratch, val, selfc, loss, part)
    assert n == diag_pos.numel()
    return sim_s, val, loss, (bs, bv, bl)


def teacher_sims(ei_plan, n, F_t=37, kernel=0, seed=1):
    t = torch.randn(n, F_t, generator=torch.Generator().manual_seed(seed)).cuda()
    sim_t = torch.empty(ei_plan.E, device="cuda")
    lib.check(lib.load().b200gnn_edge_sim_f32(t.data_ptr(), F_t, ei_plan.src.data_ptr(), ei_plan.dst.data_ptr(), ei_plan.E,
                                              kernel, sim_t.data_ptr(), lib.stream_ptr()), "edge_sim_f32")
    return sim_t


def check_equal(feat, ei, kernel):
    n = feat.shape[0]
    plan, Cm, pos_dst, pos_src, diag_pos = plan_of(ei, n)
    sim_t = teacher_sims(plan, n, kernel=kernel)
    ref = three_calls(feat, plan, Cm, pos_dst, pos_src, diag_pos, sim_t, kernel)
    got = fused(feat, plan, Cm, pos_dst, pos_src, diag_pos, sim_t, kernel)
    for name, a, b in zip(("sim_s", "val", "loss"), got[:3], ref):
        assert torch.equal(a, b), (name, kernel, feat.shape[1])
    assert all(pads_intact(b) for b in got[3])
    assert torch.isfinite(got[1]).all() and torch.isfinite(got[2]).all()
    again = fused(feat, plan, Cm, pos_dst, pos_src, diag_pos, sim_t, kernel)
    for a, b in zip(got[:3], again[:3]):
        assert torch.equal(a, b)                                              # repeatable
    return plan, got


@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
@pytest.mark.parametrize("H", HS)
def test_student_equals_three_calls_on_designed_edges(kernel, H):
    n = 3000
    ei = hub_sources_hit_special_rows(designed_edges(n))
    plan, got = check_equal(designed_feat(n, H), ei, kernel)
    counts = torch.diff(plan.rowptr.long())
    assert int(counts.max()) > 2048 and int((counts == 0).sum()) > 0 and int((counts == 1).sum()) > 0
    assert plan.E > 2 * 2048


@pytest.mark.parametrize("kernel", [0, 1, 2, 3])
def test_clamped_rows_take_the_unclamped_gradient_branch_only_above_eps(kernel):
    """Rows 1 (zero), 2 (norm 3e-9) and 3 (norm exactly 1e-8) are clamped: the cosine kernels give them no self term, so the
    diagonal of such a row gathers only what its neighbours' sb / sa put there."""
    n, H = 64, 36
    src = torch.tensor([2, 3, 1, 5, 2, 3, 6, 7], device="cuda")
    dst = torch.tensor([5, 5, 5, 2, 3, 2, 3, 3], device="cuda")
    check_equal(designed_feat(n, H), torch.stack([src, dst]), kernel)


def test_more_segments_than_warps():
    """n_seg above the grid's 2112 x 8 warps: each warp walks several segments, and must load each one's row afresh."""
    n, H = 40_000, 64
    rs = np.random.RandomState(4)
    dst = rs.randint(0, n, 160_000)
    src = rs.randint(0, n, 160_000)
    ei = torch.from_numpy(np.stack([src, dst])).cuda()
    for kernel in range(4):
        plan, _ = check_equal(designed_feat(n, H, seed=2), ei, kernel)
        assert plan.n_seg > 2112 * 8


def test_bad_arguments_are_refused_without_a_launch():
    L = lib.load()
    n, H = 200, 64
    ei = torch.stack([torch.arange(n, device="cuda"), torch.arange(n, device="cuda").flip(0)])
    feat = designed_feat(n, H)
    plan, Cm, pos_dst, pos_src, diag_pos = plan_of(ei, n)
    sim_t = teacher_sims(plan, n)
    E = plan.E
    b = lambda k: torch.empty(k, device="cuda")
    sim_s, scratch, val, selfc, loss = b(E), b(2 * E), b(Cm.val.numel()), b(Cm.val.numel()), b(1)
    part = b(int(L.b200gnn_lsp_partials(plan.n_seg)))
    args = [feat.data_ptr(), H, plan.src.data_ptr(), plan.dst.data_ptr(), plan.rowptr.data_ptr(), plan.n_seg, E,
            sim_t.data_ptr(), 0, pos_dst.data_ptr(), pos_src.data_ptr(), Cm.rowptr.data_ptr(), diag_pos.data_ptr(), n,
            sim_s.data_ptr(), scratch.data_ptr(), val.data_ptr(), selfc.data_ptr(), loss.data_ptr(), part.data_ptr(),
            lib.stream_ptr()]
    assert L.b200gnn_lsp_student_f32(*args) == 0
    torch.cuda.synchronize()
    pointers = [0, 2, 3, 4, 7, 9, 10, 11, 12, 14, 15, 16, 17, 18, 19]
    bad = [(i, None) for i in pointers] + [(6, 0), (6, -1), (5, 0), (13, 0), (8, -1), (8, 4), (1, 0),
                                           (1, lib.LSP_MAX_F + 1)]
    for i, v in bad:
        a = list(args)
        a[i] = v
        before = lib.launch_count()
        assert L.b200gnn_lsp_student_f32(*a) == -1, (i, v)
        assert lib.launch_count() == before, (i, v)
    src, idx, dst = b(4 * 8), torch.arange(4, device="cuda"), b(4 * 8)
    sargs = [src.data_ptr(), idx.data_ptr(), 4, 8, 2.0, dst.data_ptr(), 8, None, None, lib.stream_ptr()]
    assert L.b200gnn_scatter_rows_scaled_f32(*sargs) == 0
    for i, v in [(0, None), (1, None), (5, None), (2, -1), (3, 0), (6, 7), (8, dst.data_ptr())]:
        a = list(sargs)
        a[i] = v
        before = lib.launch_count()
        assert L.b200gnn_scatter_rows_scaled_f32(*a) == -1, (i, v)
        assert lib.launch_count() == before, (i, v)


@pytest.mark.parametrize("K,ldd", [(1, 1), (3, 5), (7, 7), (64, 64), (64, 68), (255, 256), (256, 256)])
def test_scatter_rows_scaled_writes_exactly_the_named_rows(K, ldd):
    N, n = 900, 500
    g = torch.Generator().manual_seed(K)
    src = torch.randn(n, K, generator=g).cuda()
    idx = torch.randperm(N, generator=g)[:n].cuda()
    scale = 0.3                                                             # not a power of two: the product rounds
    buf = torch.full((N * ldd + 2 * PAD,), float("nan"), device="cuda")
    out = buf[PAD:PAD + N * ldd].view(N, ldd)[:, :K]
    loss_aux = torch.tensor([0.7123], device="cuda")
    loss_total = torch.tensor([1.2345, 5.0, 6.0], device="cuda")
    want_total = loss_total.clone()
    want_total[0] = want_total[0] + loss_aux[0] * scale                     # fp32 product, then fp32 add
    ops.scatter_rows_scaled(src, idx, scale, out, loss_aux=loss_aux, loss_total=loss_total)
    assert torch.equal(out[idx], src * scale)
    rows = torch.ones(N, dtype=torch.bool, device="cuda")
    rows[idx] = False
    assert torch.isnan(out[rows]).all()
    assert torch.isnan(buf[PAD:PAD + N * ldd].view(N, ldd)[:, K:]).all() and pads_intact(buf)
    assert torch.equal(loss_total, want_total)
    ops.scatter_rows_scaled(src, idx, scale, out)
    assert torch.equal(out[idx], src * scale) and torch.equal(loss_total, want_total)
