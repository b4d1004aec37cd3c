"""G-CRD in the captured SIGN student step (gcrd.SIGNGCRD, SIGNStudentTrainer(..., gcrd=)): the PReLU-prologue statistics
GEMM bit for bit against the statistics GEMM of the materialised activation, the step against the reference's own
train_kd_and_aux (tests/golden/sign_gcrd.pt), against the fp64 oracle/sign_gcrd.py over three steps, against the eager
aux= step with torch heads at the ARXIV shape, graph replay against eager steps, the sampler, the refusals and the heads'
state."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion
from oracle import dropout as odrop, gcrd as og, ppi_gcrd as opg, sign_gcrd as osg
from test_oracle_sign_gcrd import GOLD, H as GOLD_H

pytestmark = pytest.mark.gpu

SAMPLE_STREAM = 1 << 62
HEAD_KEYS = osg.HEAD_KEYS


def _ops():
    from efficient_gnns_b200 import ops
    return ops


def rand_bits(n, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-2**31, 2**31 - 1, (n, (K + 31) // 32), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)


# ------------------------------------------------------------------------------------------------ 1. the kernel
@pytest.mark.parametrize("N", [64, 128, 256])
@pytest.mark.parametrize("K", [128, 512, 750, 3072])
def test_prelu_stats_gemm_equals_stats_gemm_of_the_materialised_activation(K, N):
    """Output and statistics partials bit for bit those of the statistics GEMM on prelu_bits(Z): the A fragments are the
    same bits and the epilogue the same code.  Both run through the C ABI with Z, the activation and the weight at a row
    pitch of ceil4(K), so K = 750 (the GAT teacher's width) runs with a ragged last K block and keep word (its
    materialised twin is formed over all 752 columns; the weight's two padding columns are zero)."""
    from efficient_gnns_b200 import lib
    ops, L = _ops(), lib.load()
    Kp = (K + 3) // 4 * 4
    g = torch.Generator(device="cuda").manual_seed(K * 7 + N)
    w = torch.zeros(N, Kp, device="cuda")
    w[:, :K] = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    bias = torch.randn(N, device="cuda", generator=g)
    hi, lo = ops.split_tf32(w)
    for M in (2, 127, 50000):
        z = torch.randn(M, Kp, device="cuda", generator=g)
        bits = rand_bits(M, K, M + K)
        slots = ops.gemm_stat_slots(M, N)
        x = torch.empty(M, Kp, device="cuda")
        for slope, p in ((0.25, 0.0), (-0.5, 0.5), (0.0, 0.5), (0.25, 0.5), (-0.5, 0.0), (0.0, 0.0)):
            a = torch.tensor([slope], device="cuda")
            ops.prelu_bits(z, bits, a, p, out=x)          # all Kp columns (a multiple of 4); the GEMMs read K of them
            ref, ref_part = torch.full((M, N), float("nan"), device="cuda"), torch.full((slots, 2, N), float("nan"), device="cuda")
            lib.check(L.b200gnn_gemm_tf32x3_stats_f32(x.data_ptr(), Kp, hi.data_ptr(), lo.data_ptr(), Kp, ref.data_ptr(), N, M, N,
                                                      K, bias.data_ptr(), 0, ref_part.data_ptr(), slots, lib.stream_ptr()),
                      "stats")
            out, part = torch.full((M, N), float("nan"), device="cuda"), torch.full((slots, 2, N), float("nan"), device="cuda")
            lib.check(L.b200gnn_gemm_tf32x3_prelu_stats_f32(z.data_ptr(), Kp, hi.data_ptr(), lo.data_ptr(), Kp, out.data_ptr(),
                                                            N, M, N, K, bias.data_ptr(), a.data_ptr(), bits.data_ptr(), p,
                                                            part.data_ptr(), slots, lib.stream_ptr()), "prelu_stats")
            assert torch.equal(out, ref), (M, slope, p)
            assert torch.equal(part, ref_part), (M, slope, p)
            if K % 4 == 0 and M == 127:                   # the ops wrapper: the same launch on contiguous operands
                hk, lk = ops.split_tf32(w[:, :K].contiguous())
                out2 = torch.empty(M, N, device="cuda")
                ops.gemm_tf32x3_prelu_stats(z[:, :K], a, bits, p, hk, lk, bias, out2, part)
                assert torch.equal(out2, ref) and torch.equal(part, ref_part)


def test_prelu_stats_gemm_refuses_what_the_stats_gemm_refuses():
    from efficient_gnns_b200 import lib
    ops = _ops()
    M, K = 300, 256
    z = torch.randn(M, K, device="cuda")
    bits, a = rand_bits(M, K, 1), torch.tensor([0.25], device="cuda")
    x = ops.prelu_bits(z, bits, a, 0.5)
    for N, ldc in ((48, 48), (40, 40), (100, 100), (288, 288), (128, 130)):
        hi, lo = ops.split_tf32(torch.randn(N, K, device="cuda"))
        out = torch.empty(M, ldc, device="cuda")[:, :N]
        part = torch.empty(ops.gemm_stat_slots(M, max(N, 64)) + 8, 2, max(N, 64), device="cuda")
        with pytest.raises(lib.B200GnnError):
            ops.gemm_tf32x3_stats(x, hi, lo, None, out, part)
        with pytest.raises(lib.B200GnnError):
            ops.gemm_tf32x3_prelu_stats(z, a, bits, 0.5, hi, lo, None, out, part)
    hi, lo = ops.split_tf32(torch.randn(128, K, device="cuda"))
    out = torch.empty(M, 128, device="cuda")
    small = torch.empty(ops.gemm_stat_slots(M, 128) - 1, 2, 128, device="cuda")       # too few slots
    with pytest.raises(lib.B200GnnError):
        ops.gemm_tf32x3_prelu_stats(z, a, bits, 0.5, hi, lo, None, out, small)
    with pytest.raises(lib.B200GnnError):
        ops.gemm_tf32x3_stats(x, hi, lo, None, out, small)
    with pytest.raises(lib.B200GnnError):                                                # p outside [0, 1)
        ops.gemm_tf32x3_prelu_stats(z, a, bits, 1.0, hi, lo, None, out,
                                    torch.empty(ops.gemm_stat_slots(M, 128), 2, 128, device="cuda"))


# ------------------------------------------------------------------------------------------------ helpers
def trainer(feats, n_classes, hidden, ff, gcrd=None, batch_size=64, seed=0, **kw):
    from efficient_gnns_b200.engine_sign import SIGNStudentTrainer
    return SIGNStudentTrainer(feats=feats, n_classes=n_classes, hidden=hidden, ff_layer=ff, batch_size=batch_size, seed=seed,
                              gcrd=gcrd, **kw)


def sign_gcrd(t_feat, width, **kw):
    from efficient_gnns_b200.gcrd import SIGNGCRD
    return SIGNGCRD(t_feat, width, **kw)


def head_grads(obj):
    """The heads' gradients under the reference's keys (the teacher's Linear at its own width)."""
    F_t = obj.F_t
    return {"sproj": {"0.weight": obj.gW_s, "0.bias": obj.gb_s, "1.weight": obj.ggamma_s, "1.bias": obj.gbeta_s},
            "tproj": {"0.weight": obj.gW_t[:, :F_t], "0.bias": obj.gb_t, "1.weight": obj.ggamma_t, "1.bias": obj.gbeta_t}}


def problem(seed=0, n=600, F=16, H=3, C=8, n_train=300, F_t=22):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(n, F, generator=g).cuda() for _ in range(H)]
    y = torch.randint(0, C, (n,), generator=g).cuda()
    t = (torch.randn(n, C, generator=g) * 2).cuda()
    t_feat = torch.randn(n, F_t, generator=g).cuda()
    train_idx = torch.randperm(n, generator=g)[:n_train].cuda()
    return feats, y, t, t_feat, train_idx


# ------------------------------------------------------------------------------------------------ 3. the fixture
@pytest.mark.parametrize("name", sorted(GOLD["cases"]))
def test_engine_reproduces_reference_fixture(name):
    c = GOLD["cases"][name]
    ff = c["ff"]
    hid = GOLD["hidden"]
    obj = sign_gcrd(GOLD["teacher_feat"].cuda(), GOLD_H * hid, proj_dim=GOLD["proj_dim"], max_samples=c["max_samples"],
                    nce_T=GOLD["nce_T"], beta=GOLD["beta"])
    s_sd, t_sd = opg.seeded_heads(GOLD_H * hid, GOLD["teacher_feat"].shape[1], GOLD["proj_dim"], GOLD["seeds"]["heads"])
    obj.load_student_proj_state_dict({k: v.cuda() for k, v in s_sd.items()})
    obj.load_teacher_proj_state_dict({k: v.cuda() for k, v in t_sd.items()})
    tr = trainer([f.cuda() for f in GOLD["feats"]], GOLD["n_classes"], hid, ff, gcrd=obj, dropout=GOLD["dropout"],
                 input_drop=GOLD["input_drop"], lr=GOLD["lr"], alpha=GOLD["alpha"], kd_T=GOLD["kd_T"],
                 seed=GOLD["seeds"]["dropout"])
    tr.load_state_dict({k: v.cuda() for k, v in GOLD["states"][ff].items()})
    loss = tr.train_step(GOLD["batch"].cuda(), GOLD["labels"].cuda(), GOLD["teacher_logits"].cuda(), sample=c["sample"]).cpu()
    if c["sample"] is None:
        assert torch.equal(obj.sample().cpu(), torch.arange(GOLD["batch"].numel()))
    else:
        assert torch.equal(obj.sample().cpu(), c["sample"])
    for got, ref in zip(loss, c["loss"]):
        assert abs(got.item() - ref.item()) < 1e-5 * abs(ref.item()), (loss, c["loss"])
    grads = {"model": tr.grad_dict(), **head_grads(obj)}
    for group, ref_g in c["grads"].items():
        scale = max(v.abs().max().item() for v in ref_g.values())
        for k, g in ref_g.items():
            if group != "model" and k == "0.bias":
                # a bias in front of BatchNorm: its exact gradient is 0, both sides carry rounding only
                assert grads[group][k].abs().max().item() < 1e-5 * scale, (group, k)
                continue
            assert rel_err(grads[group][k], g) < 1e-5, (group, k, rel_err(grads[group][k], g))
    after = {"model": tr.state_dict(), "sproj": obj.student_proj_state_dict(), "tproj": obj.teacher_proj_state_dict()}
    for group, ref_g in c["after"].items():
        for k, v in ref_g.items():
            if group != "model" and k == "0.bias":    # moved by lr in the direction of its rounding noise (see above)
                continue
            g = c["grads"][group][k].double()
            keep = g.abs() > 1e-2 * g.abs().max()        # Adam's first step is lr * g / (|g| + eps): compared where g is clear
            if bool(keep.any()):
                assert (after[group][k].cpu().double()[keep] - v.double()[keep]).abs().max() <= 1e-6, (group, k)
    for group, sd in c["running"].items():
        for k, v in sd.items():
            if "num_batches" in k:
                assert int(after[group][k]) == int(v) == 1
            else:
                assert rel_err(after[group][k], v) < 1e-5, (group, k)


# ------------------------------------------------------------------------------------------------ 4. fp64 oracle
@pytest.mark.parametrize("ff", [1, 2])
def test_three_steps_match_the_fp64_oracle(ff):
    """The engine's own dropout masks and Philox draws (S < B on every step) fed to oracle/sign_gcrd.py."""
    feats, y, t, t_feat, train_idx = problem(ff)
    hid, H, B, S, LR = 64, 3, 200, 150, 0.01
    obj = sign_gcrd(t_feat, H * hid, proj_dim=64, max_samples=S, beta=0.1, seed=3)
    tr = trainer(feats, 8, hid, ff, gcrd=obj, batch_size=256, seed=5, lr=LR)
    with torch.no_grad():                                   # non-default slopes, of both signs
        for k, v in tr.P.items():
            if "slope" in k:
                v.copy_(torch.linspace(-0.4, 0.3, v.numel()))
    run = osg.Run({k: v.cpu() for k, v in tr.state_dict().items()},
                  {k: v.cpu() for k, v in obj.student_proj_state_dict().items()},
                  {k: v.cpu() for k, v in obj.teacher_proj_state_dict().items()}, LR)
    fc, yc, tc, tfc = [f.cpu() for f in feats], y.cpu(), t.cpu(), t_feat.cpu()
    for step in range(3):
        b = train_idx[step * 30:step * 30 + B]
        loss = tr.train_step(b, y, t).cpu()
        sample = obj.sample().cpu()
        assert np.array_equal(sample.numpy(), og.sample_perm(B, tr.seed, SAMPLE_STREAM + step)[:S]), step
        bc = b.cpu()
        masks = osg.engine_masks(H, 16, hid, ff, B, tr.p, tr.p_in, tr.seed, step)
        ref, grads = run.step([f[bc] for f in fc], yc[bc], tc[bc], tfc[bc], masks, sample, ff, 0.1, 0.075, p=tr.p,
                              p_in=tr.p_in, alpha=tr.alpha, kd_T=tr.kd_T)
        for got, want in zip(loss, ref):
            assert abs(got.item() - want.item()) <= 2e-5 * max(1.0, abs(want.item())), (step, loss, ref)
        if step == 0:                                       # from the same state: the gradients too
            gd = tr.grad_dict()
            for k, gr in grads["model"].items():
                assert rel_err(gd[k], gr) < 2e-5, (k, rel_err(gd[k], gr))
            hg = head_grads(obj)
            for group in ("sproj", "tproj"):
                for k in ("0.weight", "1.weight", "1.bias"):
                    assert rel_err(hg[group][k], grads[group][k]) < 2e-5, (group, k, rel_err(hg[group][k], grads[group][k]))
        # the biases in front of BatchNorm have a gradient of rounding noise on both sides, so Adam moves each by lr in a
        # direction of its own; the loss does not depend on them, the running mean does: the oracle takes the engine's
        with torch.no_grad():
            run.groups["sproj"]["0.bias"].copy_(obj.b_s.double().cpu())
            run.groups["tproj"]["0.bias"].copy_(obj.b_t.double().cpu())
    # Adam divides by sqrt(v): an entry whose gradient is near Adam's eps moves by an amount that follows fp32 rounding in
    # that gradient, so the parameters after three steps are held to 5e-4 (the losses and gradients above to 2e-5)
    sd = tr.state_dict()
    for k, v in run.state("model").items():
        assert rel_err(sd[k], v) < 5e-4, k
    for mine, group in ((obj.student_proj_state_dict(), "sproj"), (obj.teacher_proj_state_dict(), "tproj")):
        for k in HEAD_KEYS:
            assert rel_err(mine[k], run.state(group)[k]) < 5e-4, (group, k)
        for k, v in run.running[group].items():
            assert rel_err(mine[k], v) < 1e-5, (group, k)
        assert int(mine["1.num_batches_tracked"]) == 3


# ------------------------------------------------------------------------------------------------ 5. ARXIV shape
def test_captured_step_at_the_arxiv_shape_equals_the_eager_aux_step():
    """6 hops of 128 features over 169,343 nodes, hidden 512 (head input 3072), 40 classes, batch 50,000, teacher features
    750 wide, at scripts/run_all_kd_and_aux.sh's settings (proj_dim 256, max_samples 16384, nce_T 0.075, beta 0.1):
    one captured G-CRD step against the eager aux= step with torch heads from the same head states and the same sample."""
    N, F, H, hid, C, B, F_t = 169_343, 128, 6, 512, 40, 50_000, 750
    g = torch.Generator(device="cuda").manual_seed(17)
    feats = [torch.randn(N, F, device="cuda", generator=g) for _ in range(H)]
    y = torch.randint(0, C, (N,), device="cuda", generator=g)
    t = torch.randn(N, C, device="cuda", generator=g) * 2
    t_feat = torch.randn(N, F_t, device="cuda", generator=g).relu()
    b = torch.randperm(N, device="cuda", generator=g)[:B]
    obj = sign_gcrd(t_feat, H * hid)
    assert (obj.P, obj.max_samples, obj.nce_T, obj.beta) == (256, 16384, 0.075, 0.1)
    s_sd, t_sd = obj.student_proj_state_dict(), obj.teacher_proj_state_dict()
    fused = trainer(feats, C, hid, 2, gcrd=obj, batch_size=B, seed=1)
    state0 = fused.state_dict()
    fused.capture([B], y, t)
    loss = fused.replay(b).clone()
    sample = obj.sample()
    assert sample.numel() == 16384 and sample.unique().numel() == 16384

    eager = trainer(feats, C, hid, 2, batch_size=B, seed=1)
    sp = torch.nn.Sequential(torch.nn.Linear(H * hid, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).cuda()
    tp = torch.nn.Sequential(torch.nn.Linear(F_t, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).cuda()
    sp.load_state_dict(s_sd)
    tp.load_state_dict(t_sd)
    yb, tfb = y[b], t_feat[b]
    aux = lambda f: criterion.nce_criterion(eager.logits().detach(), yb, sp(f), tp(tfb), 0.1, 0.075, 16384, sample)[2]  # noqa: E731
    ref = eager.train_step(b, y, t, aux=aux, beta=0.1).clone()
    assert abs(loss[0].item() - ref[0].item()) <= 2e-5 * abs(ref[0].item()), (loss, ref)
    assert loss[1].item() == ref[1].item()
    assert abs(loss[2].item() - eager.loss_aux.item()) <= 2e-5 * abs(eager.loss_aux.item()), (loss, eager.loss_aux)
    # Both routes are fp32 and reduce over 50,000 rows in different orders (BatchNorm statistics and backward, the heads'
    # input gradient, the weight gradients), and the hop FFNs' first-layer weight gradients are sums of largely cancelling
    # terms: the two differ by up to a few 1e-4 of their largest entry.  So both are held to an fp64 restatement of the
    # step (oracle/sign_gcrd.py on the GPU, the engine's own keep masks and the same sample), and the fused gradients may
    # be no further from it than twice the eager route's error, or 1e-4.
    from efficient_gnns_b200 import ops
    st = odrop.sign_streams(H, 2, 0)
    m = lambda rows, K, q, off: ops.dropout_mask(rows, K, q, fused.seed, off).bool()  # noqa: E731
    masks = dict(input=[m(B, F, fused.p_in, st[f"hop{h}"]) for h in range(H)],
                 hidden=[[m(B, hid, fused.p, st[f"hidden{h}"])] for h in range(H)], project=[m(B, hid, fused.p, st[f"hidden{H}"])],
                 cat=m(B * H, hid, fused.p, st["cat"]).view(B, H * hid))
    leaf = lambda sd: {k: v.detach().double().clone().requires_grad_(True) for k, v in sd.items()}  # noqa: E731
    m64 = leaf(state0)
    s64, t64 = (leaf({k: sd[k] for k in HEAD_KEYS}) for sd in (s_sd, t_sd))
    l64 = osg.nce_step_loss(m64, s64, t64, [f[b].double() for f in feats], yb, t[b].double(), tfb.double(), masks, sample, 2,
                            0.1, 0.075, p=fused.p, p_in=fused.p_in, alpha=fused.alpha, kd_T=fused.kd_T)[0]
    l64.backward()
    assert abs(loss[0].item() - l64.item()) <= 2e-5 * abs(l64.item())
    gf, ge = fused.grad_dict(), eager.grad_dict()
    hg = head_grads(obj)
    pairs = [(k, gf[k], ge[k], m64[k].grad) for k in ge]
    for group, mod, d64 in (("sproj", sp, s64), ("tproj", tp, t64)):
        ref_g = {k: p.grad for k, p in mod.named_parameters()}
        pairs += [(f"{group}/{k}", hg[group][k], ref_g[k], d64[k].grad) for k in ("0.weight", "1.weight", "1.bias")]
    errors = {name: (rel_err(f, g64), rel_err(e, g64)) for name, f, e, g64 in pairs}
    bad = {k: v for k, v in errors.items() if v[0] > max(2 * v[1], 1e-4)}
    assert not bad, bad
    for group, mod in (("sproj", sp), ("tproj", tp)):
        mine = obj.student_proj_state_dict() if group == "sproj" else obj.teacher_proj_state_dict()
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(mine[k], mod.state_dict()[k]) < 1e-5, (group, k)


# ------------------------------------------------------------------------------------------------ 6. graph replay
def test_replay_of_a_ragged_epoch_equals_eager_steps_bit_for_bit_and_capture_does_not_train():
    feats, y, t, t_feat, train_idx = problem(4)
    hid = 64

    def make():
        obj = sign_gcrd(t_feat, 3 * hid, proj_dim=64, max_samples=100, seed=6)
        return trainer(feats, 8, hid, 2, gcrd=obj, batch_size=128, seed=1), obj

    (eager, eo), (graphed, go) = make(), make()
    graphed.capture([128, 300 - 256], y, t)
    assert torch.equal(graphed.params, eager.params) and int(graphed.step_count) == 0
    assert torch.equal(go.params, eo.params) and torch.equal(go.exp_avg, eo.exp_avg) and int(go.step_count) == 0
    for a, b in ((go.rm_s, eo.rm_s), (go.rv_s, eo.rv_s), (go.rm_t, eo.rm_t), (go.rv_t, eo.rv_t)):
        assert torch.equal(a, b)
    le, lg, se, sg = [], [], [], []
    for epoch in range(2):
        order = eager.epoch_order(train_idx, epoch)
        for s in range(0, 300, 128):
            le.append(eager.train_step(order[s:s + 128], y, t).clone())
            se.append(eo.sample().cpu())
        lg.append(graphed.train_epoch(train_idx, y, t))
        sg.append(go.sample().cpu())
    le, lg = torch.stack(le), torch.cat(lg)
    assert lg.shape == (6, 3) and int(graphed.step_count) == 6 and int(go.step_count) == 6
    assert torch.equal(le, lg)
    assert torch.equal(eager.params, graphed.params) and torch.equal(eager.exp_avg_sq, graphed.exp_avg_sq)
    assert torch.equal(eo.params, go.params) and torch.equal(eo.exp_avg_sq, go.exp_avg_sq)
    for a, b in ((go.rm_s, eo.rm_s), (go.rv_s, eo.rv_s), (go.rm_t, eo.rm_t), (go.rv_t, eo.rv_t)):
        assert torch.equal(a, b)
    assert torch.equal(sg[-1], se[-1]) and torch.equal(se[-1], torch.arange(44))     # the last batch: S = B, no draw
    assert go.student_proj_state_dict()["1.num_batches_tracked"] == 6


# ------------------------------------------------------------------------------------------------ 7. the sampler
def test_each_step_draws_afresh_at_the_trainers_step_counter():
    feats, y, t, t_feat, train_idx = problem(5)
    obj = sign_gcrd(t_feat, 3 * 64, proj_dim=64, max_samples=50)
    tr = trainer(feats, 8, 64, 2, gcrd=obj, batch_size=128, seed=9)
    b = train_idx[:120]
    drawn = []
    for step in range(3):
        tr.train_step(b, y, t)
        want = og.sample_perm(120, tr.seed, SAMPLE_STREAM + step)[:50]
        assert np.array_equal(obj.sample().cpu().numpy(), want), step
        drawn.append(tuple(want))
    assert len(set(drawn)) == 3
    assert obj.row_sets[120].sample_ws is not None
    # S = B: no draw runs (no workspace), every row in order
    tr.train_step(train_idx[:40], y, t)
    assert obj.row_sets[40].sample_ws is None and torch.equal(obj.sample().cpu(), torch.arange(40))
    assert int(obj.step_count) == int(tr.step_count) == 4


# ------------------------------------------------------------------------------------------------ 8. refusals, state
def test_refusals_do_no_device_work_and_head_state_round_trips():
    from efficient_gnns_b200 import lib
    feats, y, t, t_feat, train_idx = problem(6)
    with pytest.raises(ValueError, match="wide"):
        trainer(feats, 8, 64, 2, gcrd=sign_gcrd(t_feat, 2 * 64))
    with pytest.raises(ValueError, match="rows"):
        trainer(feats, 8, 64, 2, gcrd=sign_gcrd(t_feat[:500], 3 * 64))
    obj = sign_gcrd(t_feat, 3 * 64, proj_dim=64, max_samples=50)
    tr = trainer(feats, 8, 64, 2, gcrd=obj, batch_size=128, seed=2)
    kd = trainer(feats, 8, 64, 2, batch_size=128, seed=2)
    tr.train_step(train_idx[:100], y, t)
    before = (lib.launch_count(), tr.params.clone(), obj.params.clone(), int(tr.step_count), int(obj.step_count), tr.epoch)
    aux = lambda f: f.sum()  # noqa: E731
    for call in (lambda: tr.train_step(train_idx[:100], y, t, aux=aux),                 # aux= with gcrd=
                 lambda: tr.train_epoch(train_idx, y, t, aux=aux),
                 lambda: kd.train_step(train_idx[:100], y, t, sample=torch.arange(50)),  # sample= without gcrd=
                 lambda: tr.train_step(train_idx[:1], y, t),                             # a batch of one row
                 lambda: tr.train_epoch(train_idx[:129], y, t),                          # ... as an epoch's ragged last batch
                 lambda: tr.capture([128, 1], y, t),
                 lambda: tr.train_step(train_idx[:100], y, t, sample=torch.arange(49))):  # not S distinct positions
        with pytest.raises(ValueError):
            call()
    assert lib.launch_count() == before[0]
    assert torch.equal(tr.params, before[1]) and torch.equal(obj.params, before[2])
    assert (int(tr.step_count), int(obj.step_count), tr.epoch) == before[3:]
    # the heads' state dicts round-trip, with num_batches_tracked = steps taken
    tr.train_step(train_idx[100:200], y, t)
    s_sd, t_sd = obj.student_proj_state_dict(), obj.teacher_proj_state_dict()
    assert int(s_sd["1.num_batches_tracked"]) == int(t_sd["1.num_batches_tracked"]) == 2
    other = sign_gcrd(t_feat, 3 * 64, proj_dim=64, max_samples=50, seed=11)
    other.load_student_proj_state_dict(s_sd)
    other.load_teacher_proj_state_dict(t_sd)
    for got, ref in ((other.student_proj_state_dict(), s_sd), (other.teacher_proj_state_dict(), t_sd)):
        for k, v in ref.items():
            assert torch.equal(got[k].cpu(), v.cpu()), k
