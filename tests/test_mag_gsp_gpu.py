"""GSP in the R-GCN student step on GraphSAINT batches (``RGCNTrainer(..., gsp=BatchGSP(...)).train_step(b, x,
teacher=t)``, the reference's MAG ``--training gpw``): the step against the eager ``teacher_logits=`` + ``aux=gpw_criterion``
route (the loss bit for bit, the gradients and parameters within the contraction's bound), the reference's own step
(tests/golden/mag_gsp.pt), the fp64 restatement oracle/mag_gsp.py over three steps, the on-device sample, one step at the
MAG scripts' size (S = 24576) against an fp64 gradient, and the refusals."""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion, lib, ops, sampling
from efficient_gnns_b200.gsp import BatchGSP
from efficient_gnns_b200.heads import SAMPLE_STREAM
from efficient_gnns_b200.lsp import BatchLSP
from efficient_gnns_b200.rgcn import RGCNTrainer
from oracle import gcrd as og, mag_gsp as omg
from test_mag_lsp_gpu import assert_same_state
from test_oracle_mag_gsp import GOLD
from test_rgcn_train_gpu import NODES, batches, small_mag

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

KERNELS = ["cosine", "poly", "l2", "rbf"]
H, H_T, C, LR, BETA = 24, 32, 7, 0.005, 10.0


def student(rel, gsp=None, seed=3, lsp=None):
    return RGCNTrainer(16, H, C, 2, 0.5, NODES, [0], len(rel), rel, lr=LR, seed=seed, gsp=gsp, lsp=lsp)


def teacher_of(rel, hidden=H_T, seed=11):
    return RGCNTrainer(16, hidden, C, 3, 0.5, NODES, [0], len(rel), rel, lr=LR, seed=seed)


def eager_aux(t_feat, tm, obj, sample):
    n = int(tm.sum())
    dummy = torch.zeros(n, 2, device="cuda"), torch.zeros(n, dtype=torch.long, device="cuda")
    return lambda f: criterion.gpw_criterion(*dummy, f[tm], t_feat[tm], obj.kernel, 1, obj.max_samples,  # noqa: E731
                                             sampled_inds=sample)[2]


def eager_step(tr, t, b, x, obj, sample):
    """The route that needs no gsp=: the teacher's own forward, gpw_criterion through ``aux=``."""
    tl = t.forward(b, x, training=False)[b.train_mask]
    return tr.train_step(b, x, teacher_logits=tl, beta=obj.beta, aux=eager_aux(t.out_feat(), b.train_mask, obj, sample)).clone()


def compare_with_eager(fused, eager, got, ref):
    """The loss vector bit for bit; the gradients within 1e-4 of their largest entry (the contraction sums dG . x in
    another order than the GEMM); Adam's first step lr * g / (|g| + eps) then moves a parameter by at most
    lr * min(2, |g_fused - g_eager| / eps) more on one side than on the other."""
    assert torch.equal(got[:2], ref[:2]) and torch.equal(got[2], eager.loss_aux), (got, ref, eager.loss_aux)
    ga, gb = fused._named(fused.grads, {}), eager._named(eager.grads, {})
    for k in gb:
        assert rel_err(ga[k], gb[k]) < 1e-4, (k, rel_err(ga[k], gb[k]))
    for t in fused.emb:
        a, e = fused.emb_m[t], eager.emb_m[t]
        assert float((a - e).abs().max()) <= 1e-4 * float(e.abs().max()), t
    bound = LR * torch.clamp((fused.grads - eager.grads).abs() / 1e-8, max=2.0) + 1e-6 * eager.params.abs()
    assert bool(((fused.params - eager.params).abs() <= bound).all())


# ------------------------------------------------------------------------------------------------ 1. the eager route
@pytest.mark.parametrize("rows", ["all", "sampled"])
@pytest.mark.parametrize("kernel", KERNELS)
def test_step_equals_the_eager_aux_step(kernel, rows):
    """Three batches with different train-row counts, each the first step of fresh trainers: every row (S >= n) or an
    injected sample of S < n rows, beta 10."""
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    sizes = set()
    for k, b in enumerate(batches(data, 3, seed=5)):
        n = int(b.train_mask.sum())
        sizes.add(n)
        S = 48 if rows == "sampled" else 24576
        assert (S < n) == (rows == "sampled")
        sample = np.random.RandomState(k).choice(n, S, replace=False) if S < n else None
        obj = BatchGSP(H, H_T, kernel, BETA, S)
        fused, eager = student(rel, gsp=obj), student(rel)
        got = fused.train_step(b, x, teacher=t, sample=None if sample is None else torch.as_tensor(sample)).clone()
        ref = eager_step(eager, t, b, x, obj, sample)
        want = torch.arange(n) if sample is None else torch.as_tensor(sample, dtype=torch.int64)
        assert torch.equal(obj.sample().cpu(), want)
        compare_with_eager(fused, eager, got, ref)
        assert int(fused.step_count) == 1
    assert len(sizes) == 3


# ------------------------------------------------------------------------------------------------ 2. the sampler
def test_each_step_draws_afresh_at_the_students_step_counter():
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    S = 40
    tr = student(rel, gsp=BatchGSP(H, H_T, "cosine", 1.0, S), seed=6)
    drawn = []
    for b in batches(data, 3, seed=7):
        step, n = int(tr.step_count), int(b.train_mask.sum())
        loss = tr.train_step(b, x, teacher=t)
        assert bool(torch.isfinite(loss).all())
        want = og.sample_perm(n, tr.seed, SAMPLE_STREAM + step)[:S]
        assert np.array_equal(tr.gsp.sample().cpu().numpy(), want), step
        drawn.append(tuple(want.tolist()))
    assert len(set(drawn)) == 3 and int(tr.step_count) == 3


# ------------------------------------------------------------------------------------------------ 3. the reference's step
def fixture_run(case):
    """One engine step on the fixture's designed batch: the student at the fixture's state (its dropout masks are this
    trainer's own, seed 0), the recorded draw injected; also a KD-only twin and the teacher."""
    c = GOLD["cases"][case]
    rel = {r: tuple(sd) for r, sd in enumerate(GOLD["relations"])}
    mk = lambda hidden, L, gsp=None: RGCNTrainer(  # noqa: E731
        GOLD["in_channels"], hidden, GOLD["out_channels"], L, 0.5, GOLD["num_nodes"], [0], len(rel), rel, lr=GOLD["lr"],
        seed=GOLD["seeds"]["dropout"], alpha=GOLD["alpha"], kd_T=GOLD["kd_T"], gsp=gsp)
    obj = BatchGSP(GOLD["hidden"], GOLD["teacher_hidden"], c["kernel"], GOLD["beta"], c["max_samples"])
    tr, kd, t = mk(GOLD["hidden"], 2, obj), mk(GOLD["hidden"], 2), mk(GOLD["teacher_hidden"], 3)
    for m, sd in ((tr, GOLD["student_state"]), (kd, GOLD["student_state"]), (t, GOLD["teacher_state"])):
        m.load_state_dict({k: v.cuda() for k, v in sd.items()})
    b = SimpleNamespace(edge_index=GOLD["edge_index"].cuda(), edge_attr=GOLD["edge_type"].cuda(),
                        node_type=GOLD["node_type"].cuda(), local_node_idx=GOLD["local_node_idx"].cuda(),
                        y=GOLD["y"].cuda(), train_mask=GOLD["train_mask"][c["mask"]].cuda())
    x = {0: GOLD["x"].cuda()}
    loss = tr.train_step(b, x, teacher=t, sample=c["sample"]).clone().double().cpu()
    return c, tr, kd, t, obj, b, x, loss


@pytest.mark.parametrize("case", [f"main/{k}" for k in KERNELS] + ["main/sampled", "one_train"])
def test_designed_batch_step_matches_the_reference(case):
    c, tr, kd, t, obj, b, x, loss = fixture_run(case)
    assert rel_err(loss, c["loss"]) <= 1e-4, (loss, c["loss"])
    got = tr._named(tr.grads, {})
    # the embedding tables' gradients: every row is in the batch, and Adam's first moment after one step is 0.1 * g
    got.update({f"emb_dict.{t}": tr.emb_m[t] / 0.1 for t in tr.emb})
    after = tr.state_dict()
    for k, g in c["grads"].items():
        assert rel_err(got[k], g) <= 1e-3, (k, rel_err(got[k], g))
        keep = g.abs() > 1e-2 * g.abs().max()               # Adam's first step, compared where the gradient is clear
        if bool(keep.any()):
            assert (after[k].cpu()[keep].double() - c["after"][k][keep].double()).abs().max() <= 1e-5, k
    if case == "one_train":
        # S = 1: both similarities are 0, so loss_aux is exactly 0 and the step is the KD step
        lk = kd.train_step(b, x, teacher=t).clone().double().cpu()
        assert float(loss[2]) == 0.0 and torch.equal(loss[:2], lk[:2])
        assert_same_state(tr, kd, "one train row")


def test_a_batch_without_train_rows_is_nan_and_steps_as_kd():
    c, tr, kd, t, obj, b, x, loss = fixture_run("no_train")
    lk = kd.train_step(b, x, teacher=t).clone()
    assert bool(torch.isnan(loss).all()) and bool(torch.isnan(c["loss"]).all()) and bool(torch.isnan(lk[:2]).all())
    assert obj.sample().numel() == 0
    assert_same_state(tr, kd, "no train row")


# ------------------------------------------------------------------------------------------------ 4. fp64 oracle
def test_three_steps_match_the_fp64_oracle():
    """The engine's own dropout masks and draws (S < n on every batch) fed to oracle/mag_gsp.py, one torch Adam over the
    fp64 model."""
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    obj = BatchGSP(H, H_T, "rbf", BETA, 64)
    tr = student(rel, gsp=obj)
    p, L = 0.5, 2
    params = {k: v.double().cpu().requires_grad_(True) for k, v in tr.state_dict().items()}
    teacher = {k: v.double().cpu() for k, v in t.state_dict().items()}
    x_cpu = {k: v.cpu() for k, v in x.items()}
    opt = torch.optim.Adam(list(params.values()), lr=LR)
    for step, b in enumerate(batches(data, 3, seed=5)):
        loss = tr.train_step(b, x, teacher=t).clone()
        n = b.node_type.numel()
        assert obj.sample().numel() == 64 < int(b.train_mask.sum())
        masks = [ops.dropout_mask(n, H, p, tr.seed, l + step * L).bool().cpu() for l in range(L - 1)]
        cb = SimpleNamespace(**{k: getattr(b, k).cpu() for k in ("edge_index", "edge_attr", "node_type", "local_node_idx", "y",
                                                                 "train_mask")})
        ref, ref_cls, ref_aux = omg.gpw_step_loss(params, teacher, x_cpu, cb, masks, "rbf", obj.sample().cpu(), BETA)
        opt.zero_grad()
        ref.backward()
        opt.step()
        for got, want in ((loss[0], ref), (loss[1], ref_cls), (loss[2], ref_aux)):
            want = float(want.detach())
            assert abs(float(got) - want) <= 2e-5 * max(1.0, abs(want)), (step, loss, ref, ref_aux)
    sd = tr.state_dict()
    for k, v in params.items():
        assert rel_err(sd[k], v) < 5e-4, k


# ------------------------------------------------------------------------------------------------ 5. MAG scale
def fp64_gradient(fs, ft, kernel, beta, rows=1024):
    """beta * d mean((sim_s - sim_t)^2) / d fs in float64, the S x S matrices formed in row chunks (fs, ft: the S sampled
    rows of the two out_feats)."""
    fs, ft = fs.double(), ft.double()
    S = fs.shape[0]
    if kernel in ("cosine", "poly"):
        nrm = fs.norm(dim=1, keepdim=True).clamp_min(1e-12)
        xs, xt = fs / nrm, ft / ft.norm(dim=1, keepdim=True).clamp_min(1e-12)
    else:
        raise NotImplementedError(kernel)
    g = torch.empty_like(xs)
    for r0 in range(0, S, rows):
        gs, gt = xs[r0:r0 + rows] @ xs.t(), xt[r0:r0 + rows] @ xt.t()
        if kernel == "cosine":
            dG = 2.0 / S ** 2 * (gs - gt)
        else:
            dG = 2.0 / S ** 2 * (gs * gs - gt * gt) * 2 * gs
        g[r0:r0 + rows] = 2 * dG @ xs                      # dG is symmetric: d xs = (dG + dG^T) xs
        del gs, gt, dG
    d = (g - xs * (xs * g).sum(1, keepdim=True)) / nrm     # the normalise backward
    return beta * d


def test_mag_scale_step_at_the_scripts_settings():
    """The 2 x 32 student against the 3 x 512 teacher on a MAG-shaped batch (20,000 roots, walk_length 2) with more than
    24,576 train rows, poly, beta 1, S = 24576 (192 chunks of 128 rows): the loss equals the eager route's bit for bit, and
    both routes' gradients at the sampled rows are held to the fp64 gradient, the fused one no further from it."""
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    from bench_rgcn import mag_graph
    data, x, num_nodes, relations, C_mag = mag_graph(1.0)
    x = {k: v.cuda() for k, v in x.items()}
    b = next(b for b in sampling.GraphSAINTRandomWalkSampler(data, batch_size=20000, walk_length=2, num_steps=6, seed=0)
             if int(b.train_mask.sum()) > 24576)
    tm = b.train_mask
    n = int(tm.sum())
    mk = lambda hidden, L, seed, gsp=None: RGCNTrainer(128, hidden, C_mag, L, 0.5, num_nodes, list(x), len(relations),  # noqa: E731
                                                       relations, lr=0.005, seed=seed, gsp=gsp)
    t = mk(512, 3, 0)
    obj = BatchGSP(32, 512)
    assert (obj.kernel, obj.beta, obj.max_samples) == ("poly", 1.0, 24576)
    fused, eager = mk(32, 2, 1, obj), mk(32, 2, 1)
    seen = {}
    fb = obj.forward_backward

    def record(*a, **k):
        seen["d"] = r = fb(*a, **k)
        return r
    obj.forward_backward = record
    got = fused.train_step(b, x, teacher=t).clone()
    sample = obj.sample().cpu()
    assert np.array_equal(sample.numpy(), og.sample_perm(n, fused.seed, SAMPLE_STREAM)[:24576])
    assert criterion.gsp_chunk_rows(24576) == 128
    ref = eager_step(eager, t, b, x, obj, sample.numpy())
    assert torch.equal(got[:2], ref[:2]) and torch.equal(got[2], eager.loss_aux), (got, ref)
    ga, gb = fused._named(fused.grads, {}), eager._named(eager.grads, {})
    for k in gb:
        assert rel_err(ga[k], gb[k]) < 1e-3, (k, rel_err(ga[k], gb[k]))
    # the gradient at the sampled rows: the fused route's (internal order), the eager route's (autograd) and fp64's
    inds = sample.cuda()
    train_int = fused._fwd["train_int"]
    d_fused = seen["d"][train_int[inds]]
    feat = fused.out_feat()[tm].detach().requires_grad_(True)
    t_feat = t.out_feat()[tm]
    with torch.enable_grad():
        eager_aux(t_feat, tm.new_ones(n), obj, sample.numpy())(feat).backward()
    d_eager = feat.grad[inds]
    d64 = fp64_gradient(fused.out_feat()[tm][inds], t_feat[inds], "poly", obj.beta)
    e_fused, e_eager = rel_err(d_fused, d64), rel_err(d_eager, d64)
    assert e_fused <= max(2 * e_eager, 1e-5), (e_fused, e_eager)


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_refusals_do_no_device_work():
    data, x, rel = small_mag(1)
    b = batches(data, 1, seed=5)[0]
    n = int(b.train_mask.sum())
    t = teacher_of(rel)
    obj = BatchGSP(H, H_T, "poly", BETA, 48)
    every = BatchGSP(H, H_T, "poly", BETA)
    tr, plain, tr_all = student(rel, gsp=obj), student(rel), student(rel, gsp=every)
    narrow = teacher_of(rel, hidden=H_T + 8)
    torch.cuda.synchronize()
    before = (lib.launch_count(), tr.params.clone(), tr_all.params.clone(), int(tr.step_count), int(tr_all.step_count))
    refusals = {
        "gsp= and the gcrd= / lsp=": lambda: student(rel, gsp=BatchGSP(H, H_T), lsp=BatchLSP(H)),
        "hidden width": lambda: student(rel, gsp=BatchGSP(H + 8, H_T)),
        "aux=": lambda: tr.train_step(b, x, teacher=t, aux=lambda f: f.sum()),
        "pass teacher=": lambda: tr.train_step(b, x),
        "pass teacher= ": lambda: tr.train_step(b, x, teacher_logits=torch.zeros(n, C, device="cuda")),
        "teacher hidden width": lambda: tr.train_step(b, x, teacher=narrow),
        "no gsp= objective": lambda: plain.train_step(b, x, teacher=t, sample=torch.arange(4)),
        "no sample to inject": lambda: tr_all.train_step(b, x, teacher=t, sample=torch.arange(n)),
    }
    for k, bad in enumerate((torch.arange(47), torch.zeros(48, dtype=torch.long), torch.arange(48) + n - 47)):
        refusals[f"sample {k}"] = lambda bad=bad: tr.train_step(b, x, teacher=t, sample=bad)
    for what, call in refusals.items():
        with pytest.raises(ValueError, match=None if what.startswith("sample") else what.strip()):
            call()
    torch.cuda.synchronize()
    assert lib.launch_count() == before[0]
    assert torch.equal(tr.params, before[1]) and torch.equal(tr_all.params, before[2])
    assert (int(tr.step_count), int(tr_all.step_count)) == before[3:]
