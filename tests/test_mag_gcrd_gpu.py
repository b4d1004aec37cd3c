"""G-CRD in the R-GCN student step on GraphSAINT batches (``RGCNTrainer(..., gcrd=BatchGCRD(...)).train_step(b, x,
teacher=t)``, the reference's MAG ``--training nce``): the step against the eager ``teacher_logits=`` + ``aux=nce_criterion``
path with torch heads and a torch Adam, the on-device sample, the reference's own step (tests/golden/mag_gcrd.pt), the fp64
restatement oracle/mag_gcrd.py over three steps, one step at the MAG scripts' size (S = 24576), and the refusals."""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion, lib, ops, sampling
from efficient_gnns_b200.gcrd import SAMPLE_STREAM, BatchGCRD
from efficient_gnns_b200.lsp import BatchLSP
from efficient_gnns_b200.rgcn import RGCNTrainer
from oracle import gcrd as og, mag_gcrd as omg
from test_mag_lsp_gpu import assert_same_state
from test_oracle_mag_gcrd import GOLD, HEAD_KEYS, seeded_heads
from test_ppi_gcrd_gpu import check_grads, head_grads, torch_heads
from test_rgcn_train_gpu import NODES, batches, small_mag

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(900)]

H, H_T, C, LR, BETA, NCE_T, PROJ = 24, 32, 7, 0.005, 0.1, 0.075, 64


def student(rel, gcrd=None, seed=3, lsp=None):
    return RGCNTrainer(16, H, C, 2, 0.5, NODES, [0], len(rel), rel, lr=LR, seed=seed, gcrd=gcrd, lsp=lsp)


def teacher_of(rel, hidden=H_T, seed=11):
    return RGCNTrainer(16, hidden, C, 3, 0.5, NODES, [0], len(rel), rel, lr=LR, seed=seed)


def heads(max_samples=24576, seed=4, hidden=H, teacher_hidden=H_T, proj=PROJ):
    return BatchGCRD(hidden, teacher_hidden, proj, max_samples=max_samples, nce_T=NCE_T, beta=BETA, seed=seed)


def eager_step(tr, t, b, x, obj, sample, lr=LR):
    """The route that needs no gcrd=: the teacher's own forward, torch heads loaded from the state dicts of obj (the fused
    step's heads as they were before it), nce_criterion through ``aux=`` and a torch Adam on the heads.  Returns (loss,
    torch heads)."""
    tm = b.train_mask
    tl = t.forward(b, x, training=False)[tm]
    t_feat = t.out_feat()
    n = int(tm.sum())
    sp, tp = torch_heads(obj)
    opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=lr)
    dummy = torch.zeros(n, 2, device="cuda"), torch.zeros(n, dtype=torch.long, device="cuda")
    aux = lambda f: criterion.nce_criterion(*dummy, sp(f[tm]), tp(t_feat[tm]), 1.0, obj.nce_T, obj.max_samples,  # noqa: E731
                                            sampled_inds=sample)[2]
    opt.zero_grad()
    loss = tr.train_step(b, x, teacher_logits=tl, beta=obj.beta, aux=aux).clone()
    opt.step()
    return loss, sp, tp


def compare_with_eager(fused, eager, got, ref, sp, tp, skip=()):
    """skip: head gradients (head_grads names) compared elsewhere."""
    obj = fused.gcrd
    assert abs(float(got[0]) - float(ref[0])) <= 2e-5 * abs(float(ref[0])), (got, ref)
    assert abs(float(got[2]) - float(eager.loss_aux)) <= 2e-5 * abs(float(eager.loss_aux)), (got, eager.loss_aux)
    assert torch.equal(got[1], ref[1]) and torch.equal(got[2], obj.loss_aux[0])
    ga, gb = fused._named(fused.grads, {}), eager._named(eager.grads, {})
    check_grads([(k, ga[k], gb[k], False) for k in gb])
    # the embedding tables' gradients: the first Adam step's first moment is (1 - 0.9) * g (compared on the device: the
    # MAG-scale tables hold millions of rows)
    for t in fused.emb:
        a, e = fused.emb_m[t], eager.emb_m[t]
        assert float((a - e).abs().max()) <= 1e-4 * float(e.abs().max()), t
    ref_g = {"s" + k: p.grad for k, p in sp.named_parameters()}
    ref_g.update({"t" + k: p.grad for k, p in tp.named_parameters()})
    pairs = [(k, g, ref_g[k], pre) for k, g, pre in head_grads(obj) if k not in skip]
    if pairs:
        check_grads(pairs)
    for mine, theirs in ((obj.student_proj_state_dict(), sp.state_dict()), (obj.teacher_proj_state_dict(), tp.state_dict())):
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(mine[k], theirs[k]) < 1e-5, k
        assert int(mine["1.num_batches_tracked"]) == int(theirs["1.num_batches_tracked"])


# ------------------------------------------------------------------------------------------------ 1. the eager path
@pytest.mark.parametrize("rows", ["all", "sampled"])
def test_step_equals_the_eager_aux_step(rows):
    """Three batches with different train-row counts, each the first step of fresh trainers and heads: every row (S >= n)
    or an injected sample of S < n rows."""
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    sizes = set()
    for k, b in enumerate(batches(data, 3, seed=5)):
        n = int(b.train_mask.sum())
        sizes.add(n)
        S = 48 if rows == "sampled" else 24576
        assert (S < n) == (rows == "sampled")
        sample = np.random.RandomState(k).choice(n, S, replace=False) if S < n else None
        fused, eager, probe = student(rel, gcrd=heads(S)), student(rel), heads(S)
        got = fused.train_step(b, x, teacher=t, sample=None if sample is None else torch.as_tensor(sample)).clone()
        ref, sp, tp = eager_step(eager, t, b, x, probe, sample)
        if sample is not None:
            assert torch.equal(fused.gcrd.sample().cpu(), torch.as_tensor(sample, dtype=torch.int64))
        else:
            assert torch.equal(fused.gcrd.sample().cpu(), torch.arange(n))
        compare_with_eager(fused, eager, got, ref, sp, tp)
        assert int(fused.gcrd.step_count) == int(fused.step_count) == 1
    assert len(sizes) == 3


# ------------------------------------------------------------------------------------------------ 2. the sampler
def test_each_step_draws_afresh_at_the_students_step_counter():
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    S = 40
    tr = student(rel, gcrd=heads(S), seed=6)
    drawn = []
    for b in batches(data, 3, seed=7):
        step, n = int(tr.step_count), int(b.train_mask.sum())
        loss = tr.train_step(b, x, teacher=t)
        assert bool(torch.isfinite(loss).all())
        want = og.sample_perm(n, tr.seed, SAMPLE_STREAM + step)[:S]
        assert np.array_equal(tr.gcrd.sample().cpu().numpy(), want), step
        drawn.append(tuple(want.tolist()))
    assert len(set(drawn)) == 3
    assert int(tr.gcrd.step_count) == int(tr.step_count) == 3


# ------------------------------------------------------------------------------------------------ 3. the reference's step
def fixture_run(case):
    """One engine step on the fixture's designed batch: the student at the fixture's state (its dropout masks are this
    trainer's own, seed 0), the heads from seeded_heads, the recorded draw injected."""
    c = GOLD["cases"][case]
    rel = {r: tuple(sd) for r, sd in enumerate(GOLD["relations"])}
    mk = lambda hidden, L, gcrd=None: RGCNTrainer(  # noqa: E731
        GOLD["in_channels"], hidden, GOLD["out_channels"], L, 0.5, GOLD["num_nodes"], [0], len(rel), rel, lr=GOLD["lr"],
        seed=GOLD["seeds"]["dropout"], alpha=GOLD["alpha"], kd_T=GOLD["kd_T"], gcrd=gcrd)
    obj = BatchGCRD(GOLD["hidden"], GOLD["teacher_hidden"], GOLD["proj_dim"], c["max_samples"], GOLD["nce_T"], GOLD["beta"],
                    seed=GOLD["seeds"]["heads"])
    for mine, seeded in zip((obj.student_proj_state_dict(), obj.teacher_proj_state_dict()), seeded_heads()):
        for k, v in seeded.items():
            assert torch.equal(mine[k].cpu(), v), k
    tr, kd, t = mk(GOLD["hidden"], 2, obj), mk(GOLD["hidden"], 2), mk(GOLD["teacher_hidden"], 3)
    for m, sd in ((tr, GOLD["student_state"]), (kd, GOLD["student_state"]), (t, GOLD["teacher_state"])):
        m.load_state_dict({k: v.cuda() for k, v in sd.items()})
    mask = "no_train" if case == "no_train" else "main"
    b = SimpleNamespace(edge_index=GOLD["edge_index"].cuda(), edge_attr=GOLD["edge_type"].cuda(),
                        node_type=GOLD["node_type"].cuda(), local_node_idx=GOLD["local_node_idx"].cuda(),
                        y=GOLD["y"].cuda(), train_mask=GOLD["train_mask"][mask].cuda())
    x = {0: GOLD["x"].cuda()}
    loss = tr.train_step(b, x, teacher=t, sample=c["sample"]).clone().double().cpu()
    return c, tr, kd, t, obj, b, x, loss


@pytest.mark.parametrize("case", ["main/all", "main/sampled"])
def test_designed_batch_step_matches_the_reference(case):
    c, tr, _, _, obj, _, _, loss = fixture_run(case)
    assert rel_err(loss, c["loss"]) <= 1e-4, (loss, c["loss"])
    if c["sample"] is None:
        assert torch.equal(obj.sample().cpu(), torch.arange(int(GOLD["train_mask"]["main"].sum())))
    got = {"model": tr._named(tr.grads, {}),
           "sproj": {k[1:]: g for k, g, _ in head_grads(obj) if k[0] == "s"},
           "tproj": {k[1:]: g for k, g, _ in head_grads(obj) if k[0] == "t"}}
    # the embedding tables' gradients: every row is in the batch, and Adam's first moment after one step is 0.1 * g
    got["model"].update({f"emb_dict.{t}": tr.emb_m[t] / 0.1 for t in tr.emb})
    after = {"model": tr.state_dict(), "sproj": obj.student_proj_state_dict(), "tproj": obj.teacher_proj_state_dict()}
    for group, ref_g in c["grads"].items():
        scale = max(v.abs().max().item() for v in ref_g.values())
        for k, g in ref_g.items():
            if group != "model" and k == "0.bias":          # in front of BatchNorm: exactly 0, rounding only
                assert got[group][k].abs().max().item() < 1e-5 * scale, (group, k)
                continue
            assert rel_err(got[group][k], g) <= 1e-3, (group, k, rel_err(got[group][k], g))
            keep = g.abs() > 1e-2 * g.abs().max()           # Adam's first step, compared where the gradient is clear
            if bool(keep.any()):                            # none where no loss is read (non-paper logits)
                mine = after[group][k].cpu()
                assert (mine[keep].double() - c["after"][group][k][keep].double()).abs().max() <= 1e-5, (group, k)
    for group, sd in c["running"].items():
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(after[group][k], sd[k]) <= 1e-5, (group, k)
        assert int(after[group]["1.num_batches_tracked"]) == int(sd["1.num_batches_tracked"]) == 1


def test_a_batch_without_train_rows_is_nan_and_steps_as_kd():
    """The reference's means over no row are NaN: every loss is NaN, the heads get zero gradients and still take their Adam
    step (num_batches_tracked advances), their running statistics stay, and the model's step is the KD-only step."""
    c, tr, kd, t, obj, b, x, loss = fixture_run("no_train")
    lk = kd.train_step(b, x, teacher=t).clone()
    assert bool(torch.isnan(loss).all()) and bool(torch.isnan(c["loss"]).all()) and bool(torch.isnan(lk[:2]).all())
    assert obj.rows is None and not bool(obj.grads.any())
    assert_same_state(tr, kd, "no train row")
    for mine, seeded, group in zip((obj.student_proj_state_dict(), obj.teacher_proj_state_dict()), seeded_heads(),
                                   ("sproj", "tproj")):
        for k, v in seeded.items():
            if k == "1.num_batches_tracked":
                assert int(mine[k]) == int(c["running"][group][k]) == 1
            else:                                           # Adam from zero moments with a zero gradient moves nothing
                assert torch.equal(mine[k].cpu(), v), (group, k)
    assert int(obj.step_count) == int(tr.step_count) == 1


# ------------------------------------------------------------------------------------------------ 4. fp64 oracle
def test_three_steps_match_the_fp64_oracle():
    """The engine's own dropout masks and draws (S < n on every batch) fed to oracle/mag_gcrd.py, one torch Adam over the
    fp64 model and both heads."""
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    obj = heads(64, seed=2)
    tr = student(rel, gcrd=obj)
    p, L = 0.5, 2
    leaf = lambda sd: {k: v.double().cpu().requires_grad_(True) for k, v in sd.items() if "running" not in k  # noqa: E731
                       and "num_batches" not in k}
    params, sproj, tproj = leaf(tr.state_dict()), leaf(obj.student_proj_state_dict()), leaf(obj.teacher_proj_state_dict())
    running = {"sproj": {k: v.double().cpu() for k, v in obj.student_proj_state_dict().items() if "running" in k},
               "tproj": {k: v.double().cpu() for k, v in obj.teacher_proj_state_dict().items() if "running" in k}}
    teacher = {k: v.double().cpu() for k, v in t.state_dict().items()}
    x_cpu = {k: v.cpu() for k, v in x.items()}
    opt = torch.optim.Adam([{"params": list(params.values())}, {"params": list(sproj.values())},
                            {"params": list(tproj.values())}], lr=LR)
    for step, b in enumerate(batches(data, 3, seed=5)):
        loss = tr.train_step(b, x, teacher=t).clone()
        n = b.node_type.numel()
        assert obj.rows.S < obj.rows.n
        masks = [ops.dropout_mask(n, H, p, tr.seed, l + step * L).bool().cpu() for l in range(L - 1)]
        cb = SimpleNamespace(**{k: getattr(b, k).cpu() for k in ("edge_index", "edge_attr", "node_type", "local_node_idx", "y",
                                                                 "train_mask")})
        ref, ref_cls, ref_aux, stats = omg.nce_step_loss(params, teacher, sproj, tproj, x_cpu, cb, masks, obj.sample().cpu(),
                                                         BETA, NCE_T)
        opt.zero_grad()
        ref.backward()
        opt.step()
        for g in running:
            omg.running_stats(running[g], stats[g], obj.rows.n)
        # the biases in front of BatchNorm have a gradient of rounding noise on both sides, so Adam moves each by lr in a
        # direction of its own; the loss does not depend on them, the running mean does: the oracle takes the engine's
        with torch.no_grad():
            sproj["0.bias"].copy_(obj.b_s.double().cpu())
            tproj["0.bias"].copy_(obj.b_t.double().cpu())
        for got, want in ((loss[0], ref), (loss[1], ref_cls), (loss[2], ref_aux)):
            want = float(want.detach())
            assert abs(float(got) - want) <= 2e-5 * max(1.0, abs(want)), (step, loss, ref, ref_aux)
    # Adam divides by sqrt(v): an entry whose gradient is near Adam's eps moves by an amount that follows fp32 rounding in
    # that gradient, so the parameters after three steps are held to 5e-4 (the losses above to 2e-5)
    sd = tr.state_dict()
    for k, v in params.items():
        assert rel_err(sd[k], v) < 5e-4, k
    for mine, ref, run in ((obj.student_proj_state_dict(), sproj, running["sproj"]),
                           (obj.teacher_proj_state_dict(), tproj, running["tproj"])):
        for k in HEAD_KEYS:
            assert rel_err(mine[k], ref[k]) < 5e-4, k
        for k, v in run.items():
            assert rel_err(mine[k], v) < 1e-5, k
        assert int(mine["1.num_batches_tracked"]) == 3


# ------------------------------------------------------------------------------------------------ 5. MAG scale
def test_mag_scale_step_at_the_scripts_settings_equals_the_eager_path():
    """The 2 x 32 student against the 3 x 512 teacher on a MAG-shaped batch with more than 24,576 train rows, at
    scripts/run_kd_and_aux.sh's settings (proj_dim 128, max_samples 24576, nce_T 0.075, beta 0.1, lr 0.005): the sampler
    at n of about 30,000 and 96 InfoNCE chunks of 256 rows, against the eager path with the same draw."""
    sys.path.insert(0, str(Path(__file__).resolve().parents[1] / "tools"))
    from bench_rgcn import mag_graph
    data, x, num_nodes, relations, C_mag = mag_graph(1.0)
    x = {k: v.cuda() for k, v in x.items()}
    b = next(b for b in sampling.GraphSAINTRandomWalkSampler(data, batch_size=24000, walk_length=2, num_steps=4, seed=0)
             if int(b.train_mask.sum()) > 24576)
    n = int(b.train_mask.sum())
    mk = lambda hidden, L, seed, gcrd=None: RGCNTrainer(128, hidden, C_mag, L, 0.5, num_nodes, list(x), len(relations),  # noqa: E731
                                                        relations, lr=0.005, seed=seed, gcrd=gcrd)
    t = mk(512, 3, 0)
    obj = BatchGCRD(32, 512)
    fused, eager = mk(32, 2, 1, obj), mk(32, 2, 1)
    assert (obj.P, obj.max_samples, obj.nce_T, obj.beta) == (128, 24576, 0.075, 0.1)
    got = fused.train_step(b, x, teacher=t).clone()
    sample = obj.sample().cpu()
    assert np.array_equal(sample.numpy(), og.sample_perm(n, fused.seed, SAMPLE_STREAM)[:24576])
    assert obj.rows.Sp == 24576 and obj.rows.nce.Z.shape[0] == 256
    probe = BatchGCRD(32, 512)                              # the same seed: obj's heads before the step
    ref, sp, tp = eager_step(eager, t, b, x, probe, sample.numpy())
    compare_with_eager(fused, eager, got, ref, sp, tp, skip=[k for k, _, _ in head_grads(obj)])
    # The heads' gradients are sums over n of about 30,000 rows of terms that largely cancel (the BatchNorm backward removes
    # their mean, and InfoNCE's positive and negative terms offset), so both fp32 routes carry cancellation error there.
    # Each is held to the fp64 gradient (the heads in float64 on the same features and draw), and the fused step must be no
    # further from it than the eager path.
    tm = b.train_mask
    sp64, tp64 = (m.double() for m in torch_heads(probe))
    inds = sample.cuda()
    ps, pt = sp64(fused.out_feat()[tm].double())[inds], tp64(t.out_feat()[tm].double())[inds]
    z = torch.nn.functional.normalize(ps) @ torch.nn.functional.normalize(pt).t() / obj.nce_T
    (torch.nn.functional.cross_entropy(z, torch.arange(len(inds), device="cuda")) * obj.beta).backward()
    del z
    g64 = {"s" + k: p.grad for k, p in sp64.named_parameters()}
    g64.update({"t" + k: p.grad for k, p in tp64.named_parameters()})
    g32 = {"s" + k: p.grad for k, p in sp.named_parameters()}
    g32.update({"t" + k: p.grad for k, p in tp.named_parameters()})
    scale = max(g.abs().max().item() for g in g64.values())
    errors = {}
    for name, mine, pre_bn in head_grads(obj):
        if pre_bn:          # a bias in front of BatchNorm: its exact gradient is 0, rounding only
            assert mine.abs().max().item() < 1e-5 * scale, name
            continue
        errors[name] = rel_err(mine, g64[name]), rel_err(g32[name], g64[name])
    assert all(e_fused <= max(2 * e_eager, 1e-4) for e_fused, e_eager in errors.values()), errors


# ------------------------------------------------------------------------------------------------ 6. refusals
def test_refusals_do_no_device_work():
    data, x, rel = small_mag(1)
    b = batches(data, 1, seed=5)[0]
    n = int(b.train_mask.sum())
    t = teacher_of(rel)
    obj = heads(48)
    tr, plain = student(rel, gcrd=obj), student(rel)
    narrow = teacher_of(rel, hidden=H_T + 8)
    one = SimpleNamespace(**{k: getattr(b, k) for k in ("edge_index", "edge_attr", "node_type", "local_node_idx", "y")})
    one.train_mask = torch.zeros_like(b.train_mask)
    one.train_mask[b.train_mask.nonzero()[0]] = True
    torch.cuda.synchronize()
    before = (lib.launch_count(), tr.params.clone(), obj.params.clone(), int(tr.step_count), int(obj.step_count),
              [v.clone() for v in (obj.rm_s, obj.rv_s, obj.rm_t, obj.rv_t)])
    refusals = {
        "lsp=": lambda: student(rel, gcrd=heads(), lsp=BatchLSP(H)),
        "hidden width": lambda: student(rel, gcrd=heads(hidden=H + 8)),
        "aux=": lambda: tr.train_step(b, x, teacher=t, aux=lambda f: f.sum()),
        "pass teacher=": lambda: tr.train_step(b, x, teacher_logits=torch.zeros(n, C, device="cuda")),
        "teacher head built for width": lambda: tr.train_step(b, x, teacher=narrow),
        "no gcrd= objective": lambda: plain.train_step(b, x, teacher=t, sample=torch.arange(4)),
        "one train row": lambda: tr.train_step(one, x, teacher=t),
    }
    for k, bad in enumerate((torch.arange(47), torch.zeros(48, dtype=torch.long), torch.arange(48) + n - 47)):
        refusals[f"sample {k}"] = lambda bad=bad: tr.train_step(b, x, teacher=t, sample=bad)
    for what, call in refusals.items():
        with pytest.raises(ValueError, match=None if what.startswith("sample") else what):
            call()
    torch.cuda.synchronize()
    assert lib.launch_count() == before[0]
    assert torch.equal(tr.params, before[1]) and torch.equal(obj.params, before[2])
    assert (int(tr.step_count), int(obj.step_count)) == before[3:5]
    for u, v in zip((obj.rm_s, obj.rv_s, obj.rm_t, obj.rv_t), before[5]):
        assert torch.equal(u, v)
