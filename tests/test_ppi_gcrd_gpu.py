"""G-CRD in the captured PPI student step (gcrd.PerGraphGCRD with engine_ppi.PPIGATTrainer): the step against the eager
``train_step(i, aux=criterion_ppi.nce_criterion(...))`` path with torch projection heads and a torch Adam, in BCE and KD form,
with every row and with an injected sample; an epoch of graph replays against the same epoch of eager steps, twice; capture
leaves every state alone; one step against the reference's own train() with --training nce (tests/golden/ppi_gcrd.pt) and
the fp64 oracle; every refusal before any launch; the launch count; the heads' state dicts."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion_ppi, engine_ppi, lib, synthetic
from efficient_gnns_b200.gcrd import PerGraphGCRD
from efficient_gnns_b200.lsp import PerGraphLSP
from oracle import ppi as oppi, ppi_gcrd as opg
from test_oracle_ppi_gcrd import GOLD, oracle_gcrd_step
from test_oracle_ppi_lsp import T_FEAT, after_entries

pytestmark = pytest.mark.gpu
BETA, NCE_T, LR = 0.1, 0.075, 0.005


@pytest.fixture(scope="module")
def problem():
    """Three PPI-shaped graphs of different sizes, the TeacherNet's out_feat [n_i, 1024] and logits on each."""
    graphs = synthetic.make_ppi_graphs("train", 0, 0.25)[:3]
    assert len({g[0].shape[0] for g in graphs}) == 3
    teacher = engine_ppi.teacher(graphs, seed=5)
    logits, feats = zip(*(teacher.predict(x.cuda(), ei.cuda(), return_feat=True) for x, _, ei in graphs))
    return graphs, [t.clone() for t in logits], [f.clone() for f in feats]


def torch_heads(obj):
    sp = torch.nn.Sequential(torch.nn.Linear(obj.H, obj.P), torch.nn.BatchNorm1d(obj.P), torch.nn.ReLU()).cuda()
    tp = torch.nn.Sequential(torch.nn.Linear(obj.F_t, obj.P), torch.nn.BatchNorm1d(obj.P), torch.nn.ReLU()).cuda()
    sp.load_state_dict({k: v.cuda() for k, v in obj.student_proj_state_dict().items()})
    tp.load_state_dict({k: v.cuda() for k, v in obj.teacher_proj_state_dict().items()})
    return sp, tp


def head_grads(obj):
    """(reference key, gradient, sits in front of a BatchNorm) of both heads."""
    return [("s0.weight", obj.gW_s, False), ("s0.bias", obj.gb_s, True), ("s1.weight", obj.ggamma_s, False),
            ("s1.bias", obj.gbeta_s, False), ("t0.weight", obj.gW_t[:, :obj.F_t], False), ("t0.bias", obj.gb_t, True),
            ("t1.weight", obj.ggamma_t, False), ("t1.bias", obj.gbeta_t, False)]


def check_grads(pairs, tol=1e-4):
    scale = max(b.abs().max().item() for _, _, b, _ in pairs)
    for name, a, b, pre_bn in pairs:
        if pre_bn:       # a bias in front of BatchNorm: its exact gradient is 0, both sides carry rounding only
            assert a.abs().max().item() < 1e-5 * scale and b.abs().max().item() < 1e-5 * scale, name
        else:
            assert rel_err(a, b) < tol, (name, rel_err(a, b))


@pytest.mark.parametrize("S", [16384, 128])
@pytest.mark.parametrize("form", ["bce", "kd"])
@pytest.mark.parametrize("i", [0, 2])
def test_step_equals_eager_aux_path(problem, form, S, i):
    graphs, logits, feats = problem
    teach = logits if form == "kd" else None
    obj = PerGraphGCRD(feats, 136, max_samples=S, nce_T=NCE_T, beta=BETA, seed=4)
    a = engine_ppi.student(graphs, teacher_logits=teach, seed=2, lr=LR, gcrd=obj)
    b = engine_ppi.student(graphs, teacher_logits=teach, seed=2, lr=LR)
    n = graphs[i][0].shape[0]
    sample = np.random.RandomState(3).choice(n, S, replace=False) if S < n else None
    sp, tp = torch_heads(obj)
    opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=LR)
    aux = lambda f: criterion_ppi.nce_criterion(b.logits().detach(), b.y[i], sp(f), tp(feats[i]), 1.0, NCE_T, S,  # noqa: E731
                                                sampled_inds=sample)[2]
    opt.zero_grad()
    ref = b.train_step(i, aux=aux, beta=BETA).clone()
    opt.step()
    got = a.train_step(i, sample=None if sample is None else torch.as_tensor(sample)).clone()
    if sample is not None:
        assert torch.equal(obj.sample().cpu(), torch.as_tensor(sample, dtype=torch.int64))
    assert abs(float(got[0]) - float(ref[0])) < 2e-5 * abs(float(ref[0]))
    assert abs(float(got[2]) - float(ref[2])) < 2e-5 * abs(float(ref[2]))
    assert torch.equal(got[1], ref[1]) and torch.equal(got[2], obj.loss_aux[0])
    ga, gb = a.named_gradients(), b.named_gradients()
    check_grads([(k, ga[k], gb[k], False) for k in gb])
    ref_g = {"s" + k: p.grad for k, p in sp.named_parameters()}
    ref_g.update({"t" + k: p.grad for k, p in tp.named_parameters()})
    check_grads([(k, g, ref_g[k], pre) for k, g, pre in head_grads(obj)])
    for mine, theirs in ((obj.student_proj_state_dict(), sp.state_dict()), (obj.teacher_proj_state_dict(), tp.state_dict())):
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(mine[k], theirs[k]) < 1e-5, k
        assert int(mine["1.num_batches_tracked"]) == int(theirs["1.num_batches_tracked"]) == 1
    assert int(obj.step_count.item()) == int(a.step_count.item()) == 1


def snapshot(tr, obj):
    out = [tr.params, tr.exp_avg, tr.exp_avg_sq, tr.step_count, obj.params, obj.exp_avg, obj.exp_avg_sq, obj.step_count,
           obj.rm_s, obj.rv_s, obj.rm_t, obj.rv_t]
    out = [t.clone() for t in out]
    for sd in (obj.student_proj_state_dict(), obj.teacher_proj_state_dict()):
        out.append(sd["1.num_batches_tracked"].clone())
    return out


def test_epoch_of_graph_replays_equals_eager_steps_bitwise():
    graphs = synthetic.make_ppi_graphs("train", 1, 0.2)[:4]
    assert len({g[0].shape[0] for g in graphs}) == 4
    gen = torch.Generator().manual_seed(7)
    feats = [torch.randn(g[0].shape[0], 1024, generator=gen).relu().cuda() for g in graphs]
    runs, samples = [], []
    for mode in ("eager", "graph"):
        obj = PerGraphGCRD(feats, 136, max_samples=96, seed=1)
        tr = engine_ppi.student(graphs, seed=3, gcrd=obj)
        if mode == "graph":
            before = snapshot(tr, obj)
            tr.capture()
            for u, v in zip(before, snapshot(tr, obj)):
                assert torch.equal(u, v)
        per_epoch = []
        for epoch in range(2):              # the second epoch replays graphs captured before any step ran
            if mode == "eager":
                rows = []
                for i in tr.epoch_order(epoch):
                    rows.append(tr.train_step(i).clone())
                    samples.append(obj.sample().cpu())
                losses = torch.stack(rows)
            else:
                losses = tr.train_epoch(epoch)
            torch.cuda.synchronize()
            per_epoch.append([losses.clone()] + snapshot(tr, obj))
        runs.append(per_epoch)
    for e0, g0 in zip(*runs):
        for u, v in zip(e0, g0):
            assert torch.equal(u, v)
    assert (runs[0][0][0][:, 2] > 0).all()
    assert len({tuple(s.tolist()) for s in samples}) == len(samples)        # every step draws afresh
    assert int(runs[1][1][8].item()) == 8                                    # the heads' Adam ran once per step


@pytest.mark.parametrize("case", ["full", "s128"])
def test_designed_graph_step_against_the_reference_and_fp64(case):
    c = GOLD["cases"][case]
    x, y, ei = GOLD["x"], GOLD["y"].float(), GOLD["edge_index"].long()
    obj = PerGraphGCRD([T_FEAT.float().cuda()], 136, proj_dim=GOLD["proj_dim"], max_samples=c["max_samples"],
                       nce_T=GOLD["nce_T"], beta=GOLD["beta"], seed=GOLD["seeds"]["heads"])
    for mine, seeded in zip((obj.student_proj_state_dict(), obj.teacher_proj_state_dict()),
                            opg.seeded_heads(136, 1024, GOLD["proj_dim"], GOLD["seeds"]["heads"])):
        for k, v in seeded.items():
            assert torch.equal(mine[k].cpu(), v), k
    tr = engine_ppi.student([(x, y, ei)], in_channels=GOLD["in_channels"], out_channels=GOLD["out_channels"],
                            lr=GOLD["lr"], gcrd=obj)
    tr.load_state_dict(oppi.seeded_state(oppi.layers_of("student", GOLD["out_channels"]), GOLD["in_channels"],
                                         GOLD["seeds"]["student"]))
    loss = tr.train_step(0, sample=c["sample"]).clone().double().cpu()
    o64 = oracle_gcrd_step(case)
    for ref in (c["loss"], o64["loss"]):
        assert rel_err(loss, ref) <= 1e-4, (loss, ref)
    got = {"model": tr.named_gradients(),
           "sproj": {k[1:]: g for k, g, _ in head_grads(obj) if k[0] == "s"},
           "tproj": {k[1:]: g for k, g, _ in head_grads(obj) if k[0] == "t"}}
    after = {"model": tr.state_dict(), "sproj": obj.student_proj_state_dict(), "tproj": obj.teacher_proj_state_dict()}
    for group, g64 in o64["grads"].items():
        scale = max(v.abs().max().item() for v in g64.values())
        for k, g in g64.items():
            if group != "model" and k == "0.bias":          # in front of BatchNorm: exactly 0, rounding only
                assert got[group][k].abs().max().item() < 1e-5 * scale, (group, k)
                continue
            assert rel_err(got[group][k], g) <= 1e-3, (group, k, rel_err(got[group][k], g))
            for part, v in c["grads"][group][k].items():
                assert rel_err(oppi.fingerprint(got[group][k].cpu())[part], v) <= 1e-3, (group, k, part)
            # Adam's first step: compared where the gradient is clearly nonzero (lr * g / |g| is a sign of noise elsewhere)
            idx = after_entries(g.numel())
            flat = g.reshape(-1)
            keep = flat[idx].abs() > 1e-2 * flat.abs().max()
            mine = after[group][k].cpu().reshape(-1)[idx]
            assert (mine[keep].double() - c["after"][group][k][keep].double()).abs().max() <= 1e-5, (group, k)
    for group, sd in c["running"].items():
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(after[group][k], sd[k]) <= 1e-5, (group, k)
            assert rel_err(after[group][k], o64["after"][group][k]) <= 1e-5, (group, k)
        assert int(after[group]["1.num_batches_tracked"]) == int(sd["1.num_batches_tracked"]) == 1


def test_refusals_before_any_launch(problem):
    graphs, _, feats = problem
    obj = PerGraphGCRD(feats, 136)
    lsp = PerGraphLSP([f[:, :136].contiguous() for f in feats], [g[2].cuda() for g in graphs], 136)
    padded = [(2, 66, True), (2, 121, False)]                                    # 66 is stored 68 wide per head
    cases = [
        lambda: engine_ppi.student(graphs, gcrd=obj, lsp=lsp),                   # two objectives
        lambda: engine_ppi.PPIGATTrainer(graphs, padded, gcrd=PerGraphGCRD(feats, 132)),   # a padded out_feat
        lambda: engine_ppi.teacher(graphs, gcrd=obj),                            # out_feat 1024 wide
        lambda: PerGraphGCRD(feats, 1024),                                       # the head's wgrad takes at most 512
        lambda: PerGraphGCRD([torch.zeros(f.shape[0], 2052, device="cuda") for f in feats], 136),   # teacher above 2048
        lambda: PerGraphGCRD(feats, 136, proj_dim=200),                          # not a multiple of 32
        lambda: PerGraphGCRD(feats, 136, proj_dim=512),                          # above 256
        lambda: PerGraphGCRD([feats[0], feats[1][0]], 136),                      # not 2-D
        lambda: engine_ppi.student(graphs[:2], gcrd=obj),                        # graph count
        lambda: engine_ppi.student(graphs[::-1], gcrd=obj),                      # graph sizes
        lambda: engine_ppi.student(graphs, gcrd=PerGraphGCRD(feats, 128)),       # hidden width
    ]
    for k, make in enumerate(cases):
        before = lib.launch_count()
        with pytest.raises(ValueError):
            make()
        assert lib.launch_count() == before, k
    tr, plain = engine_ppi.student(graphs, gcrd=obj), engine_ppi.student(graphs)
    before = lib.launch_count()
    with pytest.raises(ValueError):                                              # aux= together with gcrd=
        tr.train_step(0, aux=lambda f: f.sum())
    with pytest.raises(ValueError):                                              # sample= without gcrd=
        plain.train_step(0, sample=torch.arange(4))
    assert lib.launch_count() == before
    drawn = engine_ppi.student(graphs, gcrd=PerGraphGCRD(feats, 136, max_samples=64))
    for bad in (torch.arange(63), torch.arange(64) * 0, torch.arange(64) + graphs[0][0].shape[0] - 63):
        with pytest.raises(ValueError):                                          # wrong size, repeated, out of the graph
            drawn.train_step(0, sample=bad)


def test_launches_per_step_include_the_gcrd_part(problem):
    graphs, _, feats = problem
    plain = engine_ppi.student(graphs).launches_per_step(1)
    full = engine_ppi.student(graphs, gcrd=PerGraphGCRD(feats, 136)).launches_per_step(1)
    drawn = engine_ppi.student(graphs, gcrd=PerGraphGCRD(feats, 136, max_samples=64)).launches_per_step(1)
    # splits, statistics GEMMs and finalizes of both heads, operands, the InfoNCE chunk, its finish, the backward, two
    # BatchNorm applies, two weight gradients, the transpose, the input-gradient split and GEMM, the heads' Adam
    assert full >= plain + 20
    assert drawn > full                                                          # the sampler


def test_state_dicts_load_into_torch_heads_and_round_trip(problem):
    graphs, _, feats = problem
    obj = PerGraphGCRD(feats, 136, max_samples=64)
    tr = engine_ppi.student(graphs, gcrd=obj)
    tr.train_step(1)
    tr.train_step(0)
    sp, tp = torch_heads(obj)                                                    # strict load into nn.Sequential
    assert int(sp.state_dict()["1.num_batches_tracked"]) == 2
    other = PerGraphGCRD(feats, 136, seed=9)
    other.load_student_proj_state_dict(sp.state_dict())
    other.load_teacher_proj_state_dict(tp.state_dict())
    for a, b in ((obj.student_proj_state_dict(), other.student_proj_state_dict()),
                 (obj.teacher_proj_state_dict(), other.teacher_proj_state_dict())):
        for k in a:
            assert torch.equal(a[k].cpu(), b[k].cpu()), k
    assert obj.teacher_proj_state_dict()["0.weight"].shape == (256, 1024)
