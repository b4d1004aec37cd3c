"""GSP in the captured PPI student step (gsp.PerGraphGSP with engine_ppi.PPIGATTrainer): bit for bit the eager
``train_step(i, aux=lambda f: criterion_ppi.gpw_criterion(..., f, teacher_feat[i], kernel, 1, max_samples,
sampled_inds=...)[2], beta)`` path for every kernel in BCE and KD form, with every row and with an injected sample; two
epochs of graph replays against the same epochs of eager steps, with every row and with a fresh on-device draw per step;
one step against the reference's own train() with --training gpw (tests/golden/ppi_gsp.pt) and the fp64 oracle; the
launch count, the teacher similarities' memory and every refusal."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion_ppi, engine_ppi, lib, synthetic
from efficient_gnns_b200.gcrd import PerGraphGCRD
from efficient_gnns_b200.gsp import PerGraphGSP
from efficient_gnns_b200.lsp import PerGraphLSP
from oracle import ppi as oppi
from test_oracle_ppi_gsp import CASES, GOLD, fingerprint, oracle_gsp_step
from test_oracle_ppi_lsp import T_FEAT, after_entries

pytestmark = pytest.mark.gpu
KERNELS = ["cosine", "poly", "l2", "rbf"]
BETA = 100.0


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.fixture(scope="module")
def problem():
    """Three PPI-shaped graphs of different sizes, the TeacherNet's out_feat [n_i, 1024] and logits on each."""
    graphs = synthetic.make_ppi_graphs("train", 0, 0.25)[:3]
    assert len({g[0].shape[0] for g in graphs}) == 3
    teacher = engine_ppi.teacher(graphs, seed=5)
    logits, feats = zip(*(teacher.predict(x.cuda(), ei.cuda(), return_feat=True) for x, _, ei in graphs))
    return graphs, [t.clone() for t in logits], [f.clone() for f in feats]


def state(tr):
    return [tr.loss_out, tr.grads, tr.params, tr.exp_avg, tr.exp_avg_sq]


def assert_same(a, b):
    for k, (u, v) in enumerate(zip(state(a), state(b))):
        assert torch.equal(u, v), k


@pytest.mark.parametrize("S", [8192, 96])
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("form", ["bce", "kd"])
def test_step_equals_eager_aux_path_bitwise(problem, kernel, form, S):
    graphs, logits, feats = problem
    teach = logits if form == "kd" else None
    obj = PerGraphGSP(feats, 136, kernel=kernel, beta=BETA, max_samples=S)
    a = engine_ppi.student(graphs, teacher_logits=teach, seed=2, gsp=obj)
    b = engine_ppi.student(graphs, teacher_logits=teach, seed=2)
    for step, i in enumerate((0, 2, 1, 0)):        # several steps: d out_feat must not keep the previous graph's rows
        n = graphs[i][0].shape[0]
        sample = np.random.RandomState(step).choice(n, S, replace=False) if S < n else None
        a.train_step(i, sample=None if sample is None else torch.as_tensor(sample))
        aux = lambda f: criterion_ppi.gpw_criterion(b.logits().detach(), b.y[i], f, feats[i], kernel, 1, S,  # noqa: E731
                                                    sampled_inds=sample)[2]
        b.train_step(i, aux=aux, beta=BETA)
        if sample is not None:
            assert torch.equal(obj.sample().cpu(), torch.as_tensor(sample, dtype=torch.int64))
        assert torch.equal(obj.loss_aux, b.loss_out[2:3]) and torch.equal(a.loss_out[2:3], obj.loss_aux)
        assert_same(a, b)
    assert torch.isfinite(a.loss_out).all()
    if kernel != "rbf":         # rbf similarities of distinct 1024-wide teacher rows underflow: its term can round to 0
        assert float(a.loss_out[2]) > 0


@pytest.mark.parametrize("S", [8192, 96])
def test_epochs_of_graph_replays_equal_eager_steps_bitwise(S):
    graphs = synthetic.make_ppi_graphs("train", 1, 0.2)[:4]
    assert len({g[0].shape[0] for g in graphs}) == 4
    gen = torch.Generator().manual_seed(7)
    feats = [torch.randn(g[0].shape[0], 1024, generator=gen).relu().cuda() for g in graphs]
    runs, samples = [], []
    for mode in ("eager", "graph"):
        obj = PerGraphGSP(feats, 136, kernel="cosine", beta=BETA, max_samples=S)
        tr = engine_ppi.student(graphs, seed=3, gsp=obj)
        if mode == "graph":
            before = [t.clone() for t in (tr.params, tr.exp_avg, tr.exp_avg_sq, tr.step_count)]
            tr.capture()
            for u, v in zip(before, (tr.params, tr.exp_avg, tr.exp_avg_sq, tr.step_count)):
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
            per_epoch.append((losses.clone(), tr.params.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone()))
        runs.append(per_epoch)
    for e0, g0 in zip(*runs):
        for u, v in zip(e0, g0):
            assert torch.equal(u, v)
    assert (runs[0][0][0][:, 2] > 0).all()
    if S < min(g[0].shape[0] for g in graphs):
        assert len({tuple(s.tolist()) for s in samples}) == len(samples)         # every step draws afresh


@pytest.mark.parametrize("case", CASES)
def test_designed_graph_step_against_the_reference_and_fp64(case):
    c = GOLD["cases"][case]
    x, y, ei = GOLD["x"], GOLD["y"].float(), GOLD["edge_index"].long()
    # TeacherNet's out_feat restated in fp64 (checked against the reference's own on the CPU), rounded to fp32 as the
    # reference's teacher produces it
    obj = PerGraphGSP([T_FEAT.float().cuda()], 136, kernel=c["kernel"], beta=GOLD["beta"], max_samples=c["max_samples"])
    tr = engine_ppi.student([(x, y, ei)], in_channels=GOLD["in_channels"], out_channels=GOLD["out_channels"],
                            lr=GOLD["lr"], gsp=obj)
    tr.load_state_dict(oppi.seeded_state(oppi.layers_of("student", GOLD["out_channels"]), GOLD["in_channels"],
                                         GOLD["seeds"]["student"]))
    loss = tr.train_step(0, sample=c["sample"]).clone().double().cpu()
    o64 = oracle_gsp_step(case)
    for ref in (c["loss"], o64["loss"]):
        assert rel(loss[:2], ref[:2]) <= 1e-4
        assert abs(loss[2] - ref[2]) <= 1e-4 * abs(ref[2]) + 1e-8
    got = tr.named_gradients()
    for k, g in o64["grads"].items():
        assert rel(got[k], g) <= 1e-3, (k, rel(got[k], g))
        for part, v in c["grads"][k].items():
            assert rel(fingerprint(got[k].cpu())[part], v) <= 1e-3, (k, part)
    after = tr.state_dict()
    # the sampled case records no parameters after the step: the fp64 oracle's stand in
    refs = c["after"] if "after" in c else {k: v.reshape(-1)[after_entries(v.numel())] for k, v in o64["after"].items()}
    for k, ref in refs.items():
        # Adam's first step: compared where the gradient is clearly nonzero (lr * g / |g| is a sign of noise elsewhere)
        g = o64["grads"][k].reshape(-1)
        idx = after_entries(g.numel())
        keep = g[idx].abs() > 1e-2 * g.abs().max()
        mine = after[k].cpu().reshape(-1)[idx]
        assert (mine[keep].double() - ref[keep].double()).abs().max() <= 1e-5, k


def test_launches_per_step_include_the_gsp_part(problem):
    graphs, _, feats = problem
    plain = engine_ppi.student(graphs).launches_per_step(1)
    full = engine_ppi.student(graphs, gsp=PerGraphGSP(feats, 136)).launches_per_step(1)
    drawn = engine_ppi.student(graphs, gsp=PerGraphGSP(feats, 136, max_samples=64)).launches_per_step(1)
    # operands, the two splits, one chunk (graph 1 is below gsp_chunk_rows' 1,280 rows): the Gram GEMM, the pair pass and
    # dG . x; the finish and the backward
    assert graphs[1][0].shape[0] <= 1280
    assert full == plain + 8
    assert drawn > full                                                          # the sampler


def test_teacher_similarities_take_one_flat_allocation(problem):
    _, _, feats = problem
    obj = PerGraphGSP(feats, 136, kernel="l2")
    sizes = [int(f.shape[0]) for f in feats]
    assert obj.sim_bytes == sum(n * n * 4 for n in sizes)
    assert obj.sim_flat.numel() * 4 == obj.sim_bytes
    base = obj.sim_flat.data_ptr()
    off = 0
    for r, n in zip(obj.graphs, sizes):
        assert tuple(r.sim_t.shape) == (n, n) and r.sim_t.data_ptr() == base + off * 4
        assert torch.equal(r.sim_t.diagonal(), torch.zeros(n, device="cuda"))   # the l2 diagonal is exactly 0
        off += n * n


def test_refusals_before_any_launch(problem):
    graphs, _, feats = problem
    obj = PerGraphGSP(feats, 136)
    lsp = PerGraphLSP([f[:, :136].contiguous() for f in feats], [g[2].cuda() for g in graphs], 136)
    gcrd = PerGraphGCRD(feats, 136)
    padded = [(2, 66, True), (2, 121, False)]                                    # 66 is stored 68 wide per head
    cases = [
        lambda: engine_ppi.student(graphs, gsp=obj, lsp=lsp),                    # two objectives
        lambda: engine_ppi.student(graphs, gsp=obj, gcrd=gcrd),
        lambda: engine_ppi.PPIGATTrainer(graphs, padded, gsp=obj),               # a padded out_feat
        lambda: engine_ppi.student(graphs[:2], gsp=obj),                         # graph count
        lambda: engine_ppi.student(graphs[::-1], gsp=obj),                       # graph sizes
        lambda: engine_ppi.teacher(graphs, gsp=obj),                             # out_feat width 1024, built for 136
        lambda: PerGraphGSP(feats, 136, kernel="gaussian"),                      # unknown kernel
        lambda: PerGraphGSP(feats, 136, max_samples=0),
        lambda: PerGraphGSP([], 136),                                            # no graphs
        lambda: PerGraphGSP([feats[0], feats[1][0]], 136),                       # not 2-D
        lambda: PerGraphGSP([feats[0], feats[1][:, :512]], 136),                 # two teacher widths
        lambda: PerGraphGSP(feats, 134),                                         # not a multiple of 4
        lambda: PerGraphGSP(feats, lib.GSP_ROWS_MAX_F + 4),                      # wider than the row passes take
    ]
    for k, make in enumerate(cases):
        before = lib.launch_count()
        with pytest.raises(ValueError):
            make()
        assert lib.launch_count() == before, k
    tr, plain = engine_ppi.student(graphs, gsp=obj), engine_ppi.student(graphs)
    before = lib.launch_count()
    with pytest.raises(ValueError):                                              # aux= together with gsp=
        tr.train_step(0, aux=lambda f: f.sum())
    with pytest.raises(ValueError, match="no gcrd= objective"):                  # sample= with neither objective
        plain.train_step(0, sample=torch.arange(4))
    with pytest.raises(ValueError):                                              # S = n: no sample to inject
        tr.train_step(0, sample=torch.arange(graphs[0][0].shape[0]))
    assert lib.launch_count() == before
    drawn = engine_ppi.student(graphs, gsp=PerGraphGSP(feats, 136, max_samples=64))
    before = lib.launch_count()
    for bad in (torch.arange(63), torch.arange(64) * 0, torch.arange(64) + graphs[0][0].shape[0] - 63):
        with pytest.raises(ValueError):                                          # wrong size, repeated, out of the graph
            drawn.train_step(0, sample=bad)
    assert lib.launch_count() == before
