"""LSP in the captured PPI student step (lsp.PerGraphLSP with engine_ppi.PPIGATTrainer): bit for bit the eager
``train_step(i, aux=lambda f: criterion_ppi.lpw_criterion(...)[2], beta=beta)`` path for every kernel in BCE and KD form;
an epoch of graph replays against the same epoch of eager steps, twice; one step against the reference's own train() with
--training lpw (tests/golden/ppi_lsp.pt) and the fp64 oracle; every refusal."""
from pathlib import Path

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion_ppi, engine_ppi, lib, synthetic
from efficient_gnns_b200.lsp import PerGraphLSP
from oracle import ppi as oppi
from test_oracle_ppi_lsp import T_FEAT, after_entries, oracle_lsp_step

pytestmark = pytest.mark.gpu
GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "ppi_lsp.pt")
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
    edges = [ei.cuda() for _, _, ei in graphs]
    return graphs, [t.clone() for t in logits], [f.clone() for f in feats], edges


def state(tr):
    return [tr.loss_out, tr.grads, tr.params, tr.exp_avg, tr.exp_avg_sq]


def assert_same(a, b):
    for k, (u, v) in enumerate(zip(state(a), state(b))):
        assert torch.equal(u, v), k


def eager_step(tr, i, feats, edges, kernel, beta):
    aux = lambda f: criterion_ppi.lpw_criterion(tr.logits().detach(), tr.y[i], f, feats[i], edges[i], kernel, 1)[2]  # noqa: E731
    return tr.train_step(i, aux=aux, beta=beta)


@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("form", ["bce", "kd"])
def test_step_equals_eager_aux_path_bitwise(problem, kernel, form):
    graphs, logits, feats, edges = problem
    teach = logits if form == "kd" else None
    obj = PerGraphLSP(feats, edges, 136, kernel=kernel, beta=BETA)
    a = engine_ppi.student(graphs, teacher_logits=teach, seed=2, lsp=obj)
    b = engine_ppi.student(graphs, teacher_logits=teach, seed=2)
    for i in (0, 2, 1, 0):
        a.train_step(i)
        eager_step(b, i, feats, edges, kernel, BETA)
        assert torch.equal(obj.loss_aux, b.loss_out[2:3]) and torch.equal(a.loss_out[2:3], obj.loss_aux)
        assert_same(a, b)
    assert torch.isfinite(a.loss_out).all()


def test_epoch_of_graph_replays_equals_eager_steps_bitwise():
    graphs = synthetic.make_ppi_graphs("train", 1, 0.2)[:4]
    assert len({g[0].shape[0] for g in graphs}) == 4
    gen = torch.Generator().manual_seed(7)
    feats = [torch.randn(g[0].shape[0], 1024, generator=gen).relu().cuda() for g in graphs]
    edges = [g[2].cuda() for g in graphs]
    runs = []
    for mode in ("eager", "graph"):
        obj = PerGraphLSP(feats, edges, 136, kernel="cosine", beta=BETA)
        tr = engine_ppi.student(graphs, seed=3, lsp=obj)
        if mode == "graph":
            tr.capture()
            assert int(tr.step_count.item()) == 0
        per_epoch = []
        for epoch in range(2):              # the second epoch replays graphs captured before any step ran
            if mode == "eager":
                losses = torch.stack([tr.train_step(i).clone() for i in tr.epoch_order(epoch)])
            else:
                losses = tr.train_epoch(epoch)
            torch.cuda.synchronize()
            per_epoch.append((losses.clone(), tr.params.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone()))
        runs.append(per_epoch)
    for (e0, g0) in zip(*runs):
        for u, v in zip(e0, g0):
            assert torch.equal(u, v)
    assert (runs[0][0][0][:, 2] > 0).all()


def test_launches_per_step_include_the_lsp_part():
    graphs = synthetic.make_ppi_graphs("train", 0, 0.2)[:2]
    feats = [torch.rand(g[0].shape[0], 136, device="cuda") for g in graphs]
    plain = engine_ppi.student(graphs).launches_per_step(1)
    with_lsp = engine_ppi.student(graphs, lsp=PerGraphLSP(feats, [g[2].cuda() for g in graphs], 136)).launches_per_step(1)
    assert with_lsp >= plain + 3                        # lsp_student, the SpMM, the scaled scatter


@pytest.mark.parametrize("kernel", KERNELS)
def test_designed_graph_step_against_the_reference_and_fp64(kernel):
    case = GOLD["cases"][kernel]
    x, y, ei = GOLD["x"], GOLD["y"].float(), GOLD["edge_index"].long()
    # TeacherNet's out_feat restated in fp64 (checked against the reference's own on the CPU), rounded to fp32 as the
    # reference's teacher produces it
    obj = PerGraphLSP([T_FEAT.float().cuda()], [ei.cuda()], 136, kernel=kernel, beta=GOLD["beta"])
    tr = engine_ppi.student([(x, y, ei)], in_channels=GOLD["in_channels"], out_channels=GOLD["out_channels"],
                            lr=GOLD["lr"], lsp=obj)
    tr.load_state_dict(oppi.seeded_state(oppi.layers_of("student", GOLD["out_channels"]), GOLD["in_channels"],
                                         GOLD["seeds"]["student"]))
    loss = tr.train_step(0).clone().double().cpu()
    l64, g64, _ = oracle_lsp_step(kernel)
    for ref in (case["loss"], l64):
        assert rel(loss[:2], ref[:2]) <= 1e-4
        assert abs(loss[2] - ref[2]) <= 1e-4 * abs(ref[2]) + 1e-8
    got = tr.named_gradients()
    for k, g in g64.items():
        assert rel(got[k], g) <= 1e-3, (k, rel(got[k], g))
        for part, v in case["grads"][k].items():
            assert rel(oppi.fingerprint(got[k].cpu())[part], v) <= 1e-3, (k, part)
    after = tr.state_dict()
    for k, ref in case["after"].items():
        # Adam's first step: compared where the gradient is clearly nonzero (lr * g / |g| is a sign of noise elsewhere)
        idx = after_entries(g64[k].numel())
        g = g64[k].reshape(-1)
        keep = g[idx].abs() > 1e-2 * g.abs().max()
        mine = after[k].cpu().reshape(-1)[idx]
        assert (mine[keep].double() - ref[keep].double()).abs().max() <= 1e-5, k


def test_refusals(problem):
    graphs, _, feats, edges = problem
    n0 = graphs[0][0].shape[0]
    for bad in ([edges[0][:, :0]] + edges[1:],                                   # a graph with no edges
                [torch.cat([edges[0], torch.tensor([[0], [n0]], device="cuda")], 1)] + edges[1:]):   # outside its graph
        with pytest.raises(ValueError):
            PerGraphLSP(feats, bad, 136)
    for kw in (dict(hidden=lib.LSP_MAX_F + 4), dict(criterion="mse")):
        with pytest.raises(ValueError):
            PerGraphLSP(feats, edges, **{"hidden": 136, **kw})
    with pytest.raises(ValueError):
        PerGraphLSP(feats[:2], edges, 136)                                       # counts differ
    tr = engine_ppi.student(graphs, lsp=PerGraphLSP(feats, edges, 136))
    with pytest.raises(ValueError):                                              # aux= together with lsp=
        tr.train_step(0, aux=lambda f: f.sum())
    with pytest.raises(ValueError):                                              # built for another graph count
        engine_ppi.student(graphs[:2], lsp=PerGraphLSP(feats, edges, 136))
    with pytest.raises(ValueError):                                              # built for other graph sizes
        engine_ppi.student(graphs[::-1], lsp=PerGraphLSP(feats, edges, 136))
    with pytest.raises(ValueError):                                              # built for another hidden width
        engine_ppi.student(graphs, lsp=PerGraphLSP(feats, edges, 128))
    padded = [(2, 66, True), (2, 121, False)]                                    # 66 is stored 68 wide per head
    with pytest.raises(ValueError):
        engine_ppi.PPIGATTrainer(graphs, padded, lsp=PerGraphLSP(feats, edges, 132))
