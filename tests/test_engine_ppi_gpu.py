"""PPIGATTrainer (the fused step of the reference's PPI StudentNet / TeacherNet) and the kernels added for it.

References: tests/golden/ppi_model.pt (the reference's own classes) and oracle/ppi.py in fp64.  The designed graph of the
fixture has a hub row above the hub threshold, a node with only its self-loop, a self-loop already in edge_index and a
duplicate edge; the synthetic graphs are PPI-shaped (synthetic.make_ppi_graphs) at reduced scale."""
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion_ppi, engine_ppi, lib, ops, synthetic
from efficient_gnns_b200 import nn as enn
from efficient_gnns_b200.nn import _hub_args
from oracle import criterion as ocrit, ppi as oppi

pytestmark = pytest.mark.gpu
GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "ppi_model.pt")
U = 2.0 ** -24


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def designed():
    return GOLD["x"], GOLD["y"].float(), GOLD["edge_index"].long()


def oracle_step(kind_layers, x, y, ei, state, t=None, aux64=None, beta=1.0):
    """fp64 loss and gradients of one step (aux64(feat) -> auxiliary loss)."""
    n = x.shape[0]
    row, col = oppi.adjacency(ei, n)
    st = {k: v.double().clone().requires_grad_(True) for k, v in state.items() if "lin_r" not in k}
    st.update({k.replace("lin_l", "lin_r"): v for k, v in st.items() if "lin_l" in k})
    logits, feat = oppi.forward(x.double(), row, col, st, kind_layers)
    losses = oppi.loss(logits, y.double(), None if t is None else t.double())
    total = losses[0] + (beta * aux64(feat) if aux64 is not None else 0)
    total.backward()
    return logits.detach(), feat.detach(), torch.stack([v.detach() for v in losses]), \
        {k: v.grad for k, v in st.items() if "lin_r" not in k}


def check_grads(tr, ref, tol):
    got = tr.named_gradients()
    for k, g in ref.items():
        assert rel(got[k], g) <= tol, (k, rel(got[k], g))


# ------------------------------------------------------------------------------------------------ the new kernels alone
@pytest.fixture(scope="module")
def hub_graph():
    x, _, ei = designed()
    g = engine_ppi._Graph(ei, x.shape[0], torch.device("cuda"))
    assert g.G.n_hub >= 1
    return g


@pytest.mark.parametrize("H,D", [(2, 68), (4, 256), (2, 124), (3, 6)])
def test_gat_aggregate_elu_is_epi_bit_for_bit_and_elu(hub_graph, H, D):
    G, n, K = hub_graph.G, hub_graph.n, H * D
    gen = torch.Generator().manual_seed(K)
    cat = torch.randn(n, 2 * K, generator=gen).cuda()
    ft, res = cat[:, :K], cat[:, K:]
    a = torch.rand(G.nnz, H, generator=gen).cuda()
    bias = torch.randn(K, generator=gen).cuda()
    ref = torch.empty(n, K, device="cuda")
    ops.gat_aggregate_epi(G, None, a, ft, ref, H, res=res, bias=bias)
    ZA = torch.full((n, 2 * K + 4), float("nan"), device="cuda")          # Z and A side by side: pitched outputs, canaries
    Z, A = ZA[:, :K], ZA[:, K:2 * K]
    for _ in range(2):
        ops.gat_aggregate_elu(G, a, ft, Z, A, H, res=res, bias=bias)
        assert torch.equal(Z, ref)
    assert torch.isnan(ZA[:, 2 * K:]).all()
    e64 = F.elu(Z.double())
    assert ((A.double() - e64).abs() <= 2 * U * e64.abs() + 1e-38).all()


def test_gat_aggregate_elu_refuses_an_act_buffer_narrower_than_the_epi_width(hub_graph):
    G, n, H, D = hub_graph.G, hub_graph.n, 2, 68
    K = H * D
    ft = torch.randn(n, K, device="cuda")
    a = torch.rand(G.nnz, H, device="cuda")
    Z = torch.empty(n, K, device="cuda")
    act = torch.empty(n * K + 1, device="cuda")[1:].view(n, K)           # 4-byte aligned only: the epi path is float4
    with pytest.raises(lib.B200GnnError):
        ops.gat_aggregate_elu(G, a, ft, Z, act, H)


def test_elu_bwd_matches_autograd():
    n, K = 777, 136
    gen = torch.Generator().manual_seed(3)
    buf = torch.randn(n, 3 * K, generator=gen).cuda() * 3
    Z, dA = buf[:, :K], buf[:, K:2 * K]
    out = torch.full((n, K + 8), float("nan"), device="cuda")
    ops.elu_bwd(dA, Z, out=out[:, :K])
    z = Z.clone().requires_grad_(True)
    F.elu(z).backward(dA)
    assert ((out[:, :K] - z.grad).abs() <= 2 * U * z.grad.abs() + 1e-38).all()
    assert torch.isnan(out[:, K:]).all()
    zd = Z.double()
    ref64 = dA.double() * torch.where(zd > 0, torch.ones_like(zd), zd.exp())
    assert ((out[:, :K].double() - ref64).abs() <= 4 * U * ref64.abs() + 1e-38).all()


def tail(agg, res, bc, bl, H, Dp, C, y=None, t=None, ldga_extra=8):
    n = agg.shape[0]
    logits = torch.full((n, C + 3), float("nan"), device="cuda")
    dagg = torch.full((n, H * Dp + ldga_extra), float("nan"), device="cuda")
    dres = torch.full((n, Dp + 4), float("nan"), device="cuda")
    loss = torch.full((3,), float("nan"), device="cuda")
    if y is None:
        ops.ppi_logits_loss(agg, res, bc, bl, H, C, logits[:, :C])
    else:
        ops.ppi_logits_loss(agg, res, bc, bl, H, C, logits[:, :C], labels=y, teacher_logits=t, alpha=0.5, T=1.0,
                            d_agg=dagg[:, :H * Dp], d_res=dres[:, :Dp], loss_out=loss)
    return logits, dagg, dres, loss


@pytest.mark.parametrize("H", [2, 6])
@pytest.mark.parametrize("kd", [False, True])
def test_logits_tail_against_fp64(H, kd):
    n, C, Dp = 2345, 121, 124
    gen = torch.Generator().manual_seed(H + 10 * kd)
    aggb = torch.randn(n, H * Dp + 4, generator=gen)
    for h in range(H):
        aggb[:, h * Dp + C:(h + 1) * Dp] = 0                                # the aggregation's padded columns are zero
    agg = aggb.cuda()[:, :H * Dp]
    res = torch.randn(n, 2 * Dp, generator=gen).cuda()[:, Dp:]
    bc, bl = torch.randn(Dp, generator=gen).cuda(), torch.randn(Dp, generator=gen).cuda()
    y = (torch.rand(n, C, generator=gen) < 0.3).float().cuda()
    t = (torch.randn(n, C, generator=gen) * 2).cuda() if kd else None
    logits, dagg, dres, loss = tail(agg, res, bc, bl, H, Dp, C, y, t)
    again = tail(agg, res, bc, bl, H, Dp, C, y, t)
    for u, v in zip((logits, dagg, dres, loss), again):
        assert torch.equal(u.nan_to_num(7.0), v.nan_to_num(7.0))           # two runs: identical bits
    # fp64 restatement of the same association
    a64 = agg.double().view(n, H, Dp)[:, :, :C]
    z64 = (a64.mean(1) + bc[:C].double()) + (res[:, :C].double() + bl[:C].double())
    mag = a64.abs().mean(1) + bc[:C].double().abs() + res[:, :C].double().abs() + bl[:C].double().abs()
    assert ((logits[:, :C].double() - z64).abs() <= (H + 4) * U * mag).all()
    assert torch.isnan(logits[:, C:]).all()
    zr = z64.clone().requires_grad_(True)
    l64 = oppi.loss(zr, y.double(), None if t is None else t.double())
    l64[0].backward()
    assert (loss.double().cpu() - torch.stack([v.detach() for v in l64]).cpu()).abs().max() <= 1e-5 * l64[0].item()
    zf = logits[:, :C].double().requires_grad_(True)                   # the gradient at the kernel's own logits
    oppi.loss(zf, y.double(), None if t is None else t.double())[0].backward()
    gz = zf.grad
    tolg = 8 * U * (gz.abs() + 1.0 / (n * C))
    assert ((dres[:, :C].double() - gz).abs() <= tolg).all()
    for h in range(H):
        assert ((dagg[:, h * Dp:h * Dp + C].double() - gz / H).abs() <= tolg).all()
        assert (dagg[:, h * Dp + C:(h + 1) * Dp] == 0).all()
    assert (dres[:, C:Dp] == 0).all() and torch.isnan(dres[:, Dp:]).all() and torch.isnan(dagg[:, H * Dp:]).all()


def test_logits_tail_eval_writes_logits_only():
    n, C, Dp, H = 300, 19, 20, 2
    agg = torch.randn(n, H * Dp, device="cuda")
    res = torch.randn(n, Dp, device="cuda")
    bc, bl = torch.randn(Dp, device="cuda"), torch.randn(Dp, device="cuda")
    logits, dagg, dres, loss = tail(agg, res, bc, bl, H, Dp, C)
    assert torch.isfinite(logits[:, :C]).all() and torch.isnan(dagg).all() and torch.isnan(dres).all() and torch.isnan(loss).all()


# ------------------------------------------------------------------------------------------------ the fixture
@pytest.mark.parametrize("kind", ["student", "teacher"])
def test_presets_reproduce_the_reference_fixture(kind):
    c = GOLD["models"][kind]
    x, y, ei = designed()
    F_in, C = GOLD["in_channels"], GOLD["out_channels"]
    state = oppi.seeded_state(oppi.layers_of(kind, C), F_in, c["seed"])
    make = getattr(engine_ppi, kind)
    for mode in ("supervised", "kd"):
        t = [GOLD["teacher_logits"]] if mode == "kd" else None
        tr = make([(x, y, ei)], in_channels=F_in, out_channels=C, teacher_logits=t)
        tr.load_state_dict(state)
        logits, feat = tr.predict(x.cuda(), ei.cuda(), return_feat=True)
        for name, got in (("logits_eval", logits), ("out_feat_eval", feat)):
            fp = oppi.fingerprint(got.cpu())
            for k, v in c[name].items():
                assert rel(fp[k], v) <= 1e-4, (name, k)
        loss = tr.train_step(0).clone()
        assert rel(loss, c[mode]["loss"]) <= 1e-5
        got = tr.named_gradients()
        for k, v in c[mode]["grads"].items():
            fp = oppi.fingerprint(got[k].cpu())
            for part, ref in v.items():
                assert rel(fp[part], ref) <= 1e-3, (mode, k, part)


# ------------------------------------------------------------------------------------------------ one step against fp64
def ppi_graphs(scale=0.25, k=3, seed=0):
    return synthetic.make_ppi_graphs("train", seed, scale)[:k]


@pytest.mark.parametrize("kd", [False, True])
def test_student_step_against_fp64_oracle(kd):
    graphs = ppi_graphs()
    sizes = [g[0].shape[0] for g in graphs]
    assert len(set(sizes)) == len(sizes)
    gen = torch.Generator().manual_seed(5)
    teach = [torch.randn(g[0].shape[0], 121, generator=gen) * 2 for g in graphs] if kd else None
    tr = engine_ppi.student(graphs, teacher_logits=teach)
    state = oppi.seeded_state(oppi.layers_of("student", 121), 50, 9)
    layers = oppi.layers_of("student", 121)
    for i, (x, y, ei) in enumerate(graphs):
        tr.load_state_dict(state)
        loss = tr.train_step(i).clone()
        logits64, feat64, l64, g64 = oracle_step(layers, x, y, ei, state, None if teach is None else teach[i])
        assert rel(tr.logits(), logits64) <= 1e-5 and rel(tr.out_feat(), feat64) <= 1e-5
        assert rel(loss, l64) <= 1e-5
        check_grads(tr, g64, 1e-4)


@pytest.mark.parametrize("kind", ["student", "teacher"])
def test_designed_graph_step_against_fp64_oracle(kind):
    x, y, ei = designed()
    t = GOLD["teacher_logits"]
    tr = getattr(engine_ppi, kind)([(x, y, ei)], in_channels=10, out_channels=19, teacher_logits=[t])
    state = oppi.seeded_state(oppi.layers_of(kind, 19), 10, 4)
    tr.load_state_dict(state)
    loss = tr.train_step(0).clone()
    logits64, feat64, l64, g64 = oracle_step(oppi.layers_of(kind, 19), x, y, ei, state, t)
    assert rel(tr.logits(), logits64) <= 1e-5 and rel(tr.out_feat(), feat64) <= 1e-5 and rel(loss, l64) <= 1e-5
    check_grads(tr, g64, 1e-4)


def test_teacher_full_width_step_against_fp64_oracle():
    x, y, ei = synthetic.make_ppi_graphs("train", 3, 0.1)[0]
    tr = engine_ppi.teacher([(x, y, ei)])
    assert [len(b) for b in tr.blocks] == [4, 4, 2]                        # the 2048-wide stacked output: 4 wgrad blocks
    state = oppi.seeded_state(oppi.layers_of("teacher", 121), 50, 8)
    tr.load_state_dict(state)
    loss = tr.train_step(0).clone()
    logits64, feat64, l64, g64 = oracle_step(oppi.layers_of("teacher", 121), x, y, ei, state)
    assert rel(tr.logits(), logits64) <= 1e-5 and rel(tr.out_feat(), feat64) <= 1e-5 and rel(loss, l64) <= 1e-5
    check_grads(tr, g64, 1e-4)


@pytest.mark.parametrize("crit", ["fitnet", "lpw"])
def test_aux_hook_seeds_the_backward(crit):
    x, y, ei = ppi_graphs(k=1)[0]
    n = x.shape[0]
    gen = torch.Generator().manual_seed(2)
    tfeat = torch.randn(n, 136, generator=gen).relu()
    tr = engine_ppi.student([(x, y, ei)], teacher_feat=[tfeat])
    state = oppi.seeded_state(oppi.layers_of("student", 121), 50, 6)
    tr.load_state_dict(state)
    tf_c, ei_c = tr.teacher_feat[0], ei.cuda()
    dummy = torch.zeros(n, 2, dtype=torch.float64), torch.zeros(n, dtype=torch.long)
    if crit == "fitnet":
        aux = lambda f: criterion_ppi.fitnet_criterion(tr.logits().detach(), tr.y[0], f, tf_c, 1000)[2]     # noqa: E731
        aux64 = lambda f: ocrit.fitnet_criterion(*dummy, f, tfeat.double(), 1000)[2]                        # noqa: E731
    else:
        aux = lambda f: criterion_ppi.lpw_criterion(tr.logits().detach(), tr.y[0], f, tf_c, ei_c, "cosine", 100)[2]   # noqa: E731
        aux64 = lambda f: ocrit.lpw_criterion(*dummy, f, tfeat.double(), ei, "cosine", 100)[2]                       # noqa: E731
    loss = tr.train_step(0, aux=aux, beta=0.5).clone()
    logits64, feat64, l64, g64 = oracle_step(oppi.layers_of("student", 121), x, y, ei, state, aux64=aux64, beta=0.5)
    with torch.no_grad():
        a64 = aux64(feat64)
    assert rel(loss[0], l64[0] + 0.5 * a64) <= 1e-4 and rel(loss[2], a64) <= 1e-4
    check_grads(tr, g64, 1e-3)


# ------------------------------------------------------------------------------------------------ optimiser, padding, graphs
class ModuleNet(torch.nn.Module):
    """The reference's StudentNet composed from the package's nn.GATConv + torch.nn.Linear + F.elu (the module path)."""

    def __init__(self, layers, fin):
        super().__init__()
        for i, (H, D, concat) in enumerate(layers, start=1):
            out = H * D if concat else D
            setattr(self, f"conv{i}", enn.GATConv(fin, D, heads=H, concat=concat))
            setattr(self, f"lin{i}", torch.nn.Linear(fin, out))
            fin = out
        self.L = len(layers)

    def forward(self, x, ei):
        for i in range(1, self.L + 1):
            z = getattr(self, f"conv{i}")(x, ei) + getattr(self, f"lin{i}")(x)
            x = F.elu(z) if i < self.L else z
        return x


def true_mask(tr, graphs):
    """params-shaped mask of the entries that appear in state_dict()."""
    probe = engine_ppi.PPIGATTrainer(graphs, tr.layers, tr.F, tr.C)
    probe.load_state_dict({k: torch.ones_like(v) for k, v in tr.state_dict().items()})
    return probe.params != 0


def test_five_adam_steps_match_the_module_path_and_padding_stays_zero():
    x, y, ei = ppi_graphs(k=1)[0]
    tr = engine_ppi.student([(x, y, ei)])
    m = ModuleNet(oppi.layers_of("student", 121), 50).cuda()
    m.load_state_dict({k: v.cuda() for k, v in tr.state_dict().items()})
    opt = torch.optim.Adam(m.parameters(), lr=0.005)
    xc, yc, eic = x.cuda(), y.cuda(), ei.cuda()
    for _ in range(5):
        tr.train_step(0)
        opt.zero_grad()
        F.binary_cross_entropy_with_logits(m(xc, eic), yc).backward()
        opt.step()
    sd = tr.state_dict()
    for k, v in m.state_dict().items():
        assert rel(sd[k], v) <= 2e-3, k
    mask = true_mask(tr, [(x, y, ei)])
    for buf in (tr.params, tr.grads, tr.exp_avg, tr.exp_avg_sq):
        assert (buf[~mask] == 0).all()
    assert int(tr.step_count.item()) == 5


def test_epoch_of_graph_replays_is_bit_identical_to_eager():
    graphs = ppi_graphs(scale=0.2, k=4, seed=1)
    gen = torch.Generator().manual_seed(7)
    teach = [torch.randn(g[0].shape[0], 121, generator=gen) for g in graphs]
    runs = []
    for mode in ("eager", "graph", "graph"):
        tr = engine_ppi.student(graphs, teacher_logits=teach, seed=3)
        if mode == "graph":
            tr.capture()
            assert int(tr.step_count.item()) == 0
        order = tr.epoch_order(0)
        assert sorted(order) == list(range(4)) and order != list(range(4))
        if mode == "eager":
            losses = torch.stack([tr.train_step(i).clone() for i in order])
        else:
            losses = tr.train_epoch(0)
        torch.cuda.synchronize()
        runs.append((losses, tr.params.clone(), tr.exp_avg.clone(), tr.exp_avg_sq.clone()))
    for other in runs[1:]:
        for a, b in zip(runs[0], other):
            assert torch.equal(a, b)


def test_predict_on_a_two_graph_batch_against_fp64():
    (x1, _, e1), (x2, _, e2) = ppi_graphs(k=2)
    x = torch.cat([x1, x2])
    ei = torch.cat([e1, e2 + x1.shape[0]], dim=1)
    tr = engine_ppi.student(ppi_graphs(k=1))
    state = oppi.seeded_state(oppi.layers_of("student", 121), 50, 12)
    tr.load_state_dict(state)
    logits, feat = tr.predict(x.cuda(), ei.cuda(), return_feat=True)
    row, col = oppi.adjacency(ei, x.shape[0])
    ref, feat64 = oppi.forward(x.double(), row, col, {k: v.double() for k, v in state.items()}, oppi.layers_of("student", 121))
    assert rel(logits, ref) <= 1e-5 and rel(feat, feat64) <= 1e-5


def test_predict_plans_follow_the_graph_not_the_address():
    """Two different graphs of the same shape from fresh tensors in sequence, then one edited in place: each prediction
    uses its own adjacency."""
    tr = engine_ppi.student(ppi_graphs(k=1))
    state = oppi.seeded_state(oppi.layers_of("student", 121), 50, 13)
    tr.load_state_dict(state)
    s64 = {k: v.double() for k, v in state.items()}
    x, _, ei = ppi_graphs(k=1)[0]
    n, E = x.shape[0], ei.shape[1]
    gen = torch.Generator().manual_seed(21)

    def check(ei_dev, ei_cpu):
        got = tr.predict(x.cuda(), ei_dev)
        row, col = oppi.adjacency(ei_cpu, n)
        ref, _ = oppi.forward(x.double(), row, col, s64, oppi.layers_of("student", 121))
        assert rel(got, ref) <= 1e-5
    for _ in range(3):                                                    # same n, same E, different edges, fresh tensors
        e = torch.randint(0, n, (2, E), generator=gen)
        check(e.cuda(), e)
        torch.cuda.synchronize()
    e = torch.randint(0, n, (2, E), generator=gen)
    ed = e.cuda()
    check(ed, e)
    e[1] = torch.randint(0, n, (E,), generator=gen)                       # edited in place: a new version of the same tensor
    ed.copy_(e)
    check(ed, e)
    assert len(tr._predict_cache) <= 8


def test_state_dict_round_trip_and_refusals():
    graphs = ppi_graphs(k=1)
    for kind in ("student", "teacher"):
        tr = getattr(engine_ppi, kind)(graphs)
        sd = tr.state_dict()
        assert {k: tuple(v.shape) for k, v in sd.items()} == oppi.state_shapes(oppi.layers_of(kind, 121), 50)
        assert list(sd) == list(ModuleNet(oppi.layers_of(kind, 121), 50).state_dict())
        tr2 = getattr(engine_ppi, kind)(graphs, seed=99)
        tr2.load_state_dict(sd)
        assert all(torch.equal(v, tr2.state_dict()[k]) for k, v in sd.items())
        assert torch.equal(tr.params, tr2.params)
    for kw in (dict(dropout=0.2), dict(attn_dropout=0.1), dict(weight_decay=5e-4)):
        with pytest.raises(ValueError):
            engine_ppi.student(graphs, **kw)
