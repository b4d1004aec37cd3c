"""Fused R-GCN training step on GraphSAINT batches (efficient_gnns_b200.rgcn.RGCNTrainer) — the loop body of the reference's
MAG train() (mag_pyg/gnn.py:174-268) — and the kernels it adds: ReLU/dropout backward, embedding Adam, widened weight
gradient."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import lib, ops, sampling
from efficient_gnns_b200.graphdata import Data
from efficient_gnns_b200.rgcn import RGCNTrainer
from efficient_gnns_b200.sparse import device_argsort
from oracle import rgcn_plan as orp
from test_gemm_numerics_gpu import BIAS_HI, BIAS_LO, CANARY, _gemm_check, _gen, _mean_signed_rel, _pow2, _wgrad_beta

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]


# ------------------------------------------------------------------------------------------------ a small MAG-like graph
NODES = {0: 900, 1: 700, 2: 60, 3: 120}                   # paper (features), author, institution, field (embeddings)
BASE = [(1, 2, 900), (1, 0, 2500), (0, 0, 3000), (0, 3, 2000)]   # affiliated_with, writes, cites, has_topic


def small_mag(seed=0, F_in=16, C=7):
    g = torch.Generator().manual_seed(seed)
    rels = []
    for s, d, e in BASE:
        src, dst = torch.randint(0, NODES[s], (e,), generator=g), torch.randint(0, NODES[d], (e,), generator=g)
        rels.append((s, d, torch.stack([src, dst])))
    # reverse relations and the undirected cites relation, as main() adds them (mag_pyg/gnn.py:325-337)
    for k in (0, 1, 3):
        s, d, ei = rels[k]
        rels.append((d, s, ei.flip(0)))
    s, d, ei = rels[2]
    rels[2] = (s, d, torch.unique(torch.cat([ei, ei.flip(0)], 1), dim=1))
    off = {0: 0}
    for t in range(1, 4):
        off[t] = off[t - 1] + NODES[t - 1]
    eis, ets = [], []
    for r, (s, d, ei) in enumerate(rels):
        eis.append(torch.stack([ei[0] + off[s], ei[1] + off[d]])); ets.append(torch.full((ei.shape[1],), r))
    n = sum(NODES.values())
    node_type = torch.cat([torch.full((NODES[t],), t) for t in range(4)])
    local = torch.cat([torch.arange(NODES[t]) for t in range(4)])
    x = torch.randn(NODES[0], F_in, generator=g)
    y = torch.full((n, 1), -1, dtype=torch.long)
    y[:NODES[0], 0] = (x @ torch.randn(F_in, C, generator=g)).argmax(1)
    train = torch.zeros(n, dtype=torch.bool)
    train[:NODES[0]] = torch.rand(NODES[0], generator=g) < 0.7
    data = Data(edge_index=torch.cat(eis, 1), edge_attr=torch.cat(ets), node_type=node_type, local_node_idx=local, y=y,
                train_mask=train)
    data.num_nodes = n
    relations = {r: (s, d) for r, (s, d, _) in enumerate(rels)}
    return data.to("cuda"), {0: x.cuda()}, relations


def trainer(relations, F_in=16, H=24, C=7, L=2, p=0.5, seed=0, lr=0.01):
    return RGCNTrainer(F_in, H, C, L, p, NODES, [0], len(relations), relations, lr=lr, seed=seed)


def batches(data, n, walk_length=2, batch_size=150, seed=1):
    return list(sampling.GraphSAINTRandomWalkSampler(data, batch_size=batch_size, walk_length=walk_length, num_steps=n, seed=seed))


# ------------------------------------------------------------------------------------------------ 1. plan
def test_device_plan_is_bit_exact_against_the_oracle():
    data, _, rel = small_mag(0)
    tr = trainer(rel)
    for b in batches(data, 3):
        P = tr.plan(b)
        want = orp.batch_plan(b.edge_index.cpu().numpy(), b.edge_attr.cpu().numpy(), b.node_type.cpu().numpy(),
                              tr.rel_src.cpu().numpy(), tr.rel_dst.cpu().numpy(), tr.T)
        assert np.array_equal(P.perm.cpu().numpy(), want["perm"]) and P.vbase == want["vbase"].tolist()
        for k in ("f_rowptr", "f_col", "b_rowptr", "b_col"):
            assert np.array_equal(getattr(P, k).cpu().numpy(), want[k]), k
        assert np.array_equal(P.b_val.cpu().numpy().view(np.uint32), want["b_val"].view(np.uint32))


# ------------------------------------------------------------------------------------------------ 2. reference fixture
def fixture_trainer(G):
    relations = {r: (s, d) for r, (s, d, _) in enumerate(G["rels"])}
    tr = RGCNTrainer(16, 24, 5, 2, 0.5, G["num_nodes"], [0], len(relations), relations)
    tr.load_state_dict(G["state"])
    b = Data(edge_index=G["edge_index"], edge_attr=G["edge_type"], node_type=G["node_type"], local_node_idx=G["local_node_idx"])
    return tr, b.to("cuda"), {0: G["x_paper"].cuda()}


def test_eval_forward_and_gradients_match_the_reference_fixture(golden_rgcn):
    G = golden_rgcn
    tr, b, x = fixture_trainer(G)
    out = tr.forward(b, x, training=False)
    assert rel_err(out, G["out_forward"]) < 1e-5
    assert rel_err(tr.out_feat(), G["out_feat"]) < 1e-5
    grads = tr.gradients(b, x, G["w"].cuda())
    assert sorted(grads) == sorted(G["grads"])
    for k, v in G["grads"].items():
        assert rel_err(grads[k], v) < 5e-5, k
    sd = tr.state_dict()
    assert all(torch.equal(sd[k].cpu(), v) for k, v in G["state"].items())


# ------------------------------------------------------------------------------------------------ 3. full step vs fp64
def fp64_forward(params, x_dict, b, masks, p, L):
    """The reference's RGCN.forward (mag_pyg/gnn.py:26-137) in float64 with the engine's dropout masks injected."""
    nt, li = b.node_type.view(-1), b.local_node_idx.view(-1)
    n = nt.numel()
    h = torch.zeros(n, params["convs.0.root_lins.0.weight"].shape[1], dtype=torch.float64, device="cuda")
    for t in NODES:
        m = nt == t
        tab = x_dict[t].double() if t in x_dict else params[f"emb_dict.{t}"]
        h[m] = tab[li[m]]
    src, dst = b.edge_index
    et = b.edge_attr.view(-1)
    R = sum(1 for k in params if k.startswith("convs.0.rel_lins."))
    for i in range(L):
        W0 = params[f"convs.{i}.root_lins.0.weight"]
        out = torch.zeros(n, W0.shape[0], dtype=torch.float64, device="cuda")
        for r in range(R):
            m = et == r
            msg = h[src[m]] @ params[f"convs.{i}.rel_lins.{r}.weight"].t()
            agg = torch.zeros_like(out).index_add(0, dst[m], msg)
            cnt = torch.zeros(n, dtype=torch.float64, device="cuda").index_add(0, dst[m], torch.ones_like(dst[m], dtype=torch.float64))
            out = out + agg / cnt.clamp(min=1)[:, None]
        for t in NODES:
            m = (nt == t).nonzero().view(-1)
            out = out.index_add(0, m, h[m] @ params[f"convs.{i}.root_lins.{t}.weight"].t() + params[f"convs.{i}.root_lins.{t}.bias"])
        if i != L - 1:
            out = F.relu(out)
            if p > 0:
                out = out * masks[i] / (1 - p)
            feat = out
        h = out
    return h, feat


@pytest.mark.parametrize("mode", ["supervised", "kd"])
def test_three_steps_match_an_fp64_restatement(mode):
    data, x, rel = small_mag(1)
    p, L = 0.5, 2
    tr = trainer(rel, p=p, seed=3)
    params = {k: v.double().clone().requires_grad_(True) for k, v in tr.state_dict().items()}
    opt = torch.optim.Adam(list(params.values()), lr=0.01)
    teacher = trainer(rel, H=32, L=2, p=0.0, seed=11) if mode == "kd" else None
    for step, b in enumerate(batches(data, 3, seed=5)):
        tl = teacher.forward(b, x, training=False)[b.train_mask] if teacher else None
        loss = tr.train_step(b, x, teacher_logits=tl).clone()
        n = b.node_type.numel()
        masks = [ops.dropout_mask(n, 24, p, tr.seed, l + step * L).bool().double() for l in range(L - 1)]
        out, _ = fp64_forward(params, x, b, masks, p, L)
        o, lab = out[b.train_mask], b.y[b.train_mask].view(-1)
        if tl is None:
            ref = F.cross_entropy(o, lab)
        else:
            kd = F.kl_div(F.log_softmax(o / 4.0, 1), F.softmax(tl.double() / 4.0, 1))
            ref = kd * (0.9 * 16) + F.cross_entropy(o, lab) * 0.1
        opt.zero_grad()
        ref.backward()
        opt.step()
        assert abs(float(loss[0]) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref))), (step, float(loss[0]), float(ref))
    sd = tr.state_dict()
    for k, v in params.items():
        assert rel_err(sd[k], v) < 5e-5, k


# ------------------------------------------------------------------------------------------------ 4. module path
def test_loss_curve_matches_the_module_path_over_two_epochs():
    from test_rgcn_gpu import RelNet
    data, x, rel = small_mag(2)
    tr = trainer(rel, p=0.0, seed=7)
    net = RelNet(16, 24, 7, NODES, [0], len(rel)).cuda()
    net.load_state_dict({k: v for k, v in tr.state_dict().items()})
    opt = torch.optim.Adam(net.parameters(), lr=0.01)
    loader = sampling.GraphSAINTRandomWalkSampler(data, batch_size=150, walk_length=2, num_steps=4, seed=2)
    ours, theirs = [], []
    for epoch in range(2):
        for b in loader:
            ours.append(float(tr.train_step(b, x)[0]))
            out = net(x, b.edge_index, b.edge_attr, b.node_type, b.local_node_idx)[b.train_mask]
            loss = F.cross_entropy(out, b.y[b.train_mask].view(-1))
            opt.zero_grad()
            loss.backward()
            opt.step()
            theirs.append(float(loss))
    assert max(abs(a - b) for a, b in zip(ours, theirs)) < 1e-4, (ours, theirs)
    assert np.mean(ours[-4:]) < np.mean(ours[:4]), ours


# ------------------------------------------------------------------------------------------------ 5. embedding Adam
def test_embedding_adam_equals_typed_scatter_plus_adam():
    g = torch.Generator().manual_seed(0)
    sizes = {1: 3000, 2: 50}
    n, F_ = 4000, 128
    nt = torch.randint(0, 3, (n,), generator=g)
    li = torch.stack([torch.randint(0, sizes.get(int(t), 10), (1,), generator=g)[0] for t in nt])
    li[:200] = li[200:400]; nt[:200] = nt[200:400]               # duplicated (type, idx) pairs; most author rows untouched
    nt, li = nt.cuda(), li.cuda()
    order = device_argsort(nt, li, 3, 3000)
    tabs = {t: torch.randn(s, F_, generator=g).cuda() for t, s in sizes.items()}
    ref = {t: v.clone() for t, v in tabs.items()}
    m = {t: torch.zeros_like(v) for t, v in tabs.items()}; v_ = {t: torch.zeros_like(v) for t, v in tabs.items()}
    mr = {t: torch.zeros_like(v) for t, v in tabs.items()}; vr = {t: torch.zeros_like(v) for t, v in tabs.items()}
    head = torch.full((3000,), -1, dtype=torch.int32, device="cuda")
    step, step_r = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    for s in range(5):
        d = torch.randn(n, F_, generator=g).cuda()
        for t in tabs:
            ops.embedding_adam(d, nt, li, order, t, tabs[t], m[t], v_[t], head, step, 0.01)
        step += 1
        grads = {t: torch.zeros_like(x) for t, x in ref.items()}
        ops.typed_scatter(d, nt, li, order, grads, 3)
        for t in ref:
            st = step_r.clone()
            ops.adam_step(ref[t], grads[t], mr[t], vr[t], st, 0.01)
        step_r += 1
        for t in tabs:
            assert torch.equal(tabs[t], ref[t]) and torch.equal(m[t], mr[t]) and torch.equal(v_[t], vr[t]), (s, t)
        assert bool((head == -1).all())
    assert int(step) == 5


# ------------------------------------------------------------------------------------------------ 6. widened weight gradient
NEW_WGRAD = [(kin, nout) for kin in (64, 96, 384, 512, 1024, 1536, 2048) for nout in (32, 352, 512)] + [(128, 352), (256, 512)]


@pytest.mark.parametrize("Kin,Nout", NEW_WGRAD)
def test_widened_wgrad_bound_and_canaries(Kin, Nout):
    for nn_ in (33, 4099, 40_001):
        g = _gen(3 * nn_ + Kin + Nout)
        x = torch.randn(nn_, Kin, generator=g, device="cuda") * _pow2(Kin, g)[None, :]
        d = torch.randn(nn_, Nout, generator=g, device="cuda") * _pow2(Nout, g)[None, :]
        buf = torch.full((Kin * Nout + 64,), CANARY, dtype=torch.int32, device="cuda").view(torch.float32)
        out = buf[32:32 + Kin * Nout].view(Kin, Nout)
        ops.gemm_wgrad_tf32x3(x, d, out=out, wide=True)
        assert _gemm_check(x.t(), d.t(), out, _wgrad_beta(nn_)) <= 1.0, nn_
        bits = buf.view(torch.int32)
        assert bool((bits[:32] == CANARY).all()) and bool((bits[32 + Kin * Nout:] == CANARY).all())


@pytest.mark.parametrize("Kin,Nout", [(96, 32), (2048, 352), (1536, 512)])
def test_widened_wgrad_is_unbiased(Kin, Nout):
    g = _gen(Kin * Nout)
    x = torch.rand(20_000, Kin, generator=g, device="cuda") + 0.01
    d = torch.rand(20_000, Nout, generator=g, device="cuda") + 0.01
    m = _mean_signed_rel(ops.gemm_wgrad_tf32x3(x, d, wide=True), x.double().t() @ d.double())
    assert BIAS_LO <= m <= BIAS_HI, m


def test_wgrad_workspace_of_existing_shapes_unchanged_and_large_shapes_bounded():
    assert ops.wgrad_workspace_floats(256, 256) == 132 * 256 * 256
    assert ops.wgrad_workspace_floats(128, 40) == 132 * 128 * 64
    assert ops.wgrad_workspace_floats(2048, 512) <= 132 * 256 * 256
    assert lib.load().b200gnn_wgrad_workspace_floats(4096, 32) < 0


# ------------------------------------------------------------------------------------------------ ReLU/dropout backward
def test_relu_dropout_backward():
    g = torch.Generator(device="cuda").manual_seed(0)
    y = torch.randn(1000, 32, generator=g, device="cuda")
    out = ops.affine_relu_dropout(y, None, None, True, 0.5, 3, 1)
    d = torch.randn(1000, 32, generator=g, device="cuda")
    assert torch.equal(ops.relu_dropout_bwd(d, out, 0.5), torch.where(out > 0, d * 2.0, torch.zeros_like(d)))


def test_wgrad_shapes_outside_the_widened_range_are_reported():
    """The padded tilings are opt-in (wide=True); beyond Kin 2048, Nout 512 or off multiples of 4 the kernel refuses."""
    x, d = torch.randn(100, 64, device="cuda"), torch.randn(100, 40, device="cuda")
    with pytest.raises(lib.B200GnnError):
        ops.gemm_wgrad_tf32x3(x, d)
    want = x.double().t() @ d.double()
    assert rel_err(ops.gemm_wgrad_tf32x3(x, d, wide=True), want) < 1e-6
    for kin, nout in ((2052, 32), (128, 516), (130, 32)):
        with pytest.raises(lib.B200GnnError):
            ops.gemm_wgrad_tf32x3(torch.randn(100, kin, device="cuda"), torch.randn(100, nout, device="cuda"), wide=True)
