"""GATTrainer (the fused full-batch step of the reference's DGL GAT model) and the kernels added for it.

Graph: symmetric + self-loops, one hub above the hub threshold (split across CTAs), degree-1 rows (self-loop only).
References: tests/golden/gat_model_arxiv.pt (the reference's own class) and oracle/gat.py in fp64 with the engine's own keep
decisions injected (b200gnn_dropout_mask_u8 materialises the masks the bits / step kernels draw)."""
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops, sparse, synthetic
from efficient_gnns_b200.engine_gat import GATTrainer, padded_head
from efficient_gnns_b200.nn import _gat_aggregate
from oracle import gat as ogat, graph as og

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
sys.path.insert(0, str(GOLDEN))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).norm().item() / max(b.norm().item(), 1e-30)


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN / "gat_model_arxiv.pt")


def adj_of(row, col, n):
    return sparse.SparseTensor(row=row.cuda(), col=col.cuda(), sparse_sizes=(n, n), is_sorted=True)


@pytest.fixture(scope="module")
def graph(gold):
    n = gold["x"].shape[0]
    adj = adj_of(gold["row"], gold["col"], n)
    G = adj.storage.engine_csr_unweighted()
    assert G.n_hub >= 1 and int(adj.storage.rowcount().min()) == 1
    return adj, gold["row"], gold["col"], n


# ------------------------------------------------------------------------------------------------ the new kernels alone
@pytest.mark.parametrize("H,D,with_r", [(8, 32, True), (3, 256, True), (3, 12, False), (1, 40, True)])
def test_gat_scores_forward_and_backward_against_fp64(H, D, with_r):
    n, K = 3001, H * D
    g = torch.Generator().manual_seed(H * D)
    cat = torch.randn(n, 2 * K, generator=g).cuda()            # ft is the left half of [ft | res]: row pitch 2K
    ft = cat[:, :K]
    al = torch.randn(K, generator=g).cuda()
    ar = torch.randn(K, generator=g).cuda() if with_r else None
    sc = (torch.rand(n, generator=g) + 0.2).cuda()
    el = torch.full((n + 2, H), float("nan"), device="cuda")   # outputs among NaN canaries
    er = torch.full((n + 2, H), float("nan"), device="cuda")
    ops.gat_scores(ft, al, ar, sc, H, el=el[1:-1], er=er[1:-1] if with_r else None)
    assert torch.isnan(el[0]).all() and torch.isnan(el[-1]).all() and torch.isnan(er[0]).all() and torch.isnan(er[-1]).all()
    f64 = ft.double().view(n, H, D)
    u = 2.0 ** -24
    gam = (D + 6) * u                                          # gamma(D) of the dot product, + the scale and butterfly roundings
    ref_l = (f64 * al.double().view(H, D)).sum(-1) * sc.double().view(-1, 1)
    bnd_l = (f64.abs() * al.double().abs().view(H, D)).sum(-1) * sc.double().view(-1, 1) * gam
    assert ((el[1:-1].double() - ref_l).abs() <= bnd_l + 1e-30).all()
    if with_r:
        ref_r = (f64 * ar.double().view(H, D)).sum(-1)
        bnd_r = (f64.abs() * ar.double().abs().view(H, D)).sum(-1) * gam
        assert ((er[1:-1].double() - ref_r).abs() <= bnd_r + 1e-30).all()
    else:
        assert torch.isnan(er).all()

    d_el = torch.randn(n, H, generator=g).cuda()
    d_er = torch.randn(n, H, generator=g).cuda() if with_r else None
    dft0 = torch.randn(n, K, generator=g).cuda()
    outs = []
    for _ in range(2):
        dft = dft0.clone()
        dal = torch.full((K + 8,), float("nan"), device="cuda")
        dar = torch.full((K + 8,), float("nan"), device="cuda")
        ops.gat_scores_bwd(ft, al, ar, sc, d_el, d_er, H, dft, dal[4:-4], dar[4:-4] if with_r else None)
        outs.append((dft, dal, dar))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1][4:-4], outs[1][1][4:-4])    # repeatable
    dft, dal, dar = outs[0]
    assert torch.isnan(dal[:4]).all() and torch.isnan(dal[-4:]).all()
    gl = (d_el.double() * sc.double().view(-1, 1)).view(n, H, 1)
    ref = dft0.double().view(n, H, D) + gl * al.double().view(H, D)
    mag = dft0.double().abs().view(n, H, D) + gl.abs() * al.double().abs().view(H, D)
    if with_r:
        ref = ref + d_er.double().view(n, H, 1) * ar.double().view(H, D)
        mag = mag + d_er.double().abs().view(n, H, 1) * ar.double().abs().view(H, D)
    assert ((dft.double().view(n, H, D) - ref).abs() <= 4 * u * mag + 1e-30).all()
    # attention-vector gradients: chains of ceil(n / slots) rows per CTA, then `slots` partials
    slots = ops.gat_scores_slots(n)
    gam_n = (-(-n // slots) + slots + 4) * u
    ref_al = (gl * f64).sum(0).view(-1)
    assert ((dal[4:-4].double() - ref_al).abs() <= gam_n * (gl.abs() * f64.abs()).sum(0).view(-1) + 1e-30).all()
    if with_r:
        gr = d_er.double().view(n, H, 1)
        assert ((dar[4:-4].double() - (gr * f64).sum(0).view(-1)).abs() <= gam_n * (gr.abs() * f64.abs()).sum(0).view(-1) + 1e-30).all()


@pytest.mark.parametrize("H,D", [(8, 32), (3, 256), (3, 12), (1, 40)])
def test_gat_aggregate_epi_matches_gat_aggregate_and_the_unfused_composition(graph, H, D):
    adj, row, col, n = graph
    G = adj.storage.engine_csr_unweighted()
    K = H * D
    g = torch.Generator().manual_seed(K)
    cat = torch.randn(n, 2 * K, generator=g).cuda()
    ft, res = cat[:, :K], cat[:, K:]
    a = torch.rand(G.nnz, H, generator=g).cuda()
    base = torch.empty(n, K, device="cuda")
    _gat_aggregate(G, None, a, ft.contiguous(), base, H, D)
    out = torch.full((n, K), float("nan"), device="cuda")
    ops.gat_aggregate_epi(G, None, a, ft, out, H)
    assert torch.equal(out, base)                              # no epilogue operands: the existing kernel, bit for bit
    ss, rs_ = (torch.rand(n, generator=g) + 0.5).cuda(), (torch.rand(n, generator=g) + 0.5).cuda()
    bias = torch.randn(K, generator=g).cuda()
    stat = torch.full((ops.gat_stat_slots(G), 2, K), float("nan"), device="cuda")
    ops.gat_aggregate_epi(G, None, a, ft, out, H, src_scale=ss, row_scale=rs_, res=res, bias=bias, stat_partial=stat)
    a_s = a * ss[G.col.long()].view(-1, 1)
    _gat_aggregate(G, None, a_s, ft.contiguous(), base, H, D)
    assert torch.equal(out, (base * rs_.view(-1, 1) + res) + bias)       # same coefficient products, same order: exact
    assert torch.isfinite(stat).all()
    s64 = stat.double().sum(0)
    assert rel(s64[0], out.double().sum(0)) <= 1e-5 and rel(s64[1], out.double().pow(2).sum(0)) <= 1e-5
    # dyadic data: every sum is exact, so the slots reproduce the column sums exactly
    ft_d = (torch.randint(-8, 9, (n, K), generator=g).float() / 8).cuda()
    a_d = (torch.randint(0, 5, (G.nnz, H), generator=g).float() / 4).cuda()
    ops.gat_aggregate_epi(G, None, a_d, ft_d, out, H, stat_partial=stat)
    ref = torch.zeros(n, H, D, dtype=torch.float64).index_add_(0, row, ft_d.cpu().double().view(n, H, D)[col] * a_d.cpu().double().unsqueeze(-1))
    assert torch.equal(out.double().cpu(), ref.view(n, K))
    assert torch.equal(stat.double().sum(0).cpu()[0], ref.view(n, K).sum(0))
    assert rel(stat.double().sum(0)[1], ref.view(n, K).pow(2).sum(0)) <= 1e-6      # the hub row's square is not dyadic-exact


# ------------------------------------------------------------------------------------------------ fixture
@pytest.mark.parametrize("case", ["attn_dst", "no_attn_dst"])
def test_fixture_forward_backward_and_state_round_trip(gold, graph, case):
    adj, row, col, n = graph
    c = gold["cases"][case]
    tr = GATTrainer(adj, gold["x"].shape[1], gold["n_classes"], gold["n_hidden"], gold["n_layers"], gold["n_heads"],
                    use_attn_dst=case == "attn_dst", use_symmetric_norm=True, lr=1e-3)
    assert tr.Dp[0] > tr.Dl[0]                                   # the head width is stored padded
    tr.load_state_dict(c["state"])
    sd = tr.state_dict()
    assert set(sd) == set(c["state"])
    for k, v in c["state"].items():
        assert torch.equal(sd[k].cpu(), v), k
    x, y, idx = gold["x"].cuda(), gold["y"].cuda(), gold["train_idx"].cuda()
    logits_e = tr.forward(x, training=False)
    assert rel(logits_e, c["logits_eval"]) <= 1e-5 and rel(tr.out_feat(), c["feat_eval"]) <= 1e-5
    loss = tr.train_step(x, y, idx)
    assert rel(tr.Y[-1][:, :tr.n_classes], c["logits_train"]) <= 1e-5 and rel(tr.out_feat(), c["feat_train"]) <= 1e-5
    assert abs(loss[0].item() - c["loss"].item()) <= 1e-5 * abs(c["loss"].item())
    grads = tr.named_gradients()
    assert set(grads) == set(c["grads"])
    for k, g in c["grads"].items():
        assert fro(grads[k], g) <= 1e-4 and rel(grads[k], g) <= 5e-4, k
    for k, v in c["state_after"].items():                        # BatchNorm running statistics after one training forward
        assert rel(tr.state_dict()[k], v) <= 1e-5, k


# ------------------------------------------------------------------------------------------------ whole step vs fp64 oracle
def engine_masks(tr, step):
    n, nnz = tr.N, tr.nnz
    hid = [ops.dropout_mask(n, tr.K[0], tr.p, tr.seed, tr.stream_offset("dropout", l, step))[:, tr._cols(l)].cpu().bool()
           for l in range(tr.L - 1)] if tr.p > 0 else None
    inp = ops.dropout_mask(n, tr.in_feats, tr.p_in, tr.seed, tr.stream_offset("input", 0, step)).cpu().bool() if tr.p_in > 0 else None
    edge = [ops.dropout_mask((nnz + 3) // 4, 4, tr.p_edge, tr.seed, tr.stream_offset("edge", l, step)).view(-1)[:nnz].cpu().bool()
            for l in range(tr.L)] if tr.p_edge > 0 else None
    return inp, hid, edge


def oracle_step(tr, state, x, y, idx, teacher, row, col, masks, aux=None, beta=1.0):
    inp, hid, edge = masks
    st = {k: v.detach().cpu().double().requires_grad_("running" not in k) for k, v in state.items()}
    logits, feat = ogat.gat_forward(x.double(), row, col, st, tr.L, tr.H, tr.sym, True, tr.p, tr.p_in, inp, hid, edge)
    z = logits[idx]
    ce = torch.nn.functional.cross_entropy(z, y[idx])
    if teacher is None:
        loss = ce
    else:                                                        # kd_criterion, arxiv_pyg/criterion.py:8-21
        T, a = tr.kd_T, tr.alpha
        kd = torch.nn.functional.kl_div(torch.log_softmax(z / T, 1), torch.softmax(teacher[idx].double() / T, 1),
                                        reduction="mean")            # the reference's default reduction
        loss = (1 - a) * ce + a * T * T * kd
    if aux is not None:
        loss = loss + beta * aux(feat)
    loss.backward()
    return logits.detach(), feat.detach(), loss.detach(), {k: v.grad for k, v in st.items() if v.requires_grad}, st


@pytest.mark.parametrize("H,D,attn_dst,kd,p_edge", [(8, 32, True, False, 0.0), (8, 32, False, True, 0.3), (3, 250, True, True, 0.3),
                                                    (3, 250, False, False, 0.0)])
def test_training_step_matches_fp64_oracle_with_engine_masks(gold, graph, H, D, attn_dst, kd, p_edge):
    adj, row, col, n = graph
    g = torch.Generator().manual_seed(H)
    x = torch.randn(n, 32, generator=g)
    y, idx = gold["y"], gold["train_idx"]
    teacher = torch.randn(n, 8, generator=g) * 2 if kd else None
    tr = GATTrainer(adj, 32, 8, D, 3, H, dropout=0.75, input_drop=0.1, edge_drop=p_edge, use_attn_dst=attn_dst,
                    use_symmetric_norm=True, lr=1e-3, seed=3)
    assert tr.Dp[0] == padded_head(H, D)
    state = tr.state_dict()
    masks = engine_masks(tr, 0)
    if p_edge > 0:                                               # a destination whose every edge is dropped exists
        deg_kept = torch.zeros(n, dtype=torch.long).index_add_(0, row, masks[2][0].long())
        assert (deg_kept == 0).any()
    loss = tr.train_step(x.cuda(), y.cuda(), idx.cuda(), None if teacher is None else teacher.cuda())
    logits, feat, loss_ref, grads_ref, _ = oracle_step(tr, state, x, y, idx, teacher, row, col, masks)
    assert torch.isfinite(tr.Y[-1]).all()
    assert rel(tr.Y[-1][:, :8], logits) <= 2e-5 and rel(tr.out_feat(), feat) <= 2e-5
    assert abs(loss[0].item() - loss_ref.item()) <= 1e-5 * abs(loss_ref.item())
    grads = tr.named_gradients()
    for k, gr in grads_ref.items():
        assert fro(grads[k], gr) <= 2e-4, k


def test_aux_criterion_seeds_the_backward(gold, graph):
    adj, row, col, n = graph
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, 32, generator=g)
    y, idx = gold["y"], gold["train_idx"]
    t_feat = torch.randn(n, 3 * 10, generator=g)
    tr = GATTrainer(adj, 32, 8, 10, 3, 3, dropout=0.5, use_symmetric_norm=True, lr=1e-3, seed=1)
    state, masks = tr.state_dict(), engine_masks(tr, 0)

    def aux_of(t):
        return lambda f: (torch.nn.functional.normalize(f[idx.to(f.device)], dim=1) - t[idx.to(t.device)]).pow(2).mean()
    loss = tr.train_step(x.cuda(), y.cuda(), idx.cuda(), aux=aux_of(t_feat.cuda()), beta=0.5)
    _, _, loss_ref, grads_ref, _ = oracle_step(tr, state, x, y, idx, None, row, col, masks, aux=aux_of(t_feat.double()), beta=0.5)
    assert abs(loss[0].item() - loss_ref.item()) <= 1e-5 * abs(loss_ref.item())
    for k, gr in grads_ref.items():
        assert fro(tr.named_gradients()[k], gr) <= 2e-4, k


def test_adam_three_steps_padding_stays_zero_and_eval_draws_nothing(gold, graph):
    adj, row, col, n = graph
    g = torch.Generator().manual_seed(2)
    x = torch.randn(n, 32, generator=g)
    y, idx = gold["y"], gold["train_idx"]
    tr = GATTrainer(adj, 32, 8, 10, 3, 3, dropout=0.5, input_drop=0.1, edge_drop=0.1, use_symmetric_norm=True, lr=1e-2, seed=4)
    st = {k: v.detach().cpu().double().requires_grad_("running" not in k) for k, v in tr.state_dict().items()}
    opt = torch.optim.Adam([v for v in st.values() if v.requires_grad], lr=1e-2)
    for step in range(3):
        inp, hid, edge = engine_masks(tr, step)
        tr.train_step(x.cuda(), y.cuda(), idx.cuda())
        opt.zero_grad()
        logits, _ = ogat.gat_forward(x.double(), row, col, st, 3, 3, True, True, 0.5, 0.1, inp, hid, edge)
        torch.nn.functional.cross_entropy(logits[idx], y[idx]).backward()
        opt.step()
    sd = tr.state_dict()
    for k, v in st.items():
        if v.requires_grad:                                      # an Adam step moves an entry by at most lr
            assert (sd[k].double().cpu() - v.detach()).abs().max().item() <= 0.05 * 1e-2, k
    # padded columns: exactly zero in activations, parameters, gradients and moments
    pad = torch.ones(tr.K[0], dtype=torch.bool, device="cuda")
    pad[tr._cols(0)] = False
    assert pad.any()
    for l in range(tr.L - 1):
        assert (tr.Y[l][:, pad] == 0).all() and (tr.cat[l][:, :tr.K[l]][:, pad] == 0).all() and (tr.dY[l][:, pad] == 0).all()
        assert (tr._hidden(l)[:, pad] == 0).all()
        assert (tr.attn_l[l][pad] == 0).all() and (tr.beta[l][pad] == 0).all() and (tr.gbeta[l][pad] == 0).all()
        for W in (tr.Wfc[l], tr.Wres[l], tr.gWfc[l], tr.gWres[l]):
            assert (torch.cat(W, dim=1)[:, pad] == 0).all()
        for blk in tr.Wfc[l + 1] + tr.Wres[l + 1] + tr.gWfc[l + 1] + tr.gWres[l + 1]:
            assert (blk[pad] == 0).all()
    dead = (tr.params == 0) & (tr.grads == 0)                    # the padding (and nothing else moves without a gradient)
    assert dead.any() and (tr.exp_avg[dead] == 0).all() and (tr.exp_avg_sq[dead] == 0).all()
    # eval: running statistics, no draws, no parameter change
    bits, count, params = tr.keep_bits.clone(), tr.step_count.clone(), tr.params.clone()
    logits_e = tr.forward(x.cuda(), training=False)
    state_e = {k: v.cpu().double() for k, v in tr.state_dict().items()}
    ref_e, feat_e = ogat.gat_forward(x.double(), row, col, state_e, 3, 3, True, training=False)
    assert rel(logits_e, ref_e) <= 2e-5 and rel(tr.out_feat(), feat_e) <= 2e-5
    assert torch.equal(bits, tr.keep_bits) and torch.equal(count, tr.step_count) and torch.equal(params, tr.params)


@pytest.mark.parametrize("H,D", [(8, 32), (3, 250)])
def test_graph_replay_is_bit_identical_to_eager_and_runs_repeat(gold, graph, H, D):
    adj, row, col, n = graph
    g = torch.Generator().manual_seed(5)
    x, t = torch.randn(n, 32, generator=g).cuda(), torch.randn(n, 8, generator=g).cuda()
    y, idx = gold["y"].cuda(), gold["train_idx"].cuda()

    def make():
        return GATTrainer(adj, 32, 8, D, 3, H, dropout=0.75, input_drop=0.1, edge_drop=0.1, use_symmetric_norm=True, lr=1e-2, seed=9)
    eager, again, graphed = make(), make(), make()
    losses = []
    for _ in range(5):
        losses.append(eager.train_step(x, y, idx, t).clone())
        again.train_step(x, y, idx, t)
    assert torch.equal(eager.params, again.params) and torch.equal(eager.exp_avg_sq, again.exp_avg_sq)
    graphed.capture(x, y, idx, t, warmup=2)                      # two warm-up steps run; the capture itself runs nothing
    for _ in range(3):
        loss = graphed.replay()
    torch.cuda.synchronize()
    assert torch.equal(graphed.params, eager.params) and torch.equal(loss, losses[-1])
    assert torch.equal(graphed.running_var[0], eager.running_var[0])
    assert graphed.launches_per_step() > 0


# ------------------------------------------------------------------------------------------------ full size
def test_full_size_teacher_shape_trains():
    """ARXIV-shape synthetic graph (N = 169,343), the teacher's 3 heads of 250 stored as 3 x 256: finite, decreasing loss."""
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    r, c, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(r, c, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    adj = adj_of(torch.from_numpy(rs), torch.from_numpy(cs), n)
    tr = GATTrainer(adj, ds.x.shape[1], 40, 250, 3, 3, dropout=0.75, input_drop=0.1, edge_drop=0.1, use_attn_dst=False,
                    use_symmetric_norm=True, lr=2e-3, seed=0)
    x, y, idx = ds.x.cuda(), ds.y.squeeze(1).cuda(), ds.split_idx["train"].cuda()
    losses = [tr.train_step(x, y, idx)[0].item() for _ in range(5)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert lib.launch_count() > 0
