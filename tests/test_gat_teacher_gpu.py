"""GATTeacherTrainer (the arxiv GAT teacher's recipe on the fused GAT step) and the kernels added for it.

Kernels against fp64 or exact answers; the engine against tests/golden/gat_teacher_arxiv.pt (the reference's own gat.py)
and against oracle/gat_teacher.py in fp64 with the engine's own draws injected; CUDA-graph replay; padding; artefacts."""
import math
import sys
from pathlib import Path

import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import ops, sparse, synthetic
from efficient_gnns_b200.engine_gat_teacher import GATTeacherTrainer, HISTORY_COLUMNS
from oracle import gat_teacher as ot, graph as og

pytestmark = pytest.mark.gpu
GOLDEN = Path(__file__).resolve().parent / "golden"
sys.path.insert(0, str(GOLDEN))
U = 2.0 ** -24
EPS = 1 - math.log(2)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def fro(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).norm().item() / max(b.norm().item(), 1e-30)


@pytest.fixture(scope="module")
def gold():
    g = torch.load(GOLDEN / "gat_teacher_arxiv.pt", weights_only=False)
    g["row"], g["col"] = g["row"].long(), g["col"].long()                # stored as int32
    return g


def adj_of(row, col, n):
    return sparse.SparseTensor(row=row.cuda(), col=col.cuda(), sparse_sizes=(n, n), is_sorted=True)


def splits_of(gold):
    return {"train": gold["train_idx"], "valid": gold["val_idx"], "test": gold["test_idx"]}


def make(gold, use_labels=True, iters=1, **kw):
    n = gold["x"].shape[0]
    kw = {**dict(n_hidden=gold["n_hidden"], n_layers=gold["n_layers"], n_heads=gold["n_heads"], dropout=0.0, input_drop=0.0,
                 edge_drop=0.0), **kw}
    return GATTeacherTrainer(adj_of(gold["row"], gold["col"], n), gold["x"].cuda(), gold["y"].cuda(), splits_of(gold),
                             n_classes=gold["n_classes"], use_labels=use_labels, n_label_iters=iters, **kw)


# ------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("use_labels", [True, False])
def test_label_inputs_roles_block_and_mask_match_dropout_mask(use_labels):
    n, F, C, seed, p = 1003, 12, 7, 5, 0.5
    g = torch.Generator().manual_seed(1)
    perm = torch.randperm(n, generator=g)
    tr, ev = perm[:401], perm[401:900]                       # the last 103 rows are in no split
    labels = torch.randint(0, C, (n,), generator=g)
    row_pos = torch.full((n,), -2, dtype=torch.int32)
    row_pos[ev] = -1
    row_pos[tr] = torch.arange(tr.numel(), dtype=torch.int32)
    W = F + C + 1
    X = torch.full((n, W), float("nan"), device="cuda")
    X[:, :F] = 3.0
    role = torch.full((n,), 77, dtype=torch.uint8, device="cuda")
    cnt = torch.full((ops.teacher_slots(n),), -1, dtype=torch.int32, device="cuda")
    for step, ev_mode in ((0, False), (3, False), (0, True)):
        step_dev = torch.tensor([step], dtype=torch.int32, device="cuda")
        ops.label_inputs(X, F, C, row_pos.cuda(), labels.cuda(), role, cnt, eval=ev_mode, use_labels=use_labels,
                         mask_rate=p, seed=seed, offset=9, step_dev=step_dev, step_mul=13)
        nt = tr.numel()
        drop = ops.dropout_mask((nt + 3) // 4, 4, p, seed, 9 + 13 * step).view(-1)[:nt].cpu() == 0
        want = torch.zeros(n, dtype=torch.uint8)
        want[ev] = ops.ROLE_EVAL
        if ev_mode:
            want[tr] = ops.ROLE_INPUT
        else:
            label_rows = drop if use_labels else ~drop
            want[tr] = torch.where(label_rows, ops.ROLE_INPUT, ops.ROLE_PRED).to(torch.uint8)
        assert torch.equal(role.cpu(), want)
        assert int(cnt.sum()) == int((want == ops.ROLE_PRED).sum())
        blk = X[:, F:F + C].cpu()
        if use_labels:
            ref = torch.zeros(n, C)
            r = want == ops.ROLE_INPUT
            ref[r.nonzero().view(-1), labels[r]] = 1.0
            assert torch.equal(blk, ref)
        else:
            assert torch.isnan(blk).all()
        assert (X[:, :F] == 3.0).all() and torch.isnan(X[:, -1]).all()      # neighbours untouched


def test_label_softmax_among_canaries():
    n, C = 2001, 40
    g = torch.Generator().manual_seed(2)
    logits = (torch.randn(n, 48, generator=g) * 4).cuda()
    role = torch.randint(0, 4, (n,), generator=g, dtype=torch.uint8).cuda()
    out = torch.full((n, 50), float("nan"), device="cuda")
    ops.label_softmax(logits, C, out[:, 5:5 + C], role, (1 << 2) | (1 << 3))
    sel = (role == 2) | (role == 3)
    ref = torch.softmax(logits[:, :C].double(), 1)
    got = out[:, 5:5 + C]
    assert ((got[sel].double() - ref[sel]).abs() <= (C + 16) * U * ref[sel] + 1e-37).all()
    assert torch.isnan(got[~sel]).all() and torch.isnan(out[:, :5]).all() and torch.isnan(out[:, 5 + C:]).all()
    full = ops.label_softmax(logits, C, torch.empty(n, C, device="cuda"))
    assert ((full.double() - ref).abs() <= (C + 16) * U * ref + 1e-37).all()


def logce_ref(z, y, rows, n):
    z = z.double()
    ce = torch.logsumexp(z, 1) - z.gather(1, y.view(-1, 1)).view(-1)
    loss = (torch.log(EPS + ce[rows]) - math.log(EPS)).sum() / n if n else torch.tensor(float("nan"), dtype=torch.float64)
    sm = torch.softmax(z, 1)
    oh = torch.nn.functional.one_hot(y, z.shape[1]).double()
    w = torch.zeros(z.shape[0], dtype=torch.float64)
    if n:
        w[rows] = 1.0 / ((EPS + ce[rows]) * n)
    return loss, (sm - oh) * w.view(-1, 1), ce, sm, oh, w


@pytest.mark.parametrize("n_pred", [0, 1, 700])
def test_logce_forward_backward_and_accuracy(n_pred):
    n, C = 1500, 40
    g = torch.Generator().manual_seed(3 + n_pred)
    z = torch.randint(-3, 4, (n, C), generator=g).float() + 0.0        # integers: many ties for the argmax
    z[::3] = torch.randn(z[::3].shape, generator=g) * 3
    y = torch.randint(0, C, (n,), generator=g)
    tr = torch.randperm(n, generator=g)[:1000]
    role = torch.full((n,), ops.ROLE_EVAL, dtype=torch.uint8)
    role[tr] = ops.ROLE_INPUT
    role[tr[:n_pred]] = ops.ROLE_PRED
    slots = ops.teacher_slots(n)
    cnt = torch.zeros(slots, dtype=torch.int32)
    cnt[slots // 2] = n_pred                                           # any split over the slots
    zc = torch.full((n, 44), float("nan"), device="cuda")
    zc[:, :C] = z.cuda()
    dl = torch.zeros(n, 44, device="cuda")
    dl[:, C:] = float("nan")
    outs = torch.full((4,), float("nan"), device="cuda")
    part = torch.empty(6 * ops.teacher_slots(tr.numel()), dtype=torch.float64, device="cuda")
    ops.logce_fwd_bwd(zc, C, tr.cuda(), y.cuda(), role.cuda(), cnt.cuda(), dl, outs[1:2], outs[2:3], part)
    rows = tr[:n_pred]
    loss, grad, ce, sm, oh, w = logce_ref(z, y, rows, n_pred)
    assert torch.isnan(outs[0]) and torch.isnan(outs[3]) and torch.isnan(dl[:, C:]).all()
    if n_pred == 0:
        assert torch.isnan(outs[1]) and (dl[:, :C] == 0).all()
    else:
        assert abs(outs[1].item() - loss.item()) <= 1e-5 * abs(loss.item())
        err_ce = (C + 8) * U * (z.double().abs().max(1).values + torch.logsumexp(z.double(), 1) + z.double().abs().max(1).values)
        bound = ((C + 16) * U + err_ce.view(-1, 1) / (EPS + ce.view(-1, 1))) * (sm + oh) * w.view(-1, 1) + 1e-37
        assert ((dl[:, :C].cpu().double() - grad).abs() <= bound).all()
    hits = (torch.argmax(z[tr], 1) == y[tr]).sum().item()
    assert outs[2].item() == np.float32(hits / tr.numel())


def test_split_eval_losses_and_first_max_accuracy():
    n, C = 3000, 40
    g = torch.Generator().manual_seed(4)
    z = torch.randint(-2, 3, (n, C), generator=g).float()
    z[1::2] = torch.randn(z[1::2].shape, generator=g)
    y = torch.randint(0, C, (n,), generator=g)
    perm = torch.randperm(n, generator=g)
    idx = [perm[:1200], perm[1200:1700], perm[1700:2900]]
    loss_out = torch.full((5,), float("nan"), device="cuda")
    acc_out = torch.full((5,), float("nan"), device="cuda")
    part = torch.empty(6 * ops.teacher_slots(2900), dtype=torch.float64, device="cuda")
    ops.split_eval(z.cuda(), C, torch.cat(idx).cuda(), [i.numel() for i in idx], y.cuda(), loss_out[1:4], acc_out[1:4], part)
    assert torch.isnan(loss_out[0]) and torch.isnan(loss_out[4]) and torch.isnan(acc_out[0]) and torch.isnan(acc_out[4])
    for s, i in enumerate(idx):
        lo, *_ = logce_ref(z, y, i, i.numel())
        assert abs(loss_out[1 + s].item() - lo.item()) <= 1e-5 * abs(lo.item())
        assert acc_out[1 + s].item() == np.float32((torch.argmax(z[i], 1) == y[i]).sum().item() / i.numel())


@pytest.mark.parametrize("wd", [0.0, 5e-4])
def test_rmsprop_against_fp64_and_torch(wd):
    n = 4099
    g = torch.Generator().manual_seed(5)
    p0 = torch.randn(n, generator=g)
    p0[-7:] = 0.0                                                     # padding: zero parameter and gradient
    sq0 = torch.rand(n, generator=g) * 1e-3
    sq0[-7:] = 0.0
    lr = 0.002
    for step in (0, 1, 49, 50, 120):
        gr = torch.randn(n, generator=g) * 1e-2
        gr[-7:] = 0.0
        p, sq = p0.cuda(), sq0.cuda()
        cnt = torch.tensor([step], dtype=torch.int32, device="cuda")
        ops.rmsprop_step(p, gr.cuda(), sq, cnt, lr, 50, 0.99, 1e-8, wd)
        assert cnt.item() == step + 1
        lr_t = lr * min(step + 1, 50) / 50                            # adjust_learning_rate at epoch step + 1
        tp = torch.nn.Parameter(p0.clone())
        opt = torch.optim.RMSprop([tp], lr=lr_t, weight_decay=wd, foreach=False)
        opt.state[tp] = {"step": torch.tensor(float(step)), "square_avg": sq0.clone()}
        tp.grad = gr.clone()
        opt.step()
        p64, sq64 = p0.double().clone(), sq0.double().clone()
        ot.rmsprop_step([p64], [gr.double()], [sq64], lr_t, weight_decay=wd)
        ge = gr.double() + wd * p0.double()
        upd = lr_t * ge.abs() / (sq64.sqrt() + 1e-8)
        assert ((p.cpu().double() - p64).abs() <= 8 * U * (upd + p64.abs()) + 1e-45).all()
        assert ((sq.cpu().double() - sq64).abs() <= 4 * U * sq64 + 1e-45).all()
        assert ((p.cpu() - tp.detach()).abs().double() <= 8 * U * (upd + p64.abs()) + 1e-45).all()
        assert (p[-7:] == 0).all() and (sq[-7:] == 0).all()
    # the warm-up rate, exactly: p = 0, g = 1, square_avg = 0 -> p = -lr_t / (sqrt(fl(0.01)) + eps), in fp32
    for step in (0, 49, 50):
        p, sq = torch.zeros(4, device="cuda"), torch.zeros(4, device="cuda")
        ops.rmsprop_step(p, torch.ones(4, device="cuda"), sq, torch.tensor([step], dtype=torch.int32, device="cuda"), lr, 50)
        f = np.float32
        lr_t = f(lr * min(step + 1, 50) / 50)
        s = f(f(0.0) * f(0.99)) + f(f(f(1.0 - 0.99) * f(1.0)) * f(1.0))
        want = f(0.0) + f(f(-lr_t) * f(1.0)) / f(np.sqrt(s) + f(1e-8))
        assert (p.cpu().numpy() == want).all(), (step, p[0].item(), want)


def test_snapshot_on_strict_improvement_only_never_nan():
    src = torch.arange(16, dtype=torch.float32, device="cuda")
    dst = torch.full((24,), float("nan"), device="cuda")
    best = torch.tensor([float("inf")], device="cuda")
    cand = torch.tensor([3.0], device="cuda")
    ops.snapshot_if_better(cand, best, [(src, dst[4:20])])
    assert torch.equal(dst[4:20], src) and best.item() == 3.0 and torch.isnan(dst[:4]).all() and torch.isnan(dst[20:]).all()
    for c, moves in ((3.0, False), (float("nan"), False), (5.0, False), (2.5, True)):
        src += 1
        cand.fill_(c)
        ops.snapshot_if_better(cand, best, [(src, dst[4:20])])
        assert torch.equal(dst[4:20], src) == moves
        assert best.item() == (2.5 if moves else 3.0)


# ------------------------------------------------------------------------------------------------ engine vs fixture
@pytest.mark.parametrize("case", ["labels", "no_labels"])
def test_engine_reproduces_the_reference_script(gold, case):
    c = gold["cases"][case]
    tr = make(gold, case == "labels", 1 if case == "labels" else 0)
    assert list(tr.named_parameters()) == c["names"]
    tr.load_state_dict(c["state0"])
    for ep in c["epochs"]:
        acc, loss = tr.train_step(mask=ep["mask"])
        assert abs(loss.item() - ep["loss"]) <= 1e-4 * abs(ep["loss"]) and abs(acc.item() - ep["acc"]) <= 1.5 / 350
        accs, losses = tr.evaluate()
        for v, k in zip(accs.tolist(), ("train_acc", "val_acc", "test_acc")):
            assert abs(v - ep[k]) <= 2.5 / 170, k                     # one row of the smallest split
        for v, k in zip(losses.tolist(), ("train_loss", "val_loss", "test_loss")):
            assert abs(v - ep[k]) <= 1e-4 * abs(ep[k]), k
        if ep["pred"] is not None:                                       # kept for the last epoch
            assert fro(tr.Y[-1][:, :tr.n_classes], ep["pred"]) <= 1e-4 and fro(tr.out_feat(), ep["feat"]) <= 1e-4
        for k, v in tr.named_parameters().items():
            assert fro(v, ep["params"][k]) <= 1e-3, k
        sd = tr.model_state_dict()
        for k, v in ep["running"].items():
            if "running" in k:
                assert rel(sd[k], v) <= 1e-4, k
            else:
                assert torch.equal(sd[k], v), k


# ------------------------------------------------------------------------------------------------ engine vs fp64 oracle
def engine_draws(tr, step):
    n, nnz, out = tr.N, tr.nnz, []
    for f in range(tr.n_fwd):
        hid = [ops.dropout_mask(n, tr.K[0], tr.p, tr.seed, tr.stream_offset("dropout", l, step, f))[:, tr._cols(l)].cpu().bool()
               for l in range(tr.L - 1)]
        inp = ops.dropout_mask(n, tr.in_feats, tr.p_in, tr.seed, tr.stream_offset("input", 0, step, f)).cpu().bool()
        edge = [ops.dropout_mask((nnz + 3) // 4, 4, tr.p_edge, tr.seed, tr.stream_offset("edge", l, step, f)).view(-1)[:nnz].cpu().bool()
                for l in range(tr.L)]
        out.append((inp, hid, edge))
    nt = tr.sizes[0]
    mask = ops.dropout_mask((nt + 3) // 4, 4, tr.mask_rate, tr.seed, tr.mask_offset(step)).view(-1)[:nt].cpu() == 0
    return out, mask


@pytest.mark.parametrize("use_labels", [True, False])
def test_engine_steps_match_fp64_oracle_with_engine_draws(gold, use_labels):
    iters = 1 if use_labels else 0
    tr = make(gold, use_labels, iters, dropout=0.5, input_drop=0.25, edge_drop=0.3, seed=7)
    x, y = gold["x"].double(), gold["y"]
    row, col = gold["row"], gold["col"]
    ti, vi, te = gold["train_idx"], gold["val_idx"], gold["test_idx"]
    names = list(tr.named_parameters())
    for step in range(3):
        draws, mask = engine_draws(tr, step)
        st = {k: v.cpu().double().requires_grad_(k in names) for k, v in tr.state_dict().items()}
        params_before = {k: v.detach().clone() for k, v in tr.named_parameters().items()}
        sq_before = {k: v.double().cpu() for k, v in tr.named_square_avg().items()}
        acc, loss = tr.train_step()
        acc_r, loss_r, pred_r, _ = ot.train(x, y, row, col, ti, vi, te, st, tr.L, tr.H, tr.n_classes, use_labels, iters, mask,
                                            draws, tr.p, tr.p_in)
        assert abs(loss.item() - loss_r.item()) <= 1e-5 * abs(loss_r.item())
        assert abs(acc.item() - acc_r.item()) <= 1.5 / ti.numel()
        assert fro(tr.Y[-1][:, :tr.n_classes], pred_r) <= 2e-5
        grads = tr.named_gradients()
        for k in names:
            assert fro(grads[k], st[k].grad) <= 2e-4, k
        sd = tr.state_dict()
        for k in sd:
            if "running" in k:
                assert rel(sd[k], st[k]) <= 1e-5, k
        # the RMSprop update from the engine's own gradients, in fp64 (the rate of epoch step + 1)
        lr_t = ot.lr_at(tr.lr, step + 1)
        p64 = [params_before[k].cpu().double().clone() for k in names]
        sq64 = [sq_before[k].clone() for k in names]
        g64 = [grads[k].cpu().double() for k in names]
        ot.rmsprop_step(p64, g64, sq64, lr_t)
        after = tr.named_parameters()
        for k, p, s, gg in zip(names, p64, sq64, g64):
            upd = lr_t * gg.abs() / (s.sqrt() + 1e-8)
            assert ((after[k].cpu().double() - p).abs() <= 8 * U * (upd + p.abs()) + 1e-30).all(), k
    accs, losses = tr.evaluate()
    st = {k: v.cpu().double() for k, v in tr.state_dict().items()}
    accs_r, losses_r, pred_r, feat_r = ot.evaluate(x, y, row, col, ti, vi, te, st, tr.L, tr.H, tr.n_classes, use_labels, iters)
    assert rel(tr.Y[-1][:, :tr.n_classes], pred_r) <= 2e-5 and rel(tr.out_feat(), feat_r) <= 2e-5
    for a, b in zip(losses.tolist(), losses_r):
        assert abs(a - b.item()) <= 1e-5 * abs(b.item())


# ------------------------------------------------------------------------------------------------ graph, padding, artefacts
def test_epoch_graph_replay_is_bit_identical_and_capture_does_not_train(gold):
    kw = dict(dropout=0.75, input_drop=0.25, edge_drop=0.3, seed=3)
    eager, graphed = make(gold, **kw), make(gold, **kw)
    assert graphed.Dp[0] > graphed.Dl[0]
    rows = [eager.epoch().clone() for _ in range(4)]
    p0, c0 = graphed.params.clone(), graphed.step_count.clone()
    graphed.capture()
    torch.cuda.synchronize()
    assert torch.equal(graphed.params, p0) and torch.equal(graphed.step_count, c0) and torch.isinf(graphed.best).all()
    hist = graphed.run(4, log_every=0)
    assert hist.shape == (4, len(HISTORY_COLUMNS)) and torch.isfinite(hist).all()
    assert torch.equal(hist, torch.stack(rows).cpu())
    assert torch.equal(graphed.params, eager.params) and torch.equal(graphed.square_avg, eager.square_avg)
    assert torch.equal(graphed.running_var[0], eager.running_var[0]) and torch.equal(graphed.best, eager.best)
    assert torch.equal(graphed.final_pred(), eager.final_pred()) and torch.equal(graphed.final_feat(), eager.final_feat())
    # the snapshot holds the epoch of the lowest validation loss
    best_epoch = int(torch.argmin(hist[:, 6]))
    assert graphed.best.item() == hist[best_epoch, 6].item()
    # padding: parameters, gradients and square_avg stay exactly zero
    dead = (graphed.params == 0) & (graphed.grads == 0)
    pad = torch.ones(graphed.K[0], dtype=torch.bool, device="cuda")
    pad[graphed._cols(0)] = False
    for l in range(graphed.L - 1):
        assert (graphed.beta[l][pad] == 0).all() and (graphed.attn_l[l][pad] == 0).all()
        for W in (graphed.Wfc[l], graphed.Wres[l]):
            assert (torch.cat(W, dim=1)[:, pad] == 0).all()
    assert dead.sum() >= pad.sum() and (graphed.square_avg[dead] == 0).all()


def test_preset_parameter_count():
    n = 64
    r = torch.arange(n)
    adj = adj_of(r, r, n)
    g = torch.Generator().manual_seed(0)
    split = {"train": torch.arange(20), "valid": torch.arange(20, 40), "test": torch.arange(40, 64)}
    tr = GATTeacherTrainer(adj, torch.randn(n, 128, generator=g).cuda(), torch.arange(n) % 40, split)
    assert tr.in_feats == 168 and tr.n_parameters() == 1441580
    assert sum(v.numel() for k, v in tr.model_state_dict().items() if "running" not in k and "num_batches" not in k) == 1441580


def test_artefacts_checkpoint_and_reload(gold, tmp_path):
    tr = make(gold, dropout=0.5, input_drop=0.25, edge_drop=0.3, wd=1e-4, seed=2)
    for _ in range(3):
        tr.epoch()
    paths = tr.save(tmp_path, "gat-3L10x3h", 4)
    for d in ("output", "logits", "features", "checkpoints"):
        assert paths[d] == tmp_path / d / "gat-3L10x3h" / "4.pt" and paths[d].exists()
    n, C = tr.N, tr.n_classes
    logits, out, feat = (torch.load(paths[d]) for d in ("logits", "output", "features"))
    assert logits.shape == (n, C) and feat.shape == (n, tr.H * tr.n_hidden) and logits.dtype == torch.float32
    assert not logits.is_cuda and not feat.is_cuda
    ref = torch.softmax(logits.double(), 1)
    assert ((out.double() - ref).abs() <= (C + 16) * U * ref + 1e-37).all()
    ck = torch.load(paths["checkpoints"], weights_only=False)
    assert ck["args"].use_labels and ck["args"].n_label_iters == 1 and ck["args"].no_attn_dst and ck["args"].wd == 1e-4
    assert list(ck["model_state_dict"])[:3] == ["convs.0.attn_l", "convs.0.fc.weight", "convs.0.res_fc.weight"]
    # the optimizer state drives torch.optim.RMSprop over the reference-ordered parameters to the engine's next update
    names = list(tr.named_parameters())
    params = [torch.nn.Parameter(ck["model_state_dict"][k].clone()) for k in names]
    opt = torch.optim.RMSprop(params, lr=0.002, weight_decay=1e-4, foreach=False)
    opt.load_state_dict(ck["optimizer_state_dict"])
    assert opt.param_groups[0]["lr"] == ot.lr_at(0.002, 3)
    opt.param_groups[0]["lr"] = ot.lr_at(0.002, 4)                    # adjust_learning_rate of the next epoch
    tr.evaluate()
    eval_logits = tr.Y[-1][:, :C].clone()
    tr.train_step()
    for p, k in zip(params, names):
        p.grad = tr.named_gradients()[k].cpu()
    opt.step()
    after = tr.named_parameters()
    for p, k in zip(params, names):
        sq = opt.state[p]["square_avg"].double()
        upd = ot.lr_at(0.002, 4) * (p.grad.double() + 1e-4 * p.detach().double()).abs() / (sq.sqrt() + 1e-8)
        assert ((after[k].cpu().double() - p.detach().double()).abs() <= 16 * U * (upd + p.detach().double().abs()) + 1e-30).all(), k
    # checkpoint -> new trainer -> evaluate: the same logits, bit for bit
    again = make(gold, dropout=0.5, input_drop=0.25, edge_drop=0.3, wd=1e-4, seed=2)
    again.load_state_dict(ck["model_state_dict"])
    again.evaluate()
    assert torch.equal(again.Y[-1][:, :C], eval_logits)


# ------------------------------------------------------------------------------------------------ full size
def test_full_size_teacher_epochs(tmp_path):
    """ARXIV-shape synthetic graph (N = 169,343), the preset: a few replayed epochs, finite, artefacts at [N, 40] / [N, 750]."""
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    r, c, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(r, c, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    tr = GATTeacherTrainer(adj_of(torch.from_numpy(rs), torch.from_numpy(cs), n), ds.x.cuda(), ds.y.cuda(), ds.split_idx)
    assert tr.n_parameters() == 1441580
    tr.capture()
    hist = tr.run(4, log_every=2)
    assert torch.isfinite(hist).all() and tr.steps_taken() == 4, hist
    paths = tr.save(tmp_path, "gat-3L250x3h", 0)
    assert torch.load(paths["logits"]).shape == (n, 40) and torch.load(paths["features"]).shape == (n, 750)
