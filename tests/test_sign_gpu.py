"""SIGN student (arxiv_dgl/sign.py:105-157): the fp64 oracle against the reference class's fixture (CPU), the PReLU
prologue / backward-epilogue GEMMs and the batch gather bit for bit against their materialised twins, and the fused
training step, epochs, graph replay and inference of SIGNStudentTrainer against the oracle (GPU)."""
from pathlib import Path

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from oracle import criterion as oc
from oracle import sign as osign

GOLD = Path(__file__).resolve().parent / "golden" / "sign_model_arxiv.pt"
gpu = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


# ----------------------------------------------------------------------------- oracle vs the reference class (CPU)
@pytest.mark.parametrize("ff", [1, 2, 3])
def test_oracle_reproduces_reference_sign_class(ff):
    gold = torch.load(GOLD)
    m = gold["models"][ff]
    feats = [f.double() for f in gold["feats"]]
    sd = {k: v.double().requires_grad_(True) for k, v in m["state"].items()}
    logits, out_feat = osign.sign_forward(feats, sd, ff)
    assert rel_err(logits, m["logits_eval"]) < 1e-5 and rel_err(out_feat, m["out_feat_eval"]) < 1e-5
    b = gold["batch"]
    logits, out_feat = osign.sign_forward([f[b] for f in feats], sd, ff)
    loss = oc.cross_entropy(logits, gold["labels"][b])
    loss.backward()
    assert rel_err(logits, m["logits_train"]) < 1e-5 and rel_err(out_feat, m["out_feat_train"]) < 1e-5
    assert abs(loss.item() - m["loss"].item()) < 1e-5 * abs(m["loss"].item())
    assert set(m["grads"]) == set(sd)
    for k, g in m["grads"].items():
        assert rel_err(sd[k].grad, g) < 1e-5, k


# ----------------------------------------------------------------------------- kernels (GPU)
def _ops():
    from efficient_gnns_b200 import ops
    return ops


def rand_bits(n, K, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randint(-2**31, 2**31 - 1, (n, (K + 31) // 32), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)


def inv_keep(p):
    return (torch.tensor(1.0) / (1 - torch.tensor(p))).item() if p > 0 else 1.0


@gpu
@pytest.mark.parametrize("slope", [0.25, -0.5, 0.0])
@pytest.mark.parametrize("K", [128, 512, 3072])
def test_prelu_prologue_gemm_and_wgrad_match_materialised(K, slope):
    ops = _ops()
    M, p = 1001, 0.1
    g = torch.Generator(device="cuda").manual_seed(K)
    z = torch.randn(M, K, device="cuda", generator=g)
    a = torch.tensor([slope], device="cuda")
    bits = rand_bits(M, K, K + 1)
    x = ops.prelu_bits(z, bits, a, p)
    for N in (512, 40):
        w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
        bias = torch.randn(N, device="cuda", generator=g)
        hi, lo = ops.split_tf32(w)
        ref = ops.gemm_tf32x3(x, hi, lo, bias=bias)
        assert torch.equal(ops.gemm_tf32x3_prelu(z, a, bits, p, hi, lo, bias=bias), ref)
        gr = torch.randn(M, N, device="cuda", generator=g)
        got = ops.gemm_wgrad_tf32x3_prelu(z, a, bits, p, gr)
        blk = K if K <= 2048 else ops.WGRAD_PRELU_BLOCK
        for c0 in range(0, K, blk):
            ref_w = ops.gemm_wgrad_tf32x3(x[:, c0:c0 + blk].contiguous(), gr, wide=True)
            assert torch.equal(got[c0:c0 + blk], ref_w)
    keep = unpack(bits)[:, :K]
    assert torch.equal(x, torch.where(keep, torch.where(z > 0, z, z * a) * inv_keep(p), torch.zeros_like(z)))


@gpu
@pytest.mark.parametrize("accumulate", [False, True])
@pytest.mark.parametrize("N,K", [(512, 512), (3072, 512), (3072, 40)])
def test_prelu_backward_epilogue(N, K, accumulate):
    ops = _ops()
    M, p, slope = 777, 0.5, -0.3
    g = torch.Generator(device="cuda").manual_seed(N + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    z = torch.randn(M, N, device="cuda", generator=g)
    c0 = torch.randn(M, N, device="cuda", generator=g)
    a = torch.tensor([slope], device="cuda")
    bits = rand_bits(M, N, N)
    keep = unpack(bits)[:, :N]
    hi, lo = ops.split_tf32(W)
    dA = c0.clone() if accumulate else torch.empty(M, N, device="cuda")
    ops.gemm_tf32x3(A, hi, lo, out=dA, accumulate=accumulate)
    gk = torch.where(keep, dA * inv_keep(p), torch.zeros_like(dA))
    ref = torch.where(z > 0, gk, gk * a)
    part = torch.empty(ops.gemm_stat_slots(M, N), dtype=torch.float64, device="cuda")
    outs = []
    for _ in range(2):
        out = c0.clone() if accumulate else torch.full((M, N), float("nan"), device="cuda")
        sg = torch.full((1,), 5.0, device="cuda")
        ops.gemm_tf32x3_prelu_bwd(A, hi, lo, out, z, bits, a, p, sg, part, accumulate=accumulate)
        assert torch.equal(out, ref)
        outs.append(sg.clone())
    assert torch.equal(outs[0], outs[1])
    terms = torch.where(z <= 0, gk.double() * z.double(), torch.zeros_like(z, dtype=torch.float64))
    assert abs(outs[0].item() - terms.sum().item()) <= 1e-6 * terms.abs().sum().item()
    sg = torch.full((1,), 5.0, device="cuda")
    out = c0.clone() if accumulate else torch.empty(M, N, device="cuda")
    ops.gemm_tf32x3_prelu_bwd(A, hi, lo, out, z, bits, a, p, sg, part, accumulate=accumulate, slope_accumulate=True)
    assert sg.item() == pytest.approx(5.0 + outs[0].item(), rel=1e-6)


def unpack(bits):
    sh = torch.arange(32, device=bits.device, dtype=torch.int32)
    return ((bits.unsqueeze(-1) >> sh) & 1).bool().flatten(-2)


@gpu
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_gather_with_input_dropout_is_exact(p):
    ops = _ops()
    n, F, H, C, B = 500, 128, 3, 40, 333
    g = torch.Generator(device="cuda").manual_seed(3)
    feats = [torch.randn(n, F, device="cuda", generator=g) for _ in range(H)]
    idx = torch.randint(0, n, (B,), device="cuda", generator=g)
    labels = torch.randint(0, C, (n,), device="cuda", generator=g)
    teacher = torch.randn(n, C, device="cuda", generator=g)
    step = torch.tensor([2], dtype=torch.int32, device="cuda")
    out = torch.empty(H, B, F, device="cuda")
    lo, to = torch.empty(B, dtype=torch.int64, device="cuda"), torch.empty(B, C, device="cuda")
    ops.sign_gather(feats, idx, p, 9, 4, out, step_dev=step, step_mul=7, labels=labels, labels_out=lo, teacher=teacher,
                    teacher_out=to)
    for h in range(H):
        keep = ops.dropout_mask(B, F, p, 9, 4 + h + 2 * 7).bool()
        assert torch.equal(out[h], torch.where(keep, feats[h][idx] * inv_keep(p), torch.zeros(B, F, device="cuda")))
    assert torch.equal(lo, labels[idx]) and torch.equal(to, teacher[idx])


# ----------------------------------------------------------------------------- the trainer (GPU)
def _trainer(**kw):
    from efficient_gnns_b200.engine_sign import SIGNStudentTrainer
    return SIGNStudentTrainer(**kw)


@gpu
@pytest.mark.parametrize("ff", [1, 2, 3])
def test_engine_reproduces_reference_fixture(ff):
    gold = torch.load(GOLD)
    m = gold["models"][ff]
    feats = [f.cuda() for f in gold["feats"]]
    tr = _trainer(feats=feats, n_classes=gold["n_classes"], hidden=gold["hidden"], ff_layer=ff, dropout=0.0, input_drop=0.0,
                  batch_size=64)
    tr.load_state_dict({k: v.cuda() for k, v in m["state"].items()})
    sd = tr.state_dict()
    assert set(sd) == set(m["state"]) and all(torch.equal(sd[k].cpu(), m["state"][k]) for k in sd)
    assert rel_err(tr.predict(), m["logits_eval"]) < 1e-5
    loss = tr.train_step(gold["batch"].cuda(), gold["labels"].cuda())
    assert abs(loss[0].item() - m["loss"].item()) < 1e-5 * abs(m["loss"].item())
    assert rel_err(tr.logits(), m["logits_train"]) < 1e-5 and rel_err(tr.out_feat(), m["out_feat_train"]) < 1e-5
    gd = tr.grad_dict()
    for k, g in m["grads"].items():
        assert rel_err(gd[k], g) < 1e-5, k


def _problem(seed=0, n=600, F=16, H=3, C=8, n_train=300):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(n, F, generator=g) for _ in range(H)]
    y = torch.randint(0, C, (n,), generator=g)
    t = torch.randn(n, C, generator=g) * 2
    train_idx = torch.randperm(n, generator=g)[:n_train]
    return feats, y, t, train_idx


def _masks(tr, B, step):
    """The keep-masks of training step ``step`` (the Philox offsets the trainer draws), bool on the CPU."""
    from efficient_gnns_b200 import ops
    H, hid, ff, D, s = tr.H, tr.hidden, tr.ff, tr.D, tr.seed
    m = lambda rows, K, p, off: ops.dropout_mask(rows, K, p, s, step * D + off).bool().cpu()  # noqa: E731
    hidden = [[m(B, hid, tr.p, H + h * (ff - 1) + i) for i in range(ff - 1)] for h in range(H)]
    project = [m(B, hid, tr.p, H + H * (ff - 1) + i) for i in range(ff - 1)]
    cat = m(B * H, hid, tr.p, H + (H + 1) * (ff - 1)).view(B, H * hid)
    return dict(input=[m(B, tr.F, tr.p_in, h) for h in range(H)], hidden=hidden, project=project, cat=cat)


def _oracle_step(tr, sd, feats, y, t, b, masks, mode, head=None, t_feat=None, inds=None, beta=0.7):
    sd = {k: v.detach().cpu().double().requires_grad_(True) for k, v in sd.items()}
    logits, out_feat = osign.sign_forward([f[b].double() for f in feats], sd, tr.ff, masks, tr.p, tr.p_in)
    if mode == "supervised":
        loss = oc.cross_entropy(logits, y[b]); parts = (loss, loss)
    else:
        loss, lc, lk = oc.kd_criterion(logits, y[b], t[b].double(), tr.alpha, tr.kd_T); parts = (lc, lk)
    if mode == "fitnet":
        loss = loss + beta * oc.fitnet_criterion(logits, y[b], head(out_feat), t_feat[b], 1.0)[2]
    elif mode == "gcrd":
        loss = loss + beta * oc.nce_criterion(logits, y[b], head(out_feat), t_feat[b], 0.5, 0.075, 8192, inds)[2]
    loss.backward()
    return logits.detach(), out_feat.detach(), loss.detach(), parts, {k: v.grad for k, v in sd.items()}


@gpu
@pytest.mark.parametrize("mode", ["supervised", "kd", "fitnet", "gcrd"])
@pytest.mark.parametrize("ff", [1, 2, 3])
def test_step_matches_fp64_oracle(ff, mode):
    feats, y, t, train_idx = _problem(ff)
    tr = _trainer(feats=[f.cuda() for f in feats], n_classes=8, hidden=64, ff_layer=ff, dropout=0.5, input_drop=0.1,
                  batch_size=256, seed=5)
    with torch.no_grad():                                   # non-default slopes, of both signs
        for k, v in tr.P.items():
            if "slope" in k:
                v.copy_(torch.linspace(-0.4, 0.3, v.numel()))
    sd0 = tr.state_dict()
    b = train_idx[:200]
    head = t_feat = inds = None
    aux = None
    g = torch.Generator().manual_seed(11)
    if mode in ("fitnet", "gcrd"):
        head = torch.nn.Linear(3 * 64, 16).double()
        t_feat = torch.randn(600, 16, generator=g, dtype=torch.float64)
        inds = torch.randperm(200, generator=g)[:150]
        head_c = torch.nn.Linear(3 * 64, 16).cuda()
        head_c.load_state_dict({k: v.float() for k, v in head.state_dict().items()})
        tf_c, inds_c, yb = t_feat.float().cuda(), inds.cuda(), y[b].cuda()
        if mode == "fitnet":
            aux = lambda f: oc.fitnet_criterion(tr.logits().detach(), yb, head_c(f), tf_c[b.cuda()], 1.0)[2]  # noqa: E731
        else:
            aux = lambda f: oc.nce_criterion(tr.logits().detach(), yb, head_c(f), tf_c[b.cuda()], 0.5, 0.075, 8192, inds_c)[2]  # noqa: E731
    teacher = None if mode == "supervised" else t.cuda()
    loss = tr.train_step(b.cuda(), y.cuda(), teacher, aux=aux, beta=0.7).cpu()
    masks = _masks(tr, b.numel(), 0)
    logits, out_feat, ref_loss, parts, grads = _oracle_step(tr, sd0, feats, y, t, b, masks, mode, head, t_feat, inds)
    assert rel_err(tr.logits(), logits) < 1e-5 and rel_err(tr.out_feat(), out_feat) < 1e-5
    assert abs(loss[0].item() - ref_loss.item()) < 1e-5 * abs(ref_loss.item())
    assert abs(loss[1].item() - parts[0].item()) < 1e-5 * abs(parts[0].item())
    gd = tr.grad_dict()
    assert set(gd) == set(grads)
    for k, gr in grads.items():
        assert rel_err(gd[k], gr) < 2e-5, k


@gpu
@pytest.mark.parametrize("B", [1, 100, 44])
def test_small_and_ragged_batches(B):
    feats, y, t, train_idx = _problem(3)
    tr = _trainer(feats=[f.cuda() for f in feats], n_classes=8, hidden=64, ff_layer=2, batch_size=128, seed=2)
    sd0 = tr.state_dict()
    b = train_idx[:B]
    tr.train_step(b.cuda(), y.cuda(), t.cuda())
    logits, _, ref_loss, _, grads = _oracle_step(tr, sd0, feats, y, t, b, _masks(tr, B, 0), "kd")
    assert rel_err(tr.logits(), logits) < 1e-5
    assert abs(tr.loss_out[0].item() - ref_loss.item()) < 1e-5 * abs(ref_loss.item())
    gd = tr.grad_dict()
    for k, gr in grads.items():
        assert rel_err(gd[k], gr) < 2e-5, k


@gpu
def test_epoch_covers_every_training_node_once_and_graph_replay_is_bit_identical():
    feats, y, t, train_idx = _problem(4)
    fc, yc, tc, ic = [f.cuda() for f in feats], y.cuda(), t.cuda(), train_idx.cuda()
    mk = lambda: _trainer(feats=fc, n_classes=8, hidden=64, ff_layer=2, batch_size=128, seed=1)  # noqa: E731
    eager, graphed = mk(), mk()
    order = eager.epoch_order(ic, 0)
    assert torch.equal(order.sort().values, ic.sort().values)
    assert not torch.equal(order, eager.epoch_order(ic, 1))
    graphed.capture([128, 300 - 256], yc, tc)
    assert torch.equal(graphed.params, eager.params) and int(graphed.step_count) == 0
    le = torch.cat([eager.train_epoch(ic, yc, tc) for _ in range(2)])
    lg = torch.cat([graphed.train_epoch(ic, yc, tc) for _ in range(2)])
    assert le.shape == (6, 3) and int(eager.step_count) == 6
    assert torch.equal(le, lg)
    assert torch.equal(eager.params, graphed.params) and torch.equal(eager.exp_avg_sq, graphed.exp_avg_sq)
    assert torch.equal(eager.out_feat(), graphed.out_feat())


@gpu
def test_predict_matches_oracle_eval_logits():
    feats, y, t, train_idx = _problem(6)
    tr = _trainer(feats=[f.cuda() for f in feats], n_classes=8, hidden=64, ff_layer=3, batch_size=128, seed=3)
    tr.train_epoch(train_idx.cuda(), y.cuda(), t.cuda())          # move the parameters off their initial values
    sd = {k: v.cpu().double() for k, v in tr.state_dict().items()}
    ref, _ = osign.sign_forward([f.double() for f in feats], sd, 3)
    assert rel_err(tr.predict(batch_size=250), ref) < 1e-5


@gpu
def test_rejects_what_it_does_not_support():
    from efficient_gnns_b200 import lib
    feats = [torch.randn(10, 16, device="cuda") for _ in range(2)]
    with pytest.raises(ValueError):
        _trainer(feats=feats, n_classes=8, hidden=64, weight_decay=5e-4)
    with pytest.raises(lib.B200GnnError):
        _trainer(feats=[f.cpu() for f in feats], n_classes=8, hidden=64)
    with pytest.raises(lib.B200GnnError):
        _trainer(feats=[torch.randn(10, 18, device="cuda")], n_classes=8, hidden=64)
    with pytest.raises(lib.B200GnnError):
        _trainer(feats=feats, n_classes=10, hidden=64)
