"""GSP inside the fused student step (gsp.GSP with engine.GCNStudentTrainer / engine_sage.SAGEStudentTrainer): the step against
the eager ``train_step(aux=...)`` path with torch projection heads on the same sample and head weights, one step at the full
ARXIV shape, graph replay against eager steps, a fresh sample every step, and every refusal."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion as C, synthetic
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.gcrd import GCRD
from efficient_gnns_b200.gsp import GSP
from efficient_gnns_b200.lsp import LSP
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = pytest.mark.gpu

ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}
KERNELS = ["cosine", "poly", "l2", "rbf"]


def problem(n=3000, e=20_000, dims=(32, 64, 64, 8), seed=0, f_t=750):
    ei = skewed_edges(n, e, seed)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    g = torch.Generator().manual_seed(seed + 9)
    x = torch.randn(n, dims[0], generator=g).cuda()
    y = torch.randint(0, dims[-1], (n,), generator=g).cuda()
    t = (torch.randn(n, dims[-1], generator=g) * 2).cuda()
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values.cuda()
    t_feat = torch.randn(n, f_t, generator=g).cuda()
    return adj, x, y, t, idx, t_feat


def make(kind, adj, dims, idx, t_feat, S, kernel, p=0.5, beta=0.5, proj=64, seed=0, gsp=True):
    obj = GSP(t_feat, idx, dims[-2], proj_dim=proj, max_samples=S, kernel=kernel, beta=beta, seed=seed + 1) if gsp else None
    return ENGINES[kind](adj, list(dims), dropout=p, lr=0.01, seed=seed, gsp=obj), obj


def torch_heads(head):
    sp = torch.nn.Sequential(torch.nn.Linear(head.H, head.P), torch.nn.BatchNorm1d(head.P), torch.nn.ReLU()).cuda()
    tp = torch.nn.Sequential(torch.nn.Linear(head.F_t, head.P), torch.nn.BatchNorm1d(head.P), torch.nn.ReLU()).cuda()
    sp.load_state_dict({k: v.cuda() for k, v in head.student_proj_state_dict().items()})
    tp.load_state_dict({k: v.cuda() for k, v in head.teacher_proj_state_dict().items()})
    return sp, tp


def trainer_grads(tr):
    """(name, gradient, sits in front of a BatchNorm) for every student parameter."""
    out = []
    if isinstance(tr, GCNStudentTrainer):
        for l in range(tr.L):
            out += [(f"W{l}", tr.gW[l], False), (f"b{l}", tr.gb[l], l < tr.L - 1)]
            if l < tr.L - 1:
                out += [(f"gamma{l}", tr.ggamma[l], False), (f"beta{l}", tr.gbeta[l], False)]
    else:
        for l in range(tr.L):
            out += [(f"Wl{l}", tr.gWl[l], False), (f"bl{l}", tr.gbl[l], l < tr.L - 1), (f"Wr{l}", tr.gWr[l], False)]
            if l < tr.L - 1:
                out += [(f"gamma{l}", tr.ggamma[l], False), (f"beta{l}", tr.gbeta[l], False)]
    return out


def check_grads(pairs, tol=1e-4):
    scale = max(b.abs().max().item() for _, _, b, _ in pairs)
    for name, a, b, pre_bn in pairs:
        if pre_bn:       # a bias in front of BatchNorm: its exact gradient is 0, both sides carry rounding only
            assert a.abs().max().item() < 1e-5 * scale and b.abs().max().item() < 1e-5 * scale, name
        else:
            assert rel_err(a, b) < tol, (name, rel_err(a, b))


def eager_reference(kind, adj, dims, x, y, t, idx, t_feat, S, sample, p, beta, kernel, proj, head_state):
    """The same step on the existing path: fused student with train_step(aux=...), torch heads + torch Adam on the heads."""
    tr, _ = make(kind, adj, dims, idx, t_feat, S, kernel, p=p, beta=beta, proj=proj, gsp=False)
    sp, tp = head_state
    opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=0.01)
    tf = t_feat[idx]

    def aux(f):
        return C.gpw_criterion(tr.Y[-1][idx].detach(), y[idx], sp(f[idx]), tp(tf), kernel, 1, S, sampled_inds=sample)[2]
    opt.zero_grad()
    loss = tr.train_step(x, y, idx, t, aux=aux, beta=beta).clone()
    grads = {n: p_.grad.clone() for n, p_ in list(sp.named_parameters()) + [("t" + k, v) for k, v in tp.named_parameters()]}
    opt.step()
    return tr, loss, tr.loss_aux.clone(), grads, sp, tp


def compare_step(tr, head, ref_tr, ref_loss, ref_aux, ref_g, sp, tp, loss):
    assert abs(float(head.loss_aux) - float(ref_aux)) < 2e-5 * abs(float(ref_aux))
    assert abs(float(loss[0]) - float(ref_loss[0])) < 2e-5 * abs(float(ref_loss[0]))
    assert torch.equal(loss[1:], ref_loss[1:])
    check_grads([(n_, a, b, pre) for (n_, a, pre), (_, b, _) in zip(trainer_grads(tr), trainer_grads(ref_tr))])
    F_t = head.F_t
    check_grads([("Ws", head.gW_s, ref_g["0.weight"], False), ("bs", head.gb_s, ref_g["0.bias"], True),
                 ("gs", head.ggamma_s, ref_g["1.weight"], False), ("betas", head.gbeta_s, ref_g["1.bias"], False),
                 ("Wt", head.gW_t[:, :F_t], ref_g["t0.weight"], False), ("bt", head.gb_t, ref_g["t0.bias"], True),
                 ("gt", head.ggamma_t, ref_g["t1.weight"], False), ("betat", head.gbeta_t, ref_g["t1.bias"], False)])
    assert not head.gW_t[:, F_t:].any() and not head.W_t[:, F_t:].any()       # the padded columns stay zero
    for mine, ref in ((head.student_proj_state_dict(), sp.state_dict()), (head.teacher_proj_state_dict(), tp.state_dict())):
        for k in ("1.running_mean", "1.running_var"):
            assert rel_err(mine[k], ref[k]) < 1e-5, k
        assert int(mine["1.num_batches_tracked"]) == int(ref["1.num_batches_tracked"]) == 1
    assert int(head.step_count.item()) == 1                                  # the heads' Adam ran once


@pytest.mark.parametrize("kind", ["gcn", "sage"])
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("S", [256, 100_000])
@pytest.mark.parametrize("form", ["kd", "supervised"])
def test_fused_step_equals_eager_aux_path(kind, kernel, S, form):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    beta, proj = (10.0 if kernel == "cosine" else 0.5), 64
    tr, head = make(kind, adj, dims, idx, t_feat, S, kernel, beta=beta, proj=proj)
    n = idx.numel()
    sample = np.random.RandomState(3).choice(n, S, replace=False) if S < n else np.arange(n)
    sp, tp = torch_heads(head)
    teacher = t if form == "kd" else None
    ref = eager_reference(kind, adj, dims, x, y, teacher, idx, t_feat, S, sample if S < n else None, 0.5, beta, kernel, proj,
                          (sp, tp))
    loss = tr.train_step(x, y, idx, teacher, sample=torch.as_tensor(sample)).clone()
    assert torch.equal(head.sample().cpu(), torch.as_tensor(sample, dtype=torch.int64))
    compare_step(tr, head, *ref[:4], ref[4], ref[5], loss)


def arxiv():
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.cuda()
    perm = (ei[1] * n + ei[0]).argsort()
    adj = SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    return adj, ds.x.cuda(), ds.y.squeeze(1).cuda(), ds.teacher_logits.cuda(), ds.split_idx["train"].cuda(), ds.teacher_feat.cuda()


@pytest.mark.parametrize("kind", ["gcn", "sage"])
def test_full_arxiv_shape_one_step_at_the_script_settings(kind):
    """run_kd_and_aux.sh: cosine, beta 10, max_samples 4096, proj_dim 128, the 750-wide teacher."""
    adj, x, y, t, idx, t_feat = arxiv()
    assert t_feat.shape[1] == 750
    dims, S, beta, proj = (128, 256, 256, 40), 4096, 10.0, 128
    tr, head = make(kind, adj, dims, idx, t_feat, S, "cosine", beta=beta, proj=proj)
    sample = np.random.RandomState(0).choice(idx.numel(), S, replace=False)
    sp, tp = torch_heads(head)
    ref = eager_reference(kind, adj, dims, x, y, t, idx, t_feat, S, sample, 0.5, beta, "cosine", proj, (sp, tp))
    loss = tr.train_step(x, y, idx, t, sample=torch.as_tensor(sample)).clone()
    compare_step(tr, head, *ref[:4], ref[4], ref[5], loss)


@pytest.mark.parametrize("kind", ["gcn", "sage"])
@pytest.mark.parametrize("kernel", ["cosine", "rbf"])
def test_graph_replay_equals_eager_steps_bitwise_with_a_fresh_sample(kind, kernel):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    a, ha = make(kind, adj, dims, idx, t_feat, 256, kernel)
    b, hb = make(kind, adj, dims, idx, t_feat, 256, kernel)
    eager, samples = [], []
    for _ in range(3):
        eager.append(a.train_step(x, y, idx, t).clone())
        samples.append(ha.sample().clone())
    for k in range(2):                                                       # every step draws afresh
        assert not torch.equal(torch.sort(samples[k]).values, torch.sort(samples[k + 1]).values)
    b.capture(x, y, idx, t, warmup=0)
    for k in range(3):
        got = b.replay().clone()
        assert torch.equal(got, eager[k]), k
        assert torch.equal(hb.sample(), samples[k])
    assert torch.equal(a.params, b.params) and torch.equal(ha.params, hb.params)
    for s_a, s_b in ((ha.student_proj_state_dict(), hb.student_proj_state_dict()),
                     (ha.teacher_proj_state_dict(), hb.teacher_proj_state_dict())):
        for k in s_a:
            assert torch.equal(s_a[k], s_b[k]), k
    assert torch.equal(ha.loss_aux, hb.loss_aux)


def test_refusals():
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    with pytest.raises(ValueError):
        GSP(t_feat, idx, 64, proj_dim=64, kernel="gaussian")
    for proj in (32, 48, 100, 288):                                          # gemm_stats_supported rejects these
        with pytest.raises(ValueError):
            GSP(t_feat, idx, 64, proj_dim=proj)
    for hidden in (6, 516):
        with pytest.raises(ValueError):
            GSP(t_feat, idx, hidden, proj_dim=64)
    gsp = GSP(t_feat, idx, 64, proj_dim=64, max_samples=256)
    others = dict(gcrd=GCRD(t_feat, idx, 64, proj_dim=64, max_samples=256),
                  lsp=LSP(t_feat, idx, torch.stack([torch.arange(10), torch.arange(1, 11)]).cuda(), 64))
    for kind in ENGINES:
        for name, other in others.items():
            with pytest.raises(ValueError):
                ENGINES[kind](adj, list(dims), gsp=gsp, **{name: other})
        with pytest.raises(ValueError):                                      # bound to a student of another width
            ENGINES[kind](adj, [32, 64, 32, 8], gsp=GSP(t_feat, idx, 64, proj_dim=64, max_samples=256))
        tr = ENGINES[kind](adj, list(dims), gsp=GSP(t_feat, idx, 64, proj_dim=64, max_samples=256))
        with pytest.raises(ValueError):
            tr.train_step(x, y, idx, t, aux=lambda f: f.sum())
        n = idx.numel()
        for bad in (torch.arange(255), torch.arange(257), torch.cat([torch.arange(255), torch.tensor([0])]),
                    torch.cat([torch.arange(255), torch.tensor([n])]), torch.cat([torch.tensor([-1]), torch.arange(255)])):
            with pytest.raises(ValueError):
                tr.train_step(x, y, idx, t, sample=bad)
    # without an objective the step is the plain one: sample= is refused as before
    tr = GCNStudentTrainer(adj, list(dims))
    with pytest.raises(ValueError):
        tr.train_step(x, y, idx, t, sample=torch.arange(256))


def test_supervised_form_and_state_round_trip():
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    tr, head = make("gcn", adj, dims, idx, t_feat, 256, "rbf")
    loss = tr.train_step(x, y, idx).clone()
    assert torch.isfinite(loss).all()
    assert abs(float(loss[0]) - float(loss[1]) - 0.5 * float(head.loss_aux)) < 1e-5 * float(loss[0])
    other = GSP(t_feat, idx, 64, proj_dim=64, max_samples=256, seed=5)
    other.load_student_proj_state_dict(head.student_proj_state_dict())
    other.load_teacher_proj_state_dict(head.teacher_proj_state_dict())
    for a, b in ((head.student_proj_state_dict(), other.student_proj_state_dict()),
                 (head.teacher_proj_state_dict(), other.teacher_proj_state_dict())):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert head.launches_per_step(x, y, idx) > 0
