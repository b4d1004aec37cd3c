"""G-CRD inside the fused student step (gcrd.GCRD with engine.GCNStudentTrainer / engine_sage.SAGEStudentTrainer): the step
against the eager ``train_step(aux=...)`` path with torch projection heads on the same sample and head weights, the
on-device sampler, and graph replay against eager steps."""
import numpy as np
import pytest
import scipy.stats
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion as C, lib, synthetic
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.gcrd import GCRD, SAMPLE_STREAM
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = pytest.mark.gpu

ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}


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


def make(kind, adj, dims, idx, t_feat, S, p=0.5, beta=0.5, nce_T=0.075, proj=64, seed=0, gcrd=True):
    head = GCRD(t_feat, idx, dims[-2], proj_dim=proj, max_samples=S, nce_T=nce_T, beta=beta, seed=seed + 1) if gcrd else None
    return ENGINES[kind](adj, list(dims), dropout=p, lr=0.01, seed=seed, gcrd=head), head


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


def eager_reference(kind, adj, dims, x, y, t, idx, t_feat, S, sample, p, beta, nce_T, proj, head_state):
    """The same step on the existing path: fused student with train_step(aux=...), torch heads + torch Adam on the heads."""
    tr, _ = make(kind, adj, dims, idx, t_feat, S, p=p, beta=beta, nce_T=nce_T, proj=proj, gcrd=False)
    sp, tp = head_state
    opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=0.01)
    tf = t_feat[idx]

    def aux(f):
        return C.nce_criterion(tr.Y[-1][idx].detach(), y[idx], sp(f[idx]), tp(tf), 1.0, nce_T, S, sampled_inds=sample)[2]
    opt.zero_grad()
    loss = tr.train_step(x, y, idx, t, aux=aux, beta=beta).clone()
    grads = {n: p_.grad.clone() for n, p_ in list(sp.named_parameters()) + [("t" + k, v) for k, v in tp.named_parameters()]}
    opt.step()
    return tr, loss, tr.loss_aux.clone(), grads, sp, tp


@pytest.mark.parametrize("kind", ["gcn", "sage"])
@pytest.mark.parametrize("S", [256, 100_000])
def test_fused_step_equals_eager_aux_path(kind, S):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    beta, nce_T, proj = 0.5, 0.075, 64
    tr, head = make(kind, adj, dims, idx, t_feat, S, beta=beta, nce_T=nce_T, proj=proj)
    n = idx.numel()
    sample = np.random.RandomState(3).choice(n, S, replace=False) if S < n else np.arange(n)
    sp, tp = torch_heads(head)
    ref_tr, ref_loss, ref_aux, ref_g, sp, tp = eager_reference(kind, adj, dims, x, y, t, idx, t_feat, S,
                                                               sample if S < n else None, 0.5, beta, nce_T, proj, (sp, tp))
    loss = tr.train_step(x, y, idx, t, sample=torch.as_tensor(sample)).clone()
    assert torch.equal(head.sample().cpu(), torch.as_tensor(sample, dtype=torch.int64))
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
    assert int(head.step_count.item()) == int(tr.step_count.item()) == 1           # the heads' Adam ran once


def draw(n, seed, step):
    L = lib.load()
    perm = torch.empty(n, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(L.b200gnn_gcrd_sample_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
    st = torch.tensor([step], dtype=torch.int32, device="cuda")
    lib.check(L.b200gnn_gcrd_sample_i32(n, seed, SAMPLE_STREAM, st.data_ptr(), perm.data_ptr(), ws.data_ptr(), lib.stream_ptr()),
              "gcrd_sample_i32")
    return perm.long().cpu()


def test_sampler_distinct_deterministic_fresh_and_uniform():
    n, S = 1000, 100
    p0 = draw(n, 7, 0)
    assert torch.equal(torch.sort(p0).values, torch.arange(n))               # a permutation: any prefix is distinct
    assert torch.equal(p0, draw(n, 7, 0))                                    # a function of (seed, step) only
    assert not torch.equal(set_of(p0[:S]), set_of(draw(n, 7, 1)[:S]))       # a fresh set at the next step
    assert not torch.equal(set_of(p0[:S]), set_of(draw(n, 8, 0)[:S]))
    counts = torch.zeros(n)
    draws = 400
    for k in range(draws):
        counts[draw(n, 7, k)[:S]] += 1
    expected = draws * S / n
    stat = float(((counts - expected) ** 2 / expected).sum())
    # without replacement each count is binomial-like with variance expected * (1 - S/n): scale before the chi-square bound
    stat /= 1 - S / n
    assert scipy.stats.chi2.ppf(1e-4, n - 1) < stat < scipy.stats.chi2.ppf(1 - 1e-4, n - 1), stat


def set_of(t):
    return torch.sort(t).values


@pytest.mark.parametrize("kind", ["gcn", "sage"])
def test_graph_replay_equals_eager_steps_bitwise(kind):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    a, ha = make(kind, adj, dims, idx, t_feat, 256)
    b, hb = make(kind, adj, dims, idx, t_feat, 256)
    eager, samples = [], []
    for _ in range(3):
        eager.append(a.train_step(x, y, idx, t).clone())
        samples.append(ha.sample().clone())
    assert not torch.equal(samples[0], samples[1])                           # every step draws afresh
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


def test_supervised_form_and_state_round_trip():
    """gnn.py's CE + beta * nce (no teacher logits); the head state dicts load back into a fresh object unchanged."""
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat = problem(dims=dims)
    tr, head = make("gcn", adj, dims, idx, t_feat, 256)
    loss = tr.train_step(x, y, idx).clone()
    assert torch.isfinite(loss).all()
    assert abs(float(loss[0]) - float(loss[1]) - 0.5 * float(head.loss_aux)) < 1e-5 * float(loss[0])
    other = GCRD(t_feat, idx, 64, proj_dim=64, max_samples=256, seed=5)
    other.load_student_proj_state_dict(head.student_proj_state_dict())
    other.load_teacher_proj_state_dict(head.teacher_proj_state_dict())
    for a, b in ((head.student_proj_state_dict(), other.student_proj_state_dict()),
                 (head.teacher_proj_state_dict(), other.teacher_proj_state_dict())):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert head.teacher_proj_state_dict()["0.weight"].shape == (64, 750)
    with pytest.raises(ValueError):
        tr.train_step(x, y, idx, aux=lambda f: f.sum())


def test_full_arxiv_shape_one_step_against_eager_aux_path():
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.cuda()
    perm = (ei[1] * n + ei[0]).argsort()
    adj = SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    x, y, t = ds.x.cuda(), ds.y.squeeze(1).cuda(), ds.teacher_logits.cuda()
    idx, t_feat = ds.split_idx["train"].cuda(), ds.teacher_feat.cuda()
    dims, S, beta = (128, 256, 256, 40), 16384, 0.1
    tr, head = make("sage", adj, dims, idx, t_feat, S, beta=beta, proj=256)
    sample = np.random.RandomState(0).choice(idx.numel(), S, replace=False)
    sp, tp = torch_heads(head)
    ref_tr, ref_loss, ref_aux, ref_g, _, _ = eager_reference("sage", adj, dims, x, y, t, idx, t_feat, S, sample, 0.5, beta,
                                                             0.075, 256, (sp, tp))
    loss = tr.train_step(x, y, idx, t, sample=torch.as_tensor(sample)).clone()
    assert abs(float(head.loss_aux) - float(ref_aux)) < 2e-5 * abs(float(ref_aux))
    assert abs(float(loss[0]) - float(ref_loss[0])) < 2e-5 * abs(float(ref_loss[0]))
    check_grads([(n_, a, b, pre) for (n_, a, pre), (_, b, _) in zip(trainer_grads(tr), trainer_grads(ref_tr))])
    check_grads([("Ws", head.gW_s, ref_g["0.weight"], False), ("gs", head.ggamma_s, ref_g["1.weight"], False),
                 ("Wt", head.gW_t[:, :head.F_t], ref_g["t0.weight"], False), ("gt", head.ggamma_t, ref_g["t1.weight"], False)])
