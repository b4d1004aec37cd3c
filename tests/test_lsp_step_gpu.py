"""LSP inside the fused student step (lsp.LSP with engine.GCNStudentTrainer / engine_sage.SAGEStudentTrainer): bit for bit
the eager ``train_step(aux=lpw_criterion ...)`` path, at a small size for every kernel and loss form and at the full ARXIV
shape; graph replay against eager steps; and every refusal."""
import numpy as np
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import criterion as C, lib, synthetic
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.gcrd import GCRD
from efficient_gnns_b200.lsp import LSP
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import graph as og

pytestmark = pytest.mark.gpu

ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}
KERNELS = ["cosine", "poly", "l2", "rbf"]


def problem(n=3000, e=20_000, dims=(32, 64, 64, 8), seed=0, f_t=90):
    ei = skewed_edges(n, e, seed)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    g = torch.Generator().manual_seed(seed + 9)
    x = torch.randn(n, dims[0], generator=g).cuda()
    y = torch.randint(0, dims[-1], (n,), generator=g).cuda()
    t = (torch.randn(n, dims[-1], generator=g) * 2).cuda()
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values
    t_feat = torch.randn(n, f_t, generator=g).relu().cuda()
    # the reference's subgraph(train_idx, stack(adj_t.coo()[:2]), relabel_nodes=True)[0]
    sub = torch.from_numpy(og.subgraph(idx.numpy(), np.stack([r, c]), True)[0]).cuda()
    return adj, x, y, t, idx.cuda(), t_feat, sub


def state(tr):
    return [tr.loss_out, tr.grads, tr.params, tr.exp_avg, tr.exp_avg_sq] + (
        [torch.stack(tr.running_mean), torch.stack(tr.running_var)] if tr.L > 1 else [])


def assert_same(a, b):
    for k, (u, v) in enumerate(zip(state(a), state(b))):
        assert torch.equal(u, v), k


def twins(kind, adj, dims, idx, t_feat, sub, kernel, beta, p=0.5):
    obj = LSP(t_feat, idx, sub, dims[-2], kernel=kernel, beta=beta)
    a = ENGINES[kind](adj, list(dims), dropout=p, lr=0.01, seed=3, lsp=obj)
    b = ENGINES[kind](adj, list(dims), dropout=p, lr=0.01, seed=3)
    return a, obj, b


def eager_step(tr, x, y, idx, t, t_feat, sub, kernel, beta):
    aux = lambda f: C.lpw_criterion(tr.Y[-1][idx].detach(), y[idx], f[idx], t_feat[idx], sub, kernel, 1)[2]
    return tr.train_step(x, y, idx, t, aux=aux, beta=beta)


@pytest.mark.parametrize("kind", ["gcn", "sage"])
@pytest.mark.parametrize("kernel", KERNELS)
@pytest.mark.parametrize("form", ["kd", "supervised"])
def test_step_equals_eager_aux_path_bitwise(kind, kernel, form):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat, sub = problem(dims=dims)
    t = t if form == "kd" else None
    beta = 100.0 if kernel == "cosine" else 0.5
    a, obj, b = twins(kind, adj, dims, idx, t_feat, sub, kernel, beta)
    for _ in range(3):
        a.train_step(x, y, idx, t)
        eager_step(b, x, y, idx, t, t_feat, sub, kernel, beta)
        assert torch.equal(obj.loss_aux, b.loss_aux.view(1))
        assert_same(a, b)
    assert torch.isfinite(obj.loss_aux).all()


@pytest.mark.parametrize("kind", ["gcn", "sage"])
def test_full_arxiv_shape_one_step_bitwise(kind):
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.cuda()
    perm = (ei[1] * n + ei[0]).argsort()
    adj = SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    x, y, t = ds.x.cuda(), ds.y.squeeze(1).cuda(), ds.teacher_logits.cuda()
    idx, t_feat = ds.split_idx["train"].cuda(), ds.teacher_feat.cuda()
    r, c, _ = adj.coo()
    sub = torch.from_numpy(og.subgraph(idx.cpu().numpy(), torch.stack([r, c]).cpu().numpy(), True)[0]).cuda()
    dims = (128, 256, 256, 40)
    a, obj, b = twins(kind, adj, dims, idx, t_feat, sub, "cosine", 100.0)
    assert t_feat.shape[1] == 750 and obj.E > 500_000
    a.train_step(x, y, idx, t)
    eager_step(b, x, y, idx, t, t_feat, sub, "cosine", 100.0)
    assert torch.equal(obj.loss_aux, b.loss_aux.view(1))
    assert_same(a, b)


@pytest.mark.parametrize("kind", ["gcn", "sage"])
def test_graph_replay_equals_eager_steps_bitwise(kind):
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat, sub = problem(dims=dims)
    oa, ob = (LSP(t_feat, idx, sub, 64, kernel="cosine", beta=100.0) for _ in range(2))
    a = ENGINES[kind](adj, list(dims), seed=1, lsp=oa)
    b = ENGINES[kind](adj, list(dims), seed=1, lsp=ob)
    eager = []
    for _ in range(3):
        eager.append((a.train_step(x, y, idx, t).clone(), oa.loss_aux.clone()))
    b.capture(x, y, idx, t, warmup=0)
    for k in range(3):
        got = b.replay().clone()
        assert torch.equal(got, eager[k][0]) and torch.equal(ob.loss_aux, eager[k][1]), k
    assert torch.equal(a.params, b.params) and torch.equal(a.exp_avg_sq, b.exp_avg_sq)
    if kind == "gcn":
        before = lib.launch_count()
        n_launch = b.launches_per_step()
        assert n_launch == lib.launch_count() - before > 0


def test_refusals():
    dims = (32, 64, 64, 8)
    adj, x, y, t, idx, t_feat, sub = problem(dims=dims)
    n = idx.numel()
    with pytest.raises(ValueError):
        LSP(t_feat, idx, sub[:, :0], 64)                                           # E = 0
    with pytest.raises(ValueError):
        LSP(t_feat, idx, torch.cat([sub, torch.tensor([[0], [n]], device="cuda")], 1), 64)   # a row >= n_train
    with pytest.raises(ValueError):
        LSP(t_feat, idx, torch.cat([sub, torch.tensor([[-1], [0]], device="cuda")], 1), 64)
    with pytest.raises(ValueError):
        LSP(t_feat, idx, sub, 64, kernel="gaussian")                               # unknown kernel
    with pytest.raises(ValueError):
        LSP(t_feat, idx, sub, lib.LSP_MAX_F + 4)                                   # wider than the kernel holds
    with pytest.raises(ValueError):
        LSP(t_feat, idx, sub, 0)
    obj = LSP(t_feat, idx, sub, 64)
    with pytest.raises(ValueError):                                                # both in-step objectives
        GCNStudentTrainer(adj, list(dims), lsp=obj, gcrd=GCRD(t_feat, idx, 64, proj_dim=64, max_samples=256))
    with pytest.raises(ValueError):                                                # built for another width
        SAGEStudentTrainer(adj, [32, 128, 128, 8], lsp=obj)
    for kind in ENGINES:
        tr = ENGINES[kind](adj, list(dims), lsp=LSP(t_feat, idx, sub, 64))
        with pytest.raises(ValueError):                                            # aux= together with an LSP
            tr.train_step(x, y, idx, t, aux=lambda f: f.sum())
        with pytest.raises(ValueError):                                            # LSP draws no sample
            tr.train_step(x, y, idx, t, sample=torch.arange(4))
