"""LSP in the R-GCN student step on GraphSAINT batches (``RGCNTrainer(..., lsp=BatchLSP(...)).train_step(b, x, teacher=t)``,
the reference's MAG ``--training lpw``): the train-induced edge list on the device, the teacher's eval forward on the
student's plan, the objective against the eager ``aux=`` path bit for bit and against the fp64 restatement oracle/mag_lsp.py,
and the refusals."""
from types import SimpleNamespace

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import criterion, lib, nn, ops, sampling
from efficient_gnns_b200.lsp import BatchLSP
from efficient_gnns_b200.rgcn import RGCNTrainer
from oracle import mag_lsp as om
from test_rgcn_train_gpu import NODES, batches, small_mag

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

KERNELS = ["cosine", "poly", "l2", "rbf"]
H, C, LR = 24, 7, 0.005


def student(rel, lsp=None, seed=3, p=0.5):
    return RGCNTrainer(16, H, C, 2, p, NODES, [0], len(rel), rel, lr=LR, seed=seed, lsp=lsp)


def teacher_of(rel, seed=11):
    return RGCNTrainer(16, 32, C, 3, 0.5, NODES, [0], len(rel), rel, lr=LR, seed=seed)


def reference_edges(mask, edge_index):
    return nn.subgraph(mask, edge_index, relabel_nodes=True)[0]


def state(tr):
    return ([tr.params, tr.exp_avg, tr.exp_avg_sq, tr.step_count] + [tr.emb[t] for t in sorted(tr.emb)]
            + [tr.emb_m[t] for t in sorted(tr.emb)] + [tr.emb_v[t] for t in sorted(tr.emb)])


def assert_same_state(a, b, what):
    for k, (x, y) in enumerate(zip(state(a), state(b))):
        assert torch.equal(x, y), (what, k)


# ------------------------------------------------------------------------------------------------ 1. edge builder
def test_induced_edges_equal_subgraph_on_sampled_batches():
    data, _, _ = small_mag(0)
    for b in batches(data, 4, seed=2):
        got = sampling.induced_edges(b.edge_index, b.train_mask)
        assert got.shape[1] > 0
        assert torch.equal(got, reference_edges(b.train_mask, b.edge_index))


def test_induced_edges_designed_cases():
    dev = "cuda"
    ei = torch.tensor([[0, 1, 2, 2, 3, 3, 5, 4, 1], [1, 2, 2, 0, 4, 4, 5, 0, 1]], device=dev)     # self-loops 2->2, 5->5, 1->1; 3->4 twice
    n = 6
    cases = {
        "no train rows": torch.zeros(n, dtype=torch.bool, device=dev),
        "train rows without induced edge": torch.tensor([1, 0, 0, 1, 0, 0], dtype=torch.bool, device=dev),
        "every node a train row": torch.ones(n, dtype=torch.bool, device=dev),
        "self-loops and a duplicate": torch.tensor([0, 1, 1, 1, 1, 1], dtype=torch.bool, device=dev),
    }
    for name, mask in cases.items():
        got = sampling.induced_edges(ei, mask)
        assert torch.equal(got, reference_edges(mask, ei)), name
    assert sampling.induced_edges(ei, cases["train rows without induced edge"]).shape == (2, 0)
    assert torch.equal(sampling.induced_edges(ei, cases["every node a train row"]), ei)
    # many tiles, every offset of the last one, a row pitch wider than the edge count
    g = torch.Generator(device=dev).manual_seed(0)
    for E in (1, 1023, 1024, 1025, 70_001):
        big = torch.randint(0, 3000, (2, E + 7), generator=g, device=dev)[:, :E]
        mask = torch.rand(3000, generator=g, device=dev) < 0.4
        assert torch.equal(sampling.induced_edges(big, mask), reference_edges(mask, big)), E
    assert sampling.induced_edges(ei[:, :0], cases["every node a train row"]).shape == (2, 0)
    with pytest.raises(lib.B200GnnError, match="outside"):
        sampling.induced_edges(torch.tensor([[0, 6], [1, 1]], device=dev), cases["every node a train row"])


def test_train_rows_keep_their_rank_in_internal_order():
    """All train rows are papers and BatchPlan sorts types stably, so their internal rows ascend with their batch ids."""
    data, _, rel = small_mag(0)
    tr = student(rel)
    for b in batches(data, 3):
        P = tr.plan(b)
        rows = P.pos[b.train_mask.nonzero().view(-1)]
        assert bool((rows[1:] > rows[:-1]).all())


# ------------------------------------------------------------------------------------------------ 2. teacher in the step
def test_teacher_in_the_step_equals_teacher_logits_bit_for_bit():
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    a, b_ = student(rel), student(rel)
    t_params = t.params.clone()
    for step, b in enumerate(batches(data, 3, seed=5)):
        la = a.train_step(b, x, teacher=t).clone()
        tl = t.forward(b, x, training=False)[b.train_mask]
        lb = b_.train_step(b, x, teacher_logits=tl).clone()
        assert torch.equal(la, lb), step
        assert_same_state(a, b_, step)
    assert torch.equal(t.params, t_params) and int(t.step_count) == 0


# ------------------------------------------------------------------------------------------------ 3. LSP vs the eager path
@pytest.mark.parametrize("kernel", KERNELS)
def test_lsp_step_equals_the_eager_aux_step_bit_for_bit(kernel):
    data, x, rel = small_mag(1)
    beta = 10.0
    t = teacher_of(rel)
    fused = student(rel, lsp=BatchLSP(H, kernel, beta))
    eager = student(rel)
    for step, b in enumerate(batches(data, 3, seed=5)):
        lf = fused.train_step(b, x, teacher=t).clone()
        tl = t.forward(b, x, training=False)[b.train_mask]
        t_feat = t.out_feat()
        tm = b.train_mask
        ei = reference_edges(tm, b.edge_index)
        dummy = torch.zeros(int(tm.sum()), 2, device="cuda"), torch.zeros(int(tm.sum()), dtype=torch.long, device="cuda")
        le = eager.train_step(b, x, teacher_logits=tl, beta=beta, aux=lambda f: criterion.lpw_criterion(
            *dummy, f[tm], t_feat[tm], ei, kernel, 1)[2]).clone()
        assert torch.equal(fused.lsp.edge_index, ei), step
        assert torch.equal(lf[:2], le[:2]) and torch.equal(lf[2:], eager.loss_aux.view(1)), (step, lf, le, eager.loss_aux)
        assert_same_state(fused, eager, step)


def test_a_batch_without_induced_edge_is_nan_and_steps_as_kd():
    """The reference's kl_div mean over no term is NaN (tests/golden/mag_lsp.pt, case no_edge): loss and loss_aux are NaN
    and the step is the KD step."""
    data, x, rel = small_mag(1)
    t = teacher_of(rel)
    fused, kd = student(rel, lsp=BatchLSP(H, "rbf", 1.0)), student(rel)
    b = batches(data, 1, seed=5)[0]
    paper = ((b.node_type == 0) & ~b.train_mask).nonzero().view(-1)
    src, dst = b.edge_index
    lone = next(int(v) for v in paper if not bool(((src == v) & (dst == v)).any()))
    b.train_mask = torch.zeros_like(b.train_mask)
    b.train_mask[lone] = True
    lf = fused.train_step(b, x, teacher=t).clone()
    lk = kd.train_step(b, x, teacher=t).clone()
    assert fused.lsp.edge_index.shape == (2, 0)
    assert torch.isnan(lf[0]) and torch.isnan(lf[2]) and torch.equal(lf[1], lk[1])
    assert_same_state(fused, kd, "no edge")


# ------------------------------------------------------------------------------------------------ 4. fp64 oracle
@pytest.mark.parametrize("kernel", KERNELS)
def test_three_lsp_steps_match_the_fp64_oracle(kernel):
    data, x, rel = small_mag(1)
    p, L, beta = 0.5, 2, 10.0
    t = teacher_of(rel)
    tr = student(rel, lsp=BatchLSP(H, kernel, beta))
    # the oracle runs on the CPU (its segment softmax builds host tensors)
    params = {k: v.double().cpu().requires_grad_(True) for k, v in tr.state_dict().items()}
    teacher = {k: v.double().cpu() for k, v in t.state_dict().items()}
    x_cpu = {k: v.cpu() for k, v in x.items()}
    opt = torch.optim.Adam(list(params.values()), lr=LR)
    for step, b in enumerate(batches(data, 3, seed=5)):
        loss = tr.train_step(b, x, teacher=t).clone()
        n = b.node_type.numel()
        masks = [ops.dropout_mask(n, H, p, tr.seed, l + step * L).bool().cpu() for l in range(L - 1)]
        cb = SimpleNamespace(**{k: getattr(b, k).cpu() for k in ("edge_index", "edge_attr", "node_type", "local_node_idx", "y",
                                                                 "train_mask")})
        ref, ref_cls, ref_aux = om.lpw_step_loss(params, teacher, x_cpu, cb, masks, kernel, beta)
        opt.zero_grad()
        ref.backward()
        opt.step()
        for got, want in ((loss[0], ref), (loss[1], ref_cls), (loss[2], ref_aux)):
            assert abs(float(got) - float(want)) <= 1e-5 * max(1.0, abs(float(want))), (step, loss, ref, ref_aux)
    sd = tr.state_dict()
    for k, v in params.items():
        assert rel_err(sd[k], v) < 5e-5, k


# ------------------------------------------------------------------------------------------------ 5. validation
def test_refusals_do_no_device_work():
    data, x, rel = small_mag(1)
    b = batches(data, 1, seed=5)[0]
    t = teacher_of(rel)
    tr = student(rel, lsp=BatchLSP(H, "rbf"))
    plain = student(rel)
    other_rel = dict(rel)
    other_rel[0] = (rel[0][0], (rel[0][1] + 1) % 4)
    other_nodes = dict(NODES)
    other_nodes[3] += 1
    bad_teachers = {
        "relations": teacher_of(other_rel),
        "types": RGCNTrainer(16, 32, C, 3, 0.5, other_nodes, [0], len(rel), rel, seed=11),
        "input width": RGCNTrainer(20, 32, C, 3, 0.5, NODES, [0], len(rel), rel, seed=11),
    }
    torch.cuda.synchronize()
    before = (lib.launch_count(), tr.params.clone(), int(tr.step_count))
    with pytest.raises(ValueError, match="teacher="):
        tr.train_step(b, x)
    with pytest.raises(ValueError, match="aux="):
        tr.train_step(b, x, teacher=t, aux=lambda f: f.sum())
    with pytest.raises(ValueError, match="two teachers"):
        plain.train_step(b, x, teacher=t, teacher_logits=torch.zeros(int(b.train_mask.sum()), C, device="cuda"))
    for what, bad in bad_teachers.items():
        with pytest.raises(ValueError, match=what):
            tr.train_step(b, x, teacher=bad)
        with pytest.raises(ValueError, match=what):
            plain.train_step(b, x, teacher=bad)
    with pytest.raises(ValueError, match="kernel"):
        BatchLSP(H, "gauss")
    with pytest.raises(ValueError, match="hidden width"):
        BatchLSP(lib.LSP_MAX_F + 4)
    with pytest.raises(ValueError, match="hidden width"):
        student(rel, lsp=BatchLSP(H + 8))
    assert lib.launch_count() == before[0]
    assert torch.equal(tr.params, before[1]) and int(tr.step_count) == before[2]
