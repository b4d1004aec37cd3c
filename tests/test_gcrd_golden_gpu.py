"""The captured G-CRD step against the reference and the fp64 oracle: the engine with the recorded numpy sample reproduces
one step of the reference's own train() (tests/golden/gcrd_arxiv.pt: gnn.py's CE + beta * nce and gnn_kd_and_aux.py's
KD + beta * nce, GCN and SAGE, dropout 0); the engine with its own on-device sample and dropout masks (p = 0.5) matches
oracle/gcrd.py; and the GAT teacher's saved features/ and logits/ files feed the G-CRD student unchanged."""
from pathlib import Path

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import ops
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_gat_teacher import GATTeacherTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.gcrd import GCRD
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import gcrd as og_gcrd, graph as og

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}
CASES = ["gnn_gcn", "gnn_sage", "kd_and_aux_gcn", "kd_and_aux_sage"]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN / "gcrd_arxiv.pt", weights_only=False)


def model_grads(tr):
    """reference key -> engine gradient (both use the reference module's layouts)."""
    out = {}
    for l in range(tr.L):
        if isinstance(tr, GCNStudentTrainer):
            out[f"convs.{l}.weight"], out[f"convs.{l}.bias"] = tr.gW[l], tr.gb[l]
        else:
            out[f"convs.{l}.lin_l.weight"], out[f"convs.{l}.lin_l.bias"] = tr.gWl[l], tr.gbl[l]
            out[f"convs.{l}.lin_r.weight"] = tr.gWr[l]
        if l < tr.L - 1:
            out[f"bns.{l}.weight"], out[f"bns.{l}.bias"] = tr.ggamma[l], tr.gbeta[l]
    return out


def head_grads(h, which):
    if which == "sproj":
        return {"0.weight": h.gW_s, "0.bias": h.gb_s, "1.weight": h.ggamma_s, "1.bias": h.gbeta_s}
    return {"0.weight": h.gW_t[:, :h.F_t], "0.bias": h.gb_t, "1.weight": h.ggamma_t, "1.bias": h.gbeta_t}


def pre_bn_bias(group, key, L):
    """Biases in front of a training-mode BatchNorm: exact gradient 0, both sides carry rounding only (and Adam's first
    step, lr * g / |g|, moves them by a sign of that noise)."""
    if group == "model":
        return key.endswith("bias") and key.startswith("convs.") and not key.startswith(f"convs.{L - 1}.")
    return key == "0.bias"


def compare(tr, head, ref, tol=1e-4):
    """Engine gradients vs reference gradients (dicts under the reference's keys)."""
    got = {"model": model_grads(tr), "sproj": head_grads(head, "sproj"), "tproj": head_grads(head, "tproj")}
    for group in got:
        scale = max(g.abs().max().item() for g in ref[group].values())
        for k, g in ref[group].items():
            a = got[group][k]
            if pre_bn_bias(group, k, tr.L):
                assert a.abs().max().item() < 1e-5 * scale, (group, k)
            else:
                assert rel_err(a, g.float()) < tol, (group, k, rel_err(a, g.float()))


def adj_of(row, col, n):
    return SparseTensor(row=row.cuda(), col=col.cuda(), sparse_sizes=(n, n), is_sorted=True)


@pytest.mark.parametrize("name", CASES)
def test_engine_with_the_recorded_sample_reproduces_the_reference(gold, name):
    case, hp = gold["cases"][name], gold["hp"]
    kind = name.rsplit("_", 1)[1]
    x, y, idx, n = gold["x"].cuda(), gold["y"].cuda(), gold["train_idx"].cuda(), gold["x"].shape[0]
    C = gold["t_logits"].shape[1]
    head = GCRD(gold["t_feat"].cuda(), idx, hp["hidden"], proj_dim=hp["proj"], max_samples=hp["S"], nce_T=hp["nce_T"],
                beta=hp["beta"])
    dims = [x.shape[1]] + [hp["hidden"]] * (hp["layers"] - 1) + [C]
    tr = ENGINES[kind](adj_of(gold["sym_row"], gold["sym_col"], n), dims, dropout=0.0, lr=hp["lr"], gcrd=head)
    tr.load_state_dict({k: v.cuda() for k, v in case["init"]["model"].items()})
    head.load_student_proj_state_dict(case["init"]["sproj"])
    head.load_teacher_proj_state_dict(case["init"]["tproj"])
    t = gold["t_logits"].cuda() if name.startswith("kd") else None
    loss = tr.train_step(x, y, idx, t, sample=case["draw"]).cpu()
    assert abs(float(loss[0]) - case["loss"]) < 2e-5 * abs(case["loss"])
    assert abs(float(loss[1]) - case["loss_cls"]) < 2e-5 * abs(case["loss_cls"])
    assert abs(float(head.loss_aux) - case["loss_aux"]) < 2e-5 * abs(case["loss_aux"])
    compare(tr, head, case["grads"])
    after = {"model": tr.state_dict(), "sproj": head.student_proj_state_dict(), "tproj": head.teacher_proj_state_dict()}
    for group, ref in case["after"].items():
        for k, v in ref.items():
            if "num_batches" in k:
                if group != "model":                                    # the engine's student keeps no BN batch counter
                    assert int(after[group][k]) == int(v), (group, k)
            elif pre_bn_bias(group, k, tr.L):
                continue                                                # its step is the sign of rounding noise
            elif k in case["grads"][group]:
                # Adam's first step moves every parameter by lr * g / (|g| + eps): where |g| is at the level of the
                # gradients' rounding its sign is noise, so the step is compared where the gradient is clearly nonzero
                g = case["grads"][group][k]
                keep = g.abs() > 1e-2 * g.abs().max()
                if keep.any():
                    assert rel_err(after[group][k].cpu()[keep], v[keep].float()) < 1e-5, (group, k)
            else:                                                       # running statistics
                assert rel_err(after[group][k], v.float()) < 1e-5, (group, k)


def problem(n=3000, e=20_000, dims=(32, 64, 64, 8), seed=0, f_t=90):
    ei = skewed_edges(n, e, seed)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    g = torch.Generator().manual_seed(seed + 9)
    x = torch.randn(n, dims[0], generator=g)
    y = torch.randint(0, dims[-1], (n,), generator=g)
    t = torch.randn(n, dims[-1], generator=g) * 2
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values
    t_feat = torch.randn(n, f_t, generator=g).relu()
    return r, c, x, y, t, idx, t_feat


@pytest.mark.parametrize("kind", ["gcn", "sage"])
@pytest.mark.parametrize("S", [256, 100_000])
@pytest.mark.parametrize("form", ["kd", "supervised"])
def test_engine_matches_fp64_oracle_with_its_own_sample_and_masks(kind, S, form):
    dims, p, beta, nce_T = (32, 64, 64, 8), 0.5, 0.5, 0.075
    r, c, x, y, t, idx, t_feat = problem(dims=dims)
    n = x.shape[0]
    head = GCRD(t_feat.cuda(), idx.cuda(), dims[-2], proj_dim=64, max_samples=S, nce_T=nce_T, beta=beta, seed=3)
    tr = ENGINES[kind](adj_of(torch.from_numpy(r), torch.from_numpy(c), n), list(dims), dropout=p, lr=0.01, seed=0, gcrd=head)
    init = (tr.state_dict(), head.student_proj_state_dict(), head.teacher_proj_state_dict())
    masks = [ops.dropout_mask(n, dims[l + 1], p, tr.seed, tr.dropout_offset(l, 0)).cpu().bool() for l in range(tr.L - 1)]
    teacher = t if form == "kd" else None
    loss = tr.train_step(x.cuda(), y.cuda(), idx.cuda(), None if teacher is None else teacher.cuda()).cpu()
    sample = head.sample().cpu()
    if S < idx.numel():
        assert sample.unique().numel() == S and int(sample.min()) >= 0 and int(sample.max()) < idx.numel()
    if kind == "gcn":
        rr, cc, vv = og.gcn_norm(r, c, n)
        rowptr, col, val = torch.from_numpy(og.ind2ptr(rr, n)), torch.from_numpy(cc), torch.from_numpy(vv)
    else:
        rowptr, col, val = torch.from_numpy(og.ind2ptr(r, n)), torch.from_numpy(c), None
    cpu = lambda sd: {k: v.cpu() for k, v in sd.items()}
    ref = og_gcrd.gcrd_step(kind, x, rowptr, col, val, cpu(init[0]), cpu(init[1]), cpu(init[2]), y, idx, t_feat, teacher, sample, beta,
                            nce_T, masks=masks, p=p)
    assert abs(float(loss[0]) - ref["loss"]) < 2e-5 * abs(ref["loss"])
    assert abs(float(head.loss_aux) - ref["loss_aux"]) < 2e-5 * abs(ref["loss_aux"])
    compare(tr, head, ref["grads"])


def test_gat_teacher_artefacts_feed_the_gcrd_student(tmp_path):
    g = torch.load(GOLDEN / "gat_teacher_arxiv.pt", weights_only=False)
    n, C = g["x"].shape[0], g["n_classes"]
    adj = adj_of(g["row"].long(), g["col"].long(), n)
    splits = {"train": g["train_idx"], "valid": g["val_idx"], "test": g["test_idx"]}
    teacher = GATTeacherTrainer(adj, g["x"].cuda(), g["y"].cuda(), splits, n_classes=C, n_hidden=g["n_hidden"],
                                n_layers=g["n_layers"], n_heads=g["n_heads"], dropout=0.0, input_drop=0.0, edge_drop=0.0)
    teacher.epoch()
    paths = teacher.save(tmp_path, "gat-3L10x3h", 0)
    feat = torch.load(paths["features"]).cuda()                    # what gnn.py:277-278 loads
    logits = torch.load(paths["logits"]).cuda()
    idx = g["train_idx"].cuda()
    head = GCRD(feat, idx, 32, proj_dim=64, max_samples=128, beta=0.5)
    tr = GCNStudentTrainer(adj, [g["x"].shape[1], 32, 32, C], dropout=0.5, lr=0.01, gcrd=head)
    assert torch.equal(head.G_t[:, :feat.shape[1]], feat[idx]) and not head.G_t[:, feat.shape[1]:].any()
    loss = tr.train_step(g["x"].cuda(), g["y"].view(-1).cuda(), idx, logits).clone()
    assert torch.isfinite(loss).all() and float(loss[2]) > 0 and float(head.loss_aux) > 0
