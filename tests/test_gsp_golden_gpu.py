"""The captured GSP step against the reference: the engine with the recorded numpy sample reproduces one step of the
reference's own train() (tests/golden/gsp_arxiv.pt: gnn.py's CE + beta * gpw and gnn_kd_and_aux.py's KD + beta * gpw, GCN
and SAGE, cosine at beta 10, rbf at beta 0.5 and l2, dropout 0): losses, every gradient, the state after Adam and the
running statistics."""
from pathlib import Path

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.gsp import GSP
from efficient_gnns_b200.sparse import SparseTensor

pytestmark = pytest.mark.gpu

GOLDEN = Path(__file__).resolve().parent / "golden"
ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}
CASES = ["gnn_gcn_cosine", "gnn_sage_rbf", "kd_and_aux_gcn_rbf", "kd_and_aux_sage_cosine", "kd_and_aux_gcn_l2"]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLDEN / "gsp_arxiv.pt", weights_only=False)


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


@pytest.mark.parametrize("name", CASES)
def test_engine_with_the_recorded_sample_reproduces_the_reference(gold, name):
    case, hp = gold["cases"][name], gold["hp"]
    kind = name.split("_")[-2]
    x, y, idx, n = gold["x"].cuda(), gold["y"].cuda(), gold["train_idx"].cuda(), gold["x"].shape[0]
    C = gold["t_logits"].shape[1]
    head = GSP(gold["t_feat"].cuda(), idx, hp["hidden"], proj_dim=hp["proj"], max_samples=hp["S"], kernel=case["kernel"],
               beta=case["beta"])
    dims = [x.shape[1]] + [hp["hidden"]] * (hp["layers"] - 1) + [C]
    adj = SparseTensor(row=gold["sym_row"].cuda(), col=gold["sym_col"].cuda(), sparse_sizes=(n, n), is_sorted=True)
    tr = ENGINES[kind](adj, dims, dropout=0.0, lr=hp["lr"], gsp=head)
    tr.load_state_dict({k: v.cuda() for k, v in case["init"]["model"].items()})
    head.load_student_proj_state_dict(case["init"]["sproj"])
    head.load_teacher_proj_state_dict(case["init"]["tproj"])
    t = gold["t_logits"].cuda() if name.startswith("kd") else None
    loss = tr.train_step(x, y, idx, t, sample=case["draw"]).cpu()
    assert abs(float(loss[0]) - case["loss"]) < 2e-5 * abs(case["loss"])
    assert abs(float(loss[1]) - case["loss_cls"]) < 2e-5 * abs(case["loss_cls"])
    assert abs(float(head.loss_aux) - case["loss_aux"]) < 2e-5 * abs(case["loss_aux"])
    got = {"model": model_grads(tr), "sproj": head_grads(head, "sproj"), "tproj": head_grads(head, "tproj")}
    for group, ref in case["grads"].items():
        scale = max(g.abs().max().item() for g in ref.values())
        for k, g in ref.items():
            a = got[group][k]
            if pre_bn_bias(group, k, tr.L):
                assert a.abs().max().item() < 1e-5 * scale, (group, k)
            else:
                assert rel_err(a, g.float()) < 1e-4, (group, k, rel_err(a, g.float()))
    after = {"model": tr.state_dict(), "sproj": head.student_proj_state_dict(), "tproj": head.teacher_proj_state_dict()}
    for group, ref in case["after"].items():
        for k, v in ref.items():
            if "num_batches" in k:
                if group != "model":                                    # the engine's student keeps no BN batch counter
                    assert int(after[group][k]) == int(v), (group, k)
            elif pre_bn_bias(group, k, tr.L):
                continue                                                # its step is the sign of rounding noise
            elif k in case["grads"][group]:
                # Adam's first step moves every parameter by lr * g / (|g| + eps): compared where the gradient is clearly
                # nonzero, since where |g| is at the level of rounding its sign is noise
                g = case["grads"][group][k]
                keep = g.abs() > 1e-2 * g.abs().max()
                if keep.any():
                    assert rel_err(after[group][k].cpu()[keep], v[keep].float()) < 1e-5, (group, k)
            else:                                                       # running statistics
                assert rel_err(after[group][k], v.float()) < 1e-5, (group, k)
