"""oracle/gsp.py reproduces tests/golden/gsp_arxiv.pt: one step of the reference's own train() with --training gpw
(gnn.py's CE + beta * gpw and gnn_kd_and_aux.py's KD + beta * gpw, GCN and SAGE, cosine at beta 10, rbf at beta 0.5 and l2,
dropout 0, the recorded numpy draw)."""
from pathlib import Path

import pytest
import torch

from oracle import graph as og, gsp as og_gsp

GOLD = Path(__file__).resolve().parent / "golden" / "gsp_arxiv.pt"
CASES = ["gnn_gcn_cosine", "gnn_sage_rbf", "kd_and_aux_gcn_rbf", "kd_and_aux_sage_cosine", "kd_and_aux_gcn_l2"]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def graph_of(gold, kind):
    r, c = gold["sym_row"].numpy(), gold["sym_col"].numpy()
    n = gold["x"].shape[0]
    if kind == "gcn":
        rr, cc, vv = og.gcn_norm(r, c, n)
        return torch.from_numpy(og.ind2ptr(rr, n)), torch.from_numpy(cc), torch.from_numpy(vv)
    return torch.from_numpy(og.ind2ptr(r, n)), torch.from_numpy(c), None


def student(name):
    return name.split("_")[-2]


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def pre_bn_bias(group, key):
    """Biases whose exact gradient is 0 (they sit in front of a training-mode BatchNorm): both sides carry rounding only,
    so Adam's first step (lr * g / |g|) moves them by a sign of noise."""
    if group == "model":
        return key.endswith("bias") and ("lin_l" in key or key.startswith("convs.")) and not key.startswith("convs.2")
    return key == "0.bias"


def test_fixture_covers_both_scripts_students_and_kernels(gold):
    assert sorted(gold["cases"]) == sorted(CASES)
    assert {(c["kernel"], c["beta"]) for c in gold["cases"].values()} == {("cosine", 10.0), ("rbf", 0.5), ("l2", 0.5)}
    n_train = gold["train_idx"].numel()
    for c in gold["cases"].values():
        assert gold["hp"]["S"] < n_train and c["draw"].unique().numel() == gold["hp"]["S"]


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_train_step(gold, name):
    case, hp = gold["cases"][name], gold["hp"]
    kind = student(name)
    rowptr, col, val = graph_of(gold, kind)
    ref = og_gsp.gsp_step(kind, gold["x"], rowptr, col, val, case["init"]["model"], case["init"]["sproj"], case["init"]["tproj"],
                          gold["y"], gold["train_idx"], gold["t_feat"], gold["t_logits"] if name.startswith("kd") else None,
                          case["draw"], case["kernel"], case["beta"], hp["alpha"], hp["kd_T"], lr=hp["lr"])
    assert abs(ref["loss"] - case["loss"]) < 1e-5 * abs(case["loss"])
    assert abs(ref["loss_cls"] - case["loss_cls"]) < 1e-5 * abs(case["loss_cls"])
    assert abs(ref["loss_aux"] - case["loss_aux"]) < 1e-5 * abs(case["loss_aux"])
    for group in ("model", "sproj", "tproj"):
        scale = max(g.abs().max().item() for g in case["grads"][group].values())
        for k, g in case["grads"][group].items():
            mine = ref["grads"][group][k]
            if pre_bn_bias(group, k):
                assert mine.abs().max().item() < 1e-9 * scale and g.abs().max().item() < 1e-5 * scale, (group, k)
            else:
                assert rel(mine, g) < 1e-5, (name, group, k, rel(mine, g))
        for k, v in case["after"][group].items():
            if "num_batches" in k or pre_bn_bias(group, k) or (group == "model" and "running" in k):
                continue
            assert rel(ref["after"][group][k], v) < 1e-5, (name, group, k)
