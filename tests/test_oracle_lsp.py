"""The fp64 oracle reproduces tests/golden/lsp_arxiv.pt: one step of the reference's own train() with --training lpw
(gnn.py's CE + beta * lpw and gnn_kd_and_aux.py's KD + beta * lpw, GCN and SAGE, cosine and rbf, dropout 0)."""
from pathlib import Path

import pytest
import torch

from oracle import criterion as oc, graph as og, nn as onn

GOLD = Path(__file__).resolve().parent / "golden" / "lsp_arxiv.pt"
CASES = [f"{s}_{k}_{ker}" for s in ("gnn", "kd_and_aux") for k in ("gcn", "sage") for ker in ("cosine", "rbf")]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


def lsp_step(gold, name):
    """fp64 restatement of the recorded step: forward, CE or KD + beta * lpw_criterion, autograd, Adam's first step."""
    case, hp = gold["cases"][name], gold["hp"]
    kind, kernel = name.split("_")[-2:]
    r, c = gold["sym_row"].numpy(), gold["sym_col"].numpy()
    n = gold["x"].shape[0]
    m = {k: v.double().clone().requires_grad_(v.is_floating_point() and "running" not in k)
         for k, v in case["init"].items() if "num_batches" not in k}
    L = hp["layers"]
    ga, be = [m[f"bns.{i}.weight"] for i in range(L - 1)], [m[f"bns.{i}.bias"] for i in range(L - 1)]
    x = gold["x"].double()
    if kind == "gcn":
        rr, cc, vv = og.gcn_norm(r, c, n)
        logits, hid = onn.gcn_forward(x, torch.from_numpy(og.ind2ptr(rr, n)), torch.from_numpy(cc), torch.from_numpy(vv),
                                      [m[f"convs.{i}.weight"] for i in range(L)], [m[f"convs.{i}.bias"] for i in range(L)],
                                      ga, be, None)
    else:
        params = [dict(w_l=m[f"convs.{i}.lin_l.weight"], b_l=m[f"convs.{i}.lin_l.bias"], w_r=m[f"convs.{i}.lin_r.weight"])
                  for i in range(L)]
        logits, hid = onn.sage_forward(x, torch.from_numpy(og.ind2ptr(r, n)), torch.from_numpy(c), params, ga, be, None)
    idx = gold["train_idx"]
    z, lab = logits[idx], gold["y"][idx]
    if name.startswith("gnn"):
        loss_main = loss_cls = oc.cross_entropy(z, lab)
    else:
        loss_main, loss_cls, _ = oc.kd_criterion(z, lab, gold["t_logits"][idx].double(), hp["alpha"], hp["kd_T"])
    _, _, loss_aux = oc.lpw_criterion(z, lab, hid[idx], gold["t_feat"][idx].double(), gold["edge_index"], kernel, case["beta"])
    loss = loss_main + case["beta"] * loss_aux
    leaves = [(k, v) for k, v in m.items() if v.requires_grad]
    gr = torch.autograd.grad(loss, [v for _, v in leaves])
    grads = {k: g for (k, _), g in zip(leaves, gr)}
    after = {k: v.detach() - hp["lr"] * grads[k] / (grads[k].abs() + 1e-8) for k, v in leaves}   # Adam step 1
    return dict(loss=float(loss.detach()), loss_cls=float(loss_cls.detach()), loss_aux=float(loss_aux.detach()), grads=grads,
                after=after)


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def pre_bn_bias(key, layers):
    """Biases in front of a training-mode BatchNorm: their exact gradient is 0, both sides carry rounding only, so Adam's
    first step (lr * g / |g|) moves them by a sign of noise."""
    return key.endswith("bias") and key.startswith("convs.") and not key.startswith(f"convs.{layers - 1}.")


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_train_step(gold, name):
    case = gold["cases"][name]
    ref = lsp_step(gold, name)
    for k in ("loss", "loss_cls"):
        assert abs(ref[k] - case[k]) < 1e-5 * abs(case[k]), (k, ref[k], case[k])
    # the fp32 KL is a mean of per-edge terms pt * (log pt - log ps) that cancel to a small sum: its rounding is relative to
    # the terms (|log p| ~ log deg), not to the result, which is 6e-5 for rbf
    assert abs(ref["loss_aux"] - case["loss_aux"]) < 1e-5 * abs(case["loss_aux"]) + 1e-8, (ref["loss_aux"], case["loss_aux"])
    L = gold["hp"]["layers"]
    scale = max(g.abs().max().item() for g in case["grads"].values())
    for k, g in case["grads"].items():
        mine = ref["grads"][k]
        if pre_bn_bias(k, L):
            assert mine.abs().max().item() < 1e-9 * scale and g.abs().max().item() < 1e-5 * scale, k
        else:
            assert rel(mine, g) < 1e-5, (name, k, rel(mine, g))
    for k, v in case["after"].items():
        if "running" in k or "num_batches" in k or pre_bn_bias(k, L):
            continue
        assert rel(ref["after"][k], v) < 1e-5, (name, k)


def test_the_fixture_covers_the_lsp_term():
    """The cosine cases carry an LSP term that moves the gradients: without it the oracle's gradients differ."""
    gold = torch.load(GOLD, weights_only=False)
    case = gold["cases"]["gnn_gcn_cosine"]
    assert case["loss_aux"] > 0 and gold["t_feat"].shape[1] % 4 != 0
    no_aux = dict(gold, cases=dict(gold["cases"], gnn_gcn_cosine=dict(case, beta=0.0)))
    g0 = lsp_step(no_aux, "gnn_gcn_cosine")["grads"]["convs.0.weight"]
    assert rel(g0, case["grads"]["convs.0.weight"]) > 1e-3
