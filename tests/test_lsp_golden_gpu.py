"""The captured LSP step against the reference: the engine reproduces one step of the reference's own train() with
--training lpw (tests/golden/lsp_arxiv.pt: gnn.py's CE + beta * lpw and gnn_kd_and_aux.py's KD + beta * lpw, GCN and SAGE,
cosine at beta 100 and rbf at beta 0.5, dropout 0, a 90-wide teacher)."""
from pathlib import Path

import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200.engine import GCNStudentTrainer
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
from efficient_gnns_b200.lsp import LSP
from efficient_gnns_b200.sparse import SparseTensor

pytestmark = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / "golden" / "lsp_arxiv.pt"
ENGINES = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}
CASES = [f"{s}_{k}_{ker}" for s in ("gnn", "kd_and_aux") for k in ("gcn", "sage") for ker in ("cosine", "rbf")]


@pytest.fixture(scope="module")
def gold():
    return torch.load(GOLD, weights_only=False)


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


def pre_bn_bias(key, L):
    """Biases in front of a training-mode BatchNorm: exact gradient 0, both sides carry rounding only (and Adam's first
    step, lr * g / |g|, moves them by a sign of that noise)."""
    return key.endswith("bias") and key.startswith("convs.") and not key.startswith(f"convs.{L - 1}.")


@pytest.mark.parametrize("name", CASES)
def test_engine_reproduces_the_reference_train_step(gold, name):
    case, hp = gold["cases"][name], gold["hp"]
    kind, kernel = name.split("_")[-2:]
    x, y, idx, n = gold["x"].cuda(), gold["y"].cuda(), gold["train_idx"].cuda(), gold["x"].shape[0]
    C = gold["t_logits"].shape[1]
    obj = LSP(gold["t_feat"].cuda(), idx, gold["edge_index"].cuda(), hp["hidden"], kernel=kernel, beta=case["beta"])
    dims = [x.shape[1]] + [hp["hidden"]] * (hp["layers"] - 1) + [C]
    adj = SparseTensor(row=gold["sym_row"].cuda(), col=gold["sym_col"].cuda(), sparse_sizes=(n, n), is_sorted=True)
    tr = ENGINES[kind](adj, dims, dropout=0.0, lr=hp["lr"], lsp=obj)
    tr.load_state_dict({k: v.cuda() for k, v in case["init"].items()})
    t = gold["t_logits"].cuda() if name.startswith("kd") else None
    loss = tr.train_step(x, y, idx, t).cpu()
    assert abs(float(loss[0]) - case["loss"]) < 2e-5 * abs(case["loss"])
    assert abs(float(loss[1]) - case["loss_cls"]) < 2e-5 * abs(case["loss_cls"])
    # the KL's per-edge terms cancel to a small sum: its rounding is relative to the terms, not to the result
    assert abs(float(obj.loss_aux) - case["loss_aux"]) < 2e-5 * abs(case["loss_aux"]) + 2e-8
    got = model_grads(tr)
    scale = max(g.abs().max().item() for g in case["grads"].values())
    for k, g in case["grads"].items():
        if pre_bn_bias(k, tr.L):
            assert got[k].abs().max().item() < 1e-5 * scale, k
        else:
            assert rel_err(got[k], g.float()) < 1e-4, (k, rel_err(got[k], g.float()))
    after = tr.state_dict()
    for k, v in case["after"].items():
        if "num_batches" in k or pre_bn_bias(k, tr.L):
            continue
        if k in case["grads"]:
            # Adam's first step moves every parameter by lr * g / (|g| + eps): where |g| is at the level of the
            # gradients' rounding its sign is noise, so the step is compared where the gradient is clearly nonzero
            g = case["grads"][k]
            keep = g.abs() > 1e-2 * g.abs().max()
            if keep.any():
                assert rel_err(after[k].cpu()[keep], v[keep].float()) < 1e-5, k
        else:                                                           # running statistics
            assert rel_err(after[k], v.float()) < 1e-5, k
