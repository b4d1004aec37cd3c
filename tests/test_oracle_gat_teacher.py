"""oracle/gat_teacher.py reproduces the reference's own gat.py (tests/golden/gat_teacher_arxiv.pt): per epoch the training
loss and accuracy, the RMSprop parameters and square_avg, the BatchNorm running statistics, and evaluate()'s losses,
accuracies, prediction and ``feat``.  Each epoch starts the fp64 oracle from the fixture's state after the previous one: an
RMSprop step moves an entry by about 10 lr_t times the sign of its gradient, so free-running trajectories need not agree
elementwise."""
from pathlib import Path

import pytest
import torch

from oracle import gat_teacher as ot

GOLDEN = Path(__file__).resolve().parent / "golden"


@pytest.fixture(scope="module")
def gold():
    g = torch.load(GOLDEN / "gat_teacher_arxiv.pt", weights_only=False)
    g["row"], g["col"] = g["row"].long(), g["col"].long()                # stored as int32
    return g


def rel(a, b):
    a, b = a.detach().double(), b.detach().double()
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("case", ["labels", "no_labels"])
def test_oracle_reproduces_the_reference_recipe(gold, case):
    c = gold["cases"][case]
    use_labels, iters = case == "labels", 1 if case == "labels" else 0
    x, y = gold["x"].double(), gold["y"]
    row, col = gold["row"], gold["col"]
    tr, va, te = gold["train_idx"], gold["val_idx"], gold["test_idx"]
    L, H, C = gold["n_layers"], gold["n_heads"], gold["n_classes"]
    names = c["names"]
    assert names[:4] == ["convs.0.attn_l", "convs.0.fc.weight", "convs.0.res_fc.weight", "convs.1.attn_l"]
    prev = {k: v for k, v in c["state0"].items()}
    prev_sq = {k: torch.zeros_like(v) for k, v in prev.items() if k in names}
    for e, ep in enumerate(c["epochs"], start=1):
        assert ep["lr"] == ot.lr_at(0.002, e)
        state = {k: v.double().clone().requires_grad_(k in names) for k, v in prev.items() if "num_batches" not in k}
        acc, loss, _, _ = ot.train(x, y, row, col, tr, va, te, state, L, H, C, use_labels, iters, ep["mask"])
        assert abs(loss.item() - ep["loss"]) <= 1e-5 * abs(ep["loss"]) and abs(acc.item() - ep["acc"]) <= 1e-6
        for k, v in ep["running"].items():
            if "running" in k:
                assert rel(state[k], v) <= 1e-5, k
            else:
                assert int(v) == e * (iters + 1), k                            # one batch per training forward
        params = [state[k] for k in names]
        sq = [prev_sq[k].double().clone() for k in names]
        ot.rmsprop_step(params, [p.grad for p in params], sq, ep["lr"])
        lr_t = ep["lr"]
        for k, p, s in zip(names, params, sq):
            upd, upd_ref = p.detach() - prev[k].double(), ep["params"][k].double() - prev[k].double()
            assert (upd - upd_ref).abs().max().item() <= 20 * lr_t, k          # bounded by two sign flips
            assert (upd - upd_ref).norm().item() <= 2e-3 * upd_ref.norm().item() + 1e-12, k
            assert (s - ep["square_avg"][k].double()).norm().item() <= 1e-3 * ep["square_avg"][k].double().norm().item(), k
        # evaluate() at the fixture's state after this step
        st = {k: v.double() for k, v in ep["params"].items()}
        st.update({k: v.double() for k, v in ep["running"].items() if "running" in k})
        accs, losses, pred, feat = ot.evaluate(x, y, row, col, tr, va, te, st, L, H, C, use_labels, iters)
        for a, k in zip(accs, ("train_acc", "val_acc", "test_acc")):
            assert abs(a.item() - ep[k]) <= 1e-6, k          # fp32 means of counts: exact to one row
        for lo, k in zip(losses, ("train_loss", "val_loss", "test_loss")):
            assert abs(lo.item() - ep[k]) <= 1e-5 * abs(ep[k]), k
        if ep["pred"] is not None:                                       # kept for the last epoch
            assert rel(pred, ep["pred"]) <= 1e-5 and rel(feat, ep["feat"]) <= 1e-5
        prev = {**ep["params"], **ep["running"]}
        prev_sq = ep["square_avg"]
