"""oracle/gcrd.py reproduces tests/golden/gcrd_arxiv.pt: one step of the reference's own train() with --training nce
(gnn.py's CE + beta * nce and gnn_kd_and_aux.py's KD + beta * nce, GCN and SAGE, dropout 0, the recorded numpy draw)."""
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import gcrd as og_gcrd, graph as og
from oracle.sampling import philox4x32

GOLD = Path(__file__).resolve().parent / "golden" / "gcrd_arxiv.pt"
CASES = ["gnn_gcn", "gnn_sage", "kd_and_aux_gcn", "kd_and_aux_sage"]


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


def oracle_case(gold, name, masks=None, p=0.0, sample=None):
    case, hp = gold["cases"][name], gold["hp"]
    kind = name.rsplit("_", 1)[1]
    rowptr, col, val = graph_of(gold, kind)
    return og_gcrd.gcrd_step(kind, gold["x"], rowptr, col, val, case["init"]["model"], case["init"]["sproj"],
                             case["init"]["tproj"], gold["y"], gold["train_idx"], gold["t_feat"],
                             gold["t_logits"] if name.startswith("kd") else None,
                             case["draw"] if sample is None else sample, hp["beta"], hp["nce_T"], hp["alpha"], hp["kd_T"],
                             masks=masks, p=p, lr=hp["lr"])


def rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-30))


def pre_bn_bias(group, key):
    """Biases whose exact gradient is 0 (they sit in front of a training-mode BatchNorm): both sides carry rounding only,
    so Adam's first step (lr * g / |g|) moves them by a sign of noise."""
    if group == "model":
        return key.endswith("bias") and ("lin_l" in key or key.startswith("convs.")) and not key.startswith("convs.2")
    return key == "0.bias"


@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_the_reference_train_step(gold, name):
    case = gold["cases"][name]
    ref = oracle_case(gold, name)
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


def _seed_with_tie(n, offset):
    """The first seed whose n keys at this offset contain an equal pair (about 60 % of seeds at n = 90,941)."""
    for seed in range(64):
        key = philox4x32(seed, offset, np.arange((n + 3) // 4, dtype=np.uint64)).reshape(-1)[:n]
        if np.unique(key).size < n:
            return seed, key.astype(np.int64)
    raise AssertionError("no tied keys in 64 seeds")


def test_sample_perm_is_a_permutation_ordered_by_key_then_row():
    """oracle/gcrd.sample_perm: a permutation of [0, n), keys nondecreasing along it, and equal keys in ascending row order;
    the tie_to_higher control orders the same tie the other way, so it differs exactly where a tie is."""
    n, offset = 90_941, 1 << 62
    seed, key = _seed_with_tie(n, offset)
    perm = og_gcrd.sample_perm(n, seed, offset)
    assert perm.dtype == np.int64 and np.array_equal(np.sort(perm), np.arange(n))
    k = key[perm]
    assert (np.diff(k) >= 0).all()
    tied = np.flatnonzero(np.diff(k) == 0)
    assert tied.size > 0 and (perm[tied] < perm[tied + 1]).all()
    ctrl = og_gcrd.sample_perm(n, seed, offset, tie_to_higher=True)
    assert np.array_equal(key[ctrl], k) and (ctrl[tied] > ctrl[tied + 1]).all()
    assert not np.array_equal(ctrl, perm)
    # small n, and word i % 4 of block i >> 2: n = 5 uses block 1's first word for row 4
    w = philox4x32(3, 7, np.arange(2, dtype=np.uint64)).reshape(-1)
    assert np.array_equal(og_gcrd.sample_perm(5, 3, 7), np.argsort(w[:5], kind="stable"))
    assert np.array_equal(og_gcrd.sample_perm(1, 3, 7), [0])
