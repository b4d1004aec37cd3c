"""GSP on MAG without a GPU: the fp64 restatement oracle/mag_gsp.py reproduces one step of the reference's own MAG train()
with --training gpw (tests/golden/mag_gsp.pt, make_golden_mag_gsp.py) for every kernel, with a recorded 4-row draw, on a
batch without train rows and on a batch with one, and gsp.BatchGSP refuses bad widths and arguments before any device
work."""
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from efficient_gnns_b200 import lib
from efficient_gnns_b200.gsp import BatchGSP
from oracle import mag_gsp as omg, mag_lsp as om

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "mag_gsp.pt")
KERNELS = ["cosine", "poly", "l2", "rbf"]


def batch(mask):
    return SimpleNamespace(edge_index=GOLD["edge_index"], edge_attr=GOLD["edge_type"], node_type=GOLD["node_type"],
                           local_node_idx=GOLD["local_node_idx"], y=GOLD["y"], train_mask=GOLD["train_mask"][mask])


def oracle_step(name):
    """The fixture's case restated in fp64: (losses, grads, after)."""
    c = GOLD["cases"][name]
    st = {k: v.double().clone().requires_grad_(True) for k, v in GOLD["student_state"].items()}
    te = {k: v.double() for k, v in GOLD["teacher_state"].items()}
    loss, cls, aux = omg.gpw_step_loss(st, te, {0: GOLD["x"].double()}, batch(c["mask"]), [GOLD["keep"]], c["kernel"],
                                       c["sample"], GOLD["beta"], alpha=GOLD["alpha"], kd_T=GOLD["kd_T"])
    if torch.isfinite(loss):
        loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)).clone() for k, v in st.items()}
    om.adam(st, {k: torch.zeros_like(v) for k, v in st.items()}, {k: torch.zeros_like(v) for k, v in st.items()}, 1, GOLD["lr"])
    return torch.stack([loss, cls, aux]).detach(), grads, {k: v.detach() for k, v in st.items()}


def test_fixture_cases():
    main, none, one = (GOLD["train_mask"][k] for k in ("main", "no_train", "one_train"))
    n = int(main.sum())
    for k in KERNELS:
        c = GOLD["cases"][f"main/{k}"]
        assert c["kernel"] == k and c["max_samples"] >= n and c["sample"] is None
    s = GOLD["cases"]["main/sampled"]["sample"]
    assert 1 < s.numel() == GOLD["cases"]["main/sampled"]["max_samples"] < n and s.unique().numel() == s.numel()
    assert int(none.sum()) == 0 and int(one.sum()) == 1 and bool(main[one].all())
    assert (Path(__file__).resolve().parent / "golden" / "mag_gsp.pt").stat().st_size < 512 * 1024


@pytest.mark.parametrize("name", [f"main/{k}" for k in KERNELS] + ["main/sampled", "one_train"])
def test_oracle_reproduces_the_reference_gpw_step(name):
    c = GOLD["cases"][name]
    losses, grads, after = oracle_step(name)
    for got, ref in zip(losses, c["loss"]):
        assert abs(got - ref) <= 1e-5 * abs(ref) + 1e-8, (name, losses, c["loss"])
    scale = max(v.abs().max().item() for v in c["grads"].values())
    for k, ref in c["grads"].items():
        assert (grads[k] - ref.double()).abs().max() <= 1e-4 * max(ref.abs().max().item(), 1e-6 * scale), (name, k)
        g = ref.double()
        keep = g.abs() > 1e-2 * g.abs().max()          # Adam's first step is lr * g / (|g| + eps): compared where g is clear
        if bool(keep.any()):
            assert (after[k][keep] - c["after"][k][keep].double()).abs().max() <= 1e-5, (name, k)


def test_the_gsp_term_moves_the_step():
    """Every main case has the same KD part; the GSP term changes loss[0] and the gradient, the draw changes loss_aux."""
    main = {k: GOLD["cases"][f"main/{k}"] for k in KERNELS}
    for c in main.values():
        assert c["loss"][1] == main["cosine"]["loss"][1] and c["loss"][2] > 1e-3
    assert abs(float(GOLD["cases"]["main/sampled"]["loss"][2] - main["cosine"]["loss"][2])) > 1e-3
    a, b = main["cosine"]["grads"], main["rbf"]["grads"]
    assert any(not torch.equal(a[k], b[k]) for k in a)


def test_degenerate_batches():
    """No train row: every loss is NaN and nothing carries a gradient.  One train row: the 1 x 1 similarities are equal,
    exactly for l2 and rbf (the distance of a row to itself is 0), up to rounding for cosine and poly (|x / |x||^2 = 1)."""
    c = GOLD["cases"]["no_train"]
    assert all(torch.isnan(v) for v in c["loss"])
    assert not any(bool(g.any()) for g in c["grads"].values())
    losses, grads, _ = oracle_step("no_train")
    assert all(torch.isnan(v) for v in losses) and not any(bool(g.any()) for g in grads.values())
    one = GOLD["cases"]["one_train"]
    assert one["kernel"] == "l2" and float(one["loss"][2]) == 0.0
    st = {k: v.double().clone().requires_grad_(True) for k, v in GOLD["student_state"].items()}
    te = {k: v.double() for k, v in GOLD["teacher_state"].items()}
    for kernel in KERNELS:
        _, _, aux = omg.gpw_step_loss(st, te, {0: GOLD["x"].double()}, batch("one_train"), [GOLD["keep"]], kernel, None,
                                      GOLD["beta"])
        aux = float(aux.detach())
        assert aux == 0.0 if kernel in ("l2", "rbf") else 0.0 <= aux < 1e-28, (kernel, aux)


def test_batch_gsp_refuses_bad_widths_and_arguments():
    for kw in (dict(hidden=30),                                  # not a multiple of 4
               dict(hidden=lib.GSP_CONTRACT_MAX_F + 4),           # wider than the narrow contraction
               dict(hidden=0),
               dict(teacher_hidden=514),                          # not a multiple of 4
               dict(teacher_hidden=lib.GSP_ROWS_MAX_F + 4),       # wider than the row passes
               dict(kernel="cos"), dict(max_samples=0)):
        with pytest.raises(ValueError):
            BatchGSP(**{"hidden": 32, "teacher_hidden": 512, "device": "cpu", **kw})
    g = BatchGSP(32, 512, device="cpu")
    assert (g.H, g.F_t, g.kernel, g.beta, g.max_samples) == (32, 512, "poly", 1.0, 24576)
    assert BatchGSP(lib.GSP_CONTRACT_MAX_F, lib.GSP_ROWS_MAX_F, "rbf", device="cpu").kernel_id == 3
    # the trainer's widths: L >= 2 and the last hidden layer as built, for the student and for the teacher
    for bad in (SimpleNamespace(L=1, dims=[128, 349]), SimpleNamespace(L=2, dims=[128, 64, 349])):
        with pytest.raises(ValueError, match="hidden width 32"):
            g.bind(bad)
        with pytest.raises(ValueError, match="teacher hidden width 512"):
            g.check_teacher(bad)
    g.bind(SimpleNamespace(L=2, dims=[128, 32, 349]))
    g.check_teacher(SimpleNamespace(L=3, dims=[128, 512, 512, 349]))
    # injected samples: S distinct positions in [0, n), and none when S = n
    small = BatchGSP(32, 512, max_samples=4, device="cpu")
    for n, bad in ((10, torch.arange(3)), (10, torch.zeros(4)), (10, torch.arange(4) + 7)):
        with pytest.raises(ValueError, match="distinct"):
            small.check_batch(n, bad)
    for n in (3, 4):
        with pytest.raises(ValueError, match="no sample to inject"):
            small.check_batch(n, torch.arange(n))
    small.check_batch(10, torch.tensor([9, 0, 4, 2]))
    for n in (0, 1, 4, 10):
        small.check_batch(n)
    assert small.sample().numel() == 0
