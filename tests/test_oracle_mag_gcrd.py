"""G-CRD on MAG without a GPU: the fp64 restatement oracle/mag_gcrd.py reproduces one step of the reference's own MAG train()
with --training nce (tests/golden/mag_gcrd.pt, make_golden_mag_gcrd.py) with every train row, with a recorded 4-row draw
and on a batch without train rows, and gcrd.BatchGCRD refuses bad widths and arguments before any device work."""
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from efficient_gnns_b200.gcrd import BatchGCRD
from oracle import mag_gcrd as omg, mag_lsp as om, ppi_gcrd as opg

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "mag_gcrd.pt")
CASES = {"main/all": "main", "main/sampled": "main", "no_train": "no_train"}
HEAD_KEYS = ("0.weight", "0.bias", "1.weight", "1.bias")


def batch(mask):
    return SimpleNamespace(edge_index=GOLD["edge_index"], edge_attr=GOLD["edge_type"], node_type=GOLD["node_type"],
                           local_node_idx=GOLD["local_node_idx"], y=GOLD["y"], train_mask=GOLD["train_mask"][mask])


def seeded_heads():
    return opg.seeded_heads(GOLD["hidden"], GOLD["teacher_hidden"], GOLD["proj_dim"], GOLD["seeds"]["heads"])


def oracle_step(name):
    """The fixture's case restated in fp64: (losses, grads, after, running) grouped as model / sproj / tproj."""
    c = GOLD["cases"][name]
    leaf = lambda sd: {k: v.double().clone().requires_grad_(True) for k, v in sd.items()}  # noqa: E731
    s_sd, t_sd = seeded_heads()
    groups = {"model": leaf(GOLD["student_state"]), "sproj": leaf({k: s_sd[k] for k in HEAD_KEYS}),
              "tproj": leaf({k: t_sd[k] for k in HEAD_KEYS})}
    running = {g: {k: v.double().clone() for k, v in sd.items() if "running" in k} for g, sd in (("sproj", s_sd), ("tproj", t_sd))}
    teacher = {k: v.double() for k, v in GOLD["teacher_state"].items()}
    b = batch(CASES[name])
    loss, cls, aux, stats = omg.nce_step_loss(groups["model"], teacher, groups["sproj"], groups["tproj"], {0: GOLD["x"].double()},
                                              b, [GOLD["keep"]], c["sample"], GOLD["beta"], GOLD["nce_T"],
                                              alpha=GOLD["alpha"], kd_T=GOLD["kd_T"])
    if torch.isfinite(loss):
        loss.backward()
    params = {f"{g}/{k}": v for g, sd in groups.items() for k, v in sd.items()}
    grads = {g: {k: (v.grad if v.grad is not None else torch.zeros_like(v)).clone() for k, v in sd.items()}
             for g, sd in groups.items()}
    om.adam(params, {k: torch.zeros_like(v) for k, v in params.items()}, {k: torch.zeros_like(v) for k, v in params.items()},
            1, GOLD["lr"])
    n = int(b.train_mask.sum())
    for g in running:
        omg.running_stats(running[g], None if stats is None else stats[g], n)
    after = {g: {k: v.detach() for k, v in sd.items()} for g, sd in groups.items()}
    return torch.stack([loss, cls, aux]).detach(), grads, after, running


def test_fixture_cases():
    main, none = GOLD["train_mask"]["main"], GOLD["train_mask"]["no_train"]
    n = int(main.sum())
    assert GOLD["cases"]["main/all"]["max_samples"] >= n and GOLD["cases"]["main/all"]["sample"] is None
    s = GOLD["cases"]["main/sampled"]["sample"]
    assert 1 < s.numel() == GOLD["cases"]["main/sampled"]["max_samples"] < n and s.unique().numel() == s.numel()
    assert int(none.sum()) == 0
    assert (Path(__file__).resolve().parent / "golden" / "mag_gcrd.pt").stat().st_size < 512 * 1024


@pytest.mark.parametrize("name", ["main/all", "main/sampled"])
def test_oracle_reproduces_the_reference_nce_step(name):
    c = GOLD["cases"][name]
    losses, grads, after, running = oracle_step(name)
    for got, ref in zip(losses, c["loss"]):
        assert abs(got - ref) <= 1e-5 * abs(ref) + 1e-8, (name, losses, c["loss"])
    for group, ref_g in c["grads"].items():
        assert set(ref_g) == set(grads[group]), group
        scale = max(v.abs().max().item() for v in ref_g.values())
        for k, ref in ref_g.items():
            if group != "model" and k == "0.bias":
                # a bias in front of BatchNorm: its exact gradient is 0, the reference's carries rounding only
                assert grads[group][k].abs().max() < 1e-12 * scale and ref.abs().max() < 1e-5 * scale, (group, k)
                continue
            assert (grads[group][k] - ref.double()).abs().max() <= 1e-4 * max(ref.abs().max().item(), 1e-30), (group, k)
            g = ref.double()
            keep = g.abs() > 1e-2 * g.abs().max()      # Adam's first step is lr * g / (|g| + eps): compared where g is clear
            if bool(keep.any()):
                assert (after[group][k][keep] - c["after"][group][k][keep].double()).abs().max() <= 1e-5, (group, k)
    for group, sd in c["running"].items():
        for k in ("1.running_mean", "1.running_var"):
            assert (running[group][k] - sd[k].double()).abs().max() <= 1e-6, (group, k)
        assert int(sd["1.num_batches_tracked"]) == 1


def test_the_draw_changes_the_loss():
    """The two main cases differ only in the sample, so the recorded draw is what main/sampled tests."""
    full, drawn = GOLD["cases"]["main/all"]["loss"], GOLD["cases"]["main/sampled"]["loss"]
    assert full[1] == drawn[1] and abs(float(full[2] - drawn[2])) > 1e-3


def test_a_batch_without_train_rows_is_nan_with_zero_gradients():
    """The reference's means over no row are NaN; nothing carries a gradient, yet Adam steps every head (num_batches_tracked
    advances) and the running statistics stay as they were."""
    c = GOLD["cases"]["no_train"]
    assert all(torch.isnan(v) for v in c["loss"])
    losses, grads, after, running = oracle_step("no_train")
    assert all(torch.isnan(v) for v in losses)
    s_sd, t_sd = seeded_heads()
    for group, ref_g in c["grads"].items():
        for k, ref in ref_g.items():
            assert not bool(ref.any()) and not bool(grads[group][k].any()), (group, k)
            assert torch.equal(c["after"][group][k].double(), after[group][k]), (group, k)
    for group, sd0 in (("sproj", s_sd), ("tproj", t_sd)):
        for k in ("1.running_mean", "1.running_var"):
            assert torch.equal(c["running"][group][k], sd0[k]) and torch.equal(running[group][k], sd0[k].double()), (group, k)
        assert int(c["running"][group]["1.num_batches_tracked"]) == 1


def test_batch_gcrd_refuses_bad_widths_and_arguments():
    for kw in (dict(hidden=30),                                  # not a multiple of 4
               dict(hidden=516),                                 # wider than the student head's weight-gradient GEMM
               dict(teacher_hidden=2052),                        # wider than the teacher head's weight-gradient GEMM
               dict(proj_dim=100), dict(proj_dim=288), dict(proj_dim=32),    # not a multiple of 32 in (48, 256]
               dict(max_samples=0)):
        with pytest.raises(ValueError):
            BatchGCRD(**{"hidden": 32, "teacher_hidden": 512, "device": "cpu", **kw})
    g = BatchGCRD(32, 512, device="cpu")
    assert (g.H, g.F_t, g.P, g.max_samples, g.nce_T, g.beta) == (32, 512, 128, 24576, 0.075, 0.1)
    assert set(g.student_proj_state_dict()) == set(g.teacher_proj_state_dict()) == {
        "0.weight", "0.bias", "1.weight", "1.bias", "1.running_mean", "1.running_var", "1.num_batches_tracked"}
    assert g.teacher_proj_state_dict()["0.weight"].shape == (128, 512)
    # the trainer's widths: L >= 2 and the last hidden layer as built, for the student and for the teacher
    for bad in (SimpleNamespace(L=1, dims=[128, 349]), SimpleNamespace(L=2, dims=[128, 64, 349])):
        with pytest.raises(ValueError, match="hidden"):
            g.bind(bad)
        with pytest.raises(ValueError, match="teacher"):
            g.check_teacher(bad)
    g.bind(SimpleNamespace(L=2, dims=[128, 32, 349]))
    g.check_teacher(SimpleNamespace(L=3, dims=[128, 512, 512, 349]))
    # a batch with one train row, and injected samples that are not S distinct positions in [0, n)
    with pytest.raises(ValueError, match="one train row"):
        g.check_batch(1)
    small = BatchGCRD(32, 512, max_samples=4, device="cpu")
    for n, bad in ((10, torch.arange(3)), (10, torch.zeros(4)), (10, torch.arange(4) + 7), (3, torch.arange(4))):
        with pytest.raises(ValueError, match="distinct"):
            small.check_batch(n, bad)
    small.check_batch(10, torch.tensor([9, 0, 4, 2]))
    small.check_batch(3, torch.tensor([2, 0, 1]))
    small.check_batch(0)
