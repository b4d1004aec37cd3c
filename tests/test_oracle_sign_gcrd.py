"""G-CRD on the SIGN student without a GPU: the fp64 restatement oracle/sign_gcrd.py reproduces one step of the reference's
own train_kd_and_aux with --training nce (tests/golden/sign_gcrd.pt, make_golden_sign_gcrd.py) for ff_layer 1 and 2, with
every row and with a recorded 12-row draw, and gcrd.SIGNGCRD refuses bad widths and arguments before any device work."""
from pathlib import Path

import pytest
import torch

from efficient_gnns_b200.gcrd import SIGNGCRD
from oracle import ppi_gcrd as opg, sign_gcrd as osg

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "sign_gcrd.pt")
H = len(GOLD["feats"])


def masks(ff):
    return osg.engine_masks(H, GOLD["feats"][0].shape[1], GOLD["hidden"], ff, GOLD["batch"].numel(), GOLD["dropout"],
                            GOLD["input_drop"], GOLD["seeds"]["dropout"], 0)


def oracle_step(name):
    c = GOLD["cases"][name]
    ff = c["ff"]
    s_sd, t_sd = opg.seeded_heads(H * GOLD["hidden"], GOLD["teacher_feat"].shape[1], GOLD["proj_dim"], GOLD["seeds"]["heads"])
    run = osg.Run(GOLD["states"][ff], s_sd, t_sd, GOLD["lr"])
    b = GOLD["batch"]
    losses, grads = run.step([f[b] for f in GOLD["feats"]], GOLD["labels"][b], GOLD["teacher_logits"][b],
                             GOLD["teacher_feat"][b], masks(ff), c["sample"], ff, GOLD["beta"], GOLD["nce_T"],
                             p=GOLD["dropout"], p_in=GOLD["input_drop"], alpha=GOLD["alpha"], kd_T=GOLD["kd_T"])
    return losses, grads, {g: run.state(g) for g in run.groups}, run.running


def test_fixture_cases():
    B = GOLD["batch"].numel()
    for ff in (1, 2):
        assert GOLD["cases"][f"ff{ff}/all"]["max_samples"] >= B and GOLD["cases"][f"ff{ff}/all"]["sample"] is None
        s = GOLD["cases"][f"ff{ff}/sampled"]["sample"]
        assert 1 < s.numel() == GOLD["cases"][f"ff{ff}/sampled"]["max_samples"] < B and s.unique().numel() == s.numel()
    assert GOLD["teacher_feat"].shape[1] % 4                     # the engine pads the teacher rows
    assert (Path(__file__).resolve().parent / "golden" / "sign_gcrd.pt").stat().st_size < 640 * 1024


@pytest.mark.parametrize("name", sorted(GOLD["cases"]))
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
                assert (after[group][k][keep] - c["after"][group][k][keep].double()).abs().max() <= 1e-6, (group, k)
    for group, sd in c["running"].items():
        for k in ("1.running_mean", "1.running_var"):
            assert (running[group][k] - sd[k].double()).abs().max() <= 1e-6, (group, k)
        assert int(sd["1.num_batches_tracked"]) == 1


def test_the_draw_changes_the_loss():
    """The all and sampled cases differ only in the sample, so the recorded draw is what the sampled cases test."""
    for ff in (1, 2):
        full, drawn = GOLD["cases"][f"ff{ff}/all"]["loss"], GOLD["cases"][f"ff{ff}/sampled"]["loss"]
        assert full[1] == drawn[1] and abs(float(full[2] - drawn[2])) > 1e-3


def test_sign_gcrd_refuses_bad_widths_and_arguments():
    t = torch.randn(10, 750)
    for kw in (dict(hidden=3070),                                # not a multiple of 32 (the keep words of the head's input)
               dict(hidden=0),
               dict(teacher_feat=torch.randn(10, 2052)),         # wider than the teacher head's weight-gradient GEMM
               dict(teacher_feat=torch.randn(10)),
               dict(proj_dim=100), dict(proj_dim=288), dict(proj_dim=32),    # not a multiple of 32 in (48, 256]
               dict(max_samples=0)):
        with pytest.raises(ValueError):
            SIGNGCRD(**{"teacher_feat": t, "hidden": 3072, **kw})
    g = SIGNGCRD(t, 3072)
    assert (g.H, g.F_t, g.Ft_pad, g.N, g.P, g.max_samples, g.nce_T, g.beta) == (3072, 750, 752, 10, 256, 16384, 0.075, 0.1)
    assert torch.equal(g.t_feat[:, 750:], torch.zeros(10, 2)) and torch.equal(g.t_feat[:, :750], t)
    assert set(g.student_proj_state_dict()) == set(g.teacher_proj_state_dict()) == {
        "0.weight", "0.bias", "1.weight", "1.bias", "1.running_mean", "1.running_var", "1.num_batches_tracked"}
    assert g.student_proj_state_dict()["0.weight"].shape == (256, 3072)
    assert g.teacher_proj_state_dict()["0.weight"].shape == (256, 750)
    with pytest.raises(ValueError, match="one row"):
        g.check_batch(1)
    small = SIGNGCRD(t, 3072, max_samples=4)
    for n, bad in ((10, torch.arange(3)), (10, torch.zeros(4)), (10, torch.arange(4) + 7), (3, torch.arange(4))):
        with pytest.raises(ValueError, match="distinct"):
            small.check_batch(n, bad)
    small.check_batch(10, torch.tensor([9, 0, 4, 2]))
    small.check_batch(3, torch.tensor([2, 0, 1]))


def test_head_state_dicts_round_trip():
    s_sd, t_sd = opg.seeded_heads(96, 22, 64, 5)
    g = SIGNGCRD(torch.randn(10, 22), 96, proj_dim=64)
    s_sd = dict(s_sd, **{"1.num_batches_tracked": torch.tensor(7), "1.running_mean": torch.randn(64)})
    g.load_student_proj_state_dict(s_sd)
    g.load_teacher_proj_state_dict(t_sd)
    for got, ref in ((g.student_proj_state_dict(), s_sd), (g.teacher_proj_state_dict(), t_sd)):
        assert set(got) == set(ref)
        for k in ref:
            assert torch.equal(got[k], ref[k]), k
    assert torch.equal(g.W_t[:, 22:], torch.zeros(64, 2))
