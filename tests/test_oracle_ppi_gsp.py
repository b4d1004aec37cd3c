"""GSP on PPI without a GPU: the fp64 restatement (oracle.ppi_gsp.gsp_step: StudentNet, GSP between its out_feat and the
teacher's, one Adam step) reproduces one step of the reference's own train() with --training gpw (tests/golden/ppi_gsp.pt,
make_golden_ppi_gsp.py) for the four kernels with every row and for a recorded 128-row draw, and gsp.PerGraphGSP refuses
malformed per-graph inputs before it touches a device."""
from pathlib import Path

import pytest
import torch

from efficient_gnns_b200 import lib
from efficient_gnns_b200.gsp import PerGraphGSP
from oracle import ppi as oppi, ppi_gsp as ogsp
from test_oracle_ppi_lsp import T_FEAT, after_entries

GOLD_PATH = Path(__file__).resolve().parent / "golden" / "ppi_gsp.pt"
GOLD = torch.load(GOLD_PATH)
CASES = ["cosine", "poly", "l2", "rbf", "cosine_s128"]


def oracle_gsp_step(case: str, dtype=torch.float64):
    """The fixture's step restated in ``dtype`` (oracle.ppi_gsp.gsp_step on the designed graph and the seeded student)."""
    c = GOLD["cases"][case]
    model = oppi.seeded_state(oppi.layers_of("student", GOLD["out_channels"]), GOLD["in_channels"], GOLD["seeds"]["student"])
    return ogsp.gsp_step(GOLD["x"], GOLD["y"].to(dtype), GOLD["edge_index"].long(), model, T_FEAT, c["kernel"], c["sample"],
                         beta=GOLD["beta"], lr=GOLD["lr"], dtype=dtype)


def fingerprint(t: torch.Tensor):
    return oppi.fingerprint(t, n_sample=GOLD["fp_samples"])


def test_fixture_cases():
    n = GOLD["x"].shape[0]
    assert GOLD_PATH.stat().st_size < 500_000
    for case in CASES[:4]:
        c = GOLD["cases"][case]
        assert c["kernel"] == case and c["max_samples"] >= n and c["sample"] is None and "after" in c
    s = GOLD["cases"]["cosine_s128"]["sample"]
    assert s.numel() == 128 and s.unique().numel() == 128 and 0 <= int(s.min()) and int(s.max()) < n
    assert GOLD["beta"] == 100.0


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_gpw_step(case):
    c = GOLD["cases"][case]
    got = oracle_gsp_step(case)
    ref = c["loss"]
    assert abs(got["loss"][0] - ref[0]) <= 1e-5 * abs(ref[0]) and abs(got["loss"][1] - ref[1]) <= 1e-5 * abs(ref[1])
    # the rbf similarities of distinct rows underflow on this graph: the term's rounding is relative to its pairs, not to
    # the mean
    assert abs(got["loss"][2] - ref[2]) <= 1e-5 * abs(ref[2]) + 1e-8
    assert set(c["grads"]) == set(got["grads"])
    for k, fp_gold in c["grads"].items():
        fp = fingerprint(got["grads"][k])
        for part, v in fp_gold.items():
            a, b = fp[part].double(), v.double()
            assert (a - b).abs().max() <= 1e-4 * max(b.abs().max().item(), 1e-30), (k, part)
    for k, ref in c.get("after", {}).items():
        # Adam's first step moves a parameter by lr * g / (|g| + eps): compared where the gradient is clearly nonzero
        g = got["grads"][k].reshape(-1)
        idx = after_entries(g.numel())
        keep = g[idx].abs() > 1e-2 * g.abs().max()
        assert (got["after"][k].reshape(-1)[idx][keep] - ref[keep].double()).abs().max() <= 1e-5, k


def test_the_draw_and_the_kernel_change_the_loss():
    """The sampled case differs from the cosine case only in the sample, so the recorded draw is what it tests; every kernel
    gives its own GSP term."""
    cases = GOLD["cases"]
    full, s128 = cases["cosine"]["loss"], cases["cosine_s128"]["loss"]
    assert full[1] == s128[1] and abs(float(full[2] - s128[2])) > 1e-3
    assert len({float(cases[k]["loss"][2]) for k in CASES[:4]}) == 4


def feats(sizes=(40, 55), width=24):
    gen = torch.Generator().manual_seed(0)
    return [torch.randn(n, width, generator=gen) for n in sizes]


def test_per_graph_gsp_refuses_malformed_inputs():
    t = feats()
    for kw in (dict(teacher_feat=[]),                                           # no graphs
               dict(teacher_feat=[t[0], t[1][0]]),                              # not [n, F_t]
               dict(teacher_feat=[t[0], torch.randn(55, 28)]),                  # two teacher widths
               dict(hidden=134),                                                # not a multiple of 4
               dict(hidden=lib.GSP_ROWS_MAX_F + 4),                             # wider than the row passes take
               dict(hidden=0),
               dict(kernel="gaussian"),
               dict(max_samples=0)):
        with pytest.raises(ValueError):
            PerGraphGSP(**{"teacher_feat": t, "hidden": 136, "device": "cpu", **kw})
