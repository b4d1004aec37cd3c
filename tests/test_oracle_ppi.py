"""oracle/ppi.py (the plain-torch restatement of the reference's PPI StudentNet / TeacherNet) reproduces the fixture the
reference's own classes produced (tests/golden/make_golden_ppi.py): eval logits, out_feat, the supervised and kd losses and
every parameter gradient, fp32 and fp64."""
from pathlib import Path

import pytest
import torch

from oracle import ppi as oppi

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "ppi_model.pt")


def close(fp_gold, t, tol):
    """Every part of the fingerprint of t within tol of the fixture's, relative to the part's largest entry."""
    fp = oppi.fingerprint(t)
    assert fp.keys() == fp_gold.keys()
    for k, v in fp_gold.items():
        a, b = fp[k].double(), v.double()
        assert (a - b).abs().max().item() <= tol * max(b.abs().max().item(), 1e-30), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("kind", ["student", "teacher"])
def test_oracle_reproduces_reference_ppi_models(kind, dtype):
    c = GOLD["models"][kind]
    tol = 2e-5 if dtype == torch.float32 else 5e-6          # the fixture itself is fp32
    layers = oppi.layers_of(kind, GOLD["out_channels"])
    x = GOLD["x"].to(dtype)
    n = x.shape[0]
    row, col = oppi.adjacency(GOLD["edge_index"].long(), n)
    assert int(torch.bincount(row, minlength=n).max()) > 256 and int(torch.bincount(row, minlength=n).min()) == 1
    y, t = GOLD["y"].to(dtype), GOLD["teacher_logits"].to(dtype)
    base = oppi.seeded_state(layers, GOLD["in_channels"], c["seed"])
    with torch.no_grad():
        logits, feat = oppi.forward(x, row, col, {k: v.to(dtype) for k, v in base.items()}, layers)
    close(c["logits_eval"], logits, tol)
    close(c["out_feat_eval"], feat, tol)
    for mode in ("supervised", "kd"):
        state = {k: v.to(dtype, copy=True).requires_grad_(True) for k, v in base.items() if "lin_r" not in k}
        state.update({k.replace("lin_l", "lin_r"): v for k, v in state.items() if "lin_l" in k})
        logits, _ = oppi.forward(x, row, col, state, layers)
        losses = oppi.loss(logits, y, t if mode == "kd" else None)
        losses[0].backward()
        ref = c[mode]
        assert (torch.stack([v.detach() for v in losses]).double() - ref["loss"].double()).abs().max() <= tol * ref["loss"].abs().max()
        named = {k: v for k, v in state.items() if "lin_r" not in k}
        assert set(ref["grads"]) == set(named)
        for k, g in ref["grads"].items():
            close(g, named[k].grad, 10 * tol)


def test_state_shapes_match_the_reference_module():
    for kind in ("student", "teacher"):
        sd = oppi.seeded_state(oppi.layers_of(kind, 121), 50, 0)
        assert {k: tuple(v.shape) for k, v in sd.items()} == oppi.state_shapes(oppi.layers_of(kind, 121), 50)
        assert sd["conv1.lin_r.weight"] is sd["conv1.lin_l.weight"]
