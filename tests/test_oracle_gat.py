"""oracle/gat.py (the plain-torch restatement of the reference's GAT model) reproduces the fixture the reference's own class
produced (tests/golden/make_golden_gat_model.py): logits, feat, loss and every parameter gradient, fp32 and fp64."""
from pathlib import Path

import pytest
import torch

from oracle import gat as ogat

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "gat_model_arxiv.pt")


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
@pytest.mark.parametrize("case", ["attn_dst", "no_attn_dst"])
def test_oracle_reproduces_reference_gat(case, dtype):
    c = GOLD["cases"][case]
    tol = 2e-5 if dtype == torch.float32 else 5e-6          # the fixture itself is fp32
    state = {k: v.detach().clone().to(dtype).requires_grad_("running" not in k) for k, v in c["state"].items()}
    x, row, col = GOLD["x"].to(dtype), GOLD["row"], GOLD["col"]
    logits, feat = ogat.gat_forward(x, row, col, state, GOLD["n_layers"], GOLD["n_heads"], True, training=True)
    loss = torch.nn.functional.cross_entropy(logits[GOLD["train_idx"]], GOLD["y"][GOLD["train_idx"]])
    loss.backward()

    def rel(a, b):
        return (a.double() - b.double()).abs().max().item() / max(b.double().abs().max().item(), 1e-30)
    assert rel(logits.detach(), c["logits_train"]) <= tol
    assert rel(feat.detach(), c["feat_train"]) <= tol
    assert abs(loss.item() - c["loss"].item()) <= tol * abs(c["loss"].item())
    assert set(c["grads"]) == {k for k, v in state.items() if v.requires_grad}
    for k, g in c["grads"].items():
        assert rel(state[k].grad, g) <= 10 * tol, k
    with torch.no_grad():
        logits_e, feat_e = ogat.gat_forward(x, row, col, state, GOLD["n_layers"], GOLD["n_heads"], True, training=False)
    assert rel(logits_e, c["logits_eval"]) <= tol and rel(feat_e, c["feat_eval"]) <= tol


def test_edge_keep_all_dropped_destination_outputs_its_residual():
    c = GOLD["cases"]["attn_dst"]
    state = {k: v.double() for k, v in c["state"].items()}
    x, row, col = GOLD["x"].double(), GOLD["row"], GOLD["col"]
    keep = torch.ones(row.numel(), dtype=torch.bool)
    keep[row == 5] = False
    out = ogat.gat_conv(x, row, col, x.shape[0], state["convs.0.fc.weight"], state["convs.0.attn_l"], state["convs.0.attn_r"],
                        state["convs.0.res_fc.weight"], GOLD["n_heads"], True, keep)
    res = torch.nn.functional.linear(x, state["convs.0.res_fc.weight"]).view(out.shape)
    assert torch.equal(out[5], res[5]) and torch.isfinite(out).all()
