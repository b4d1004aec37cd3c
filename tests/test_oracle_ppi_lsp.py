"""LSP on PPI without a GPU: the fp64 restatement (oracle/ppi.py's StudentNet + oracle/criterion.py's lpw_criterion)
reproduces one step of the reference's own train() with --training lpw (tests/golden/ppi_lsp.pt, make_golden_ppi_lsp.py),
and lsp.PerGraphLSP refuses malformed per-graph inputs before it touches a device."""
from pathlib import Path

import pytest
import torch

from efficient_gnns_b200 import lib
from efficient_gnns_b200.lsp import PerGraphLSP
from oracle import criterion as ocrit, ppi as oppi

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "ppi_lsp.pt")
KERNELS = ["cosine", "poly", "l2", "rbf"]


def after_entries(numel: int) -> torch.Tensor:
    """The flat entries of each parameter the fixture records after the step (make_golden_ppi_lsp.after_entries)."""
    return torch.randperm(numel, generator=torch.Generator().manual_seed(0))[:256]


def teacher_feat() -> torch.Tensor:
    """TeacherNet's out_feat [300, 1024] on the designed graph, restated in fp64 from its seeded state (the fixture keeps
    only the fingerprint of the reference's own, which test_teacher_features_match_the_reference checks this against)."""
    layers = oppi.layers_of("teacher", GOLD["out_channels"])
    state = oppi.seeded_state(layers, GOLD["in_channels"], GOLD["seeds"]["teacher"])
    row, col = oppi.adjacency(GOLD["edge_index"].long(), GOLD["x"].shape[0])
    with torch.no_grad():
        return oppi.forward(GOLD["x"].double(), row, col, {k: v.double() for k, v in state.items()}, layers)[1]


T_FEAT = teacher_feat()


def oracle_lsp_step(kernel, dtype=torch.float64):
    """Losses, gradients and the parameters after Adam's first step, restated in ``dtype``."""
    x, y, ei = GOLD["x"].to(dtype), GOLD["y"].to(dtype), GOLD["edge_index"].long()
    layers = oppi.layers_of("student", GOLD["out_channels"])
    base = oppi.seeded_state(layers, GOLD["in_channels"], GOLD["seeds"]["student"])
    st = {k: v.to(dtype, copy=True).requires_grad_(True) for k, v in base.items() if "lin_r" not in k}
    st.update({k.replace("lin_l", "lin_r"): v for k, v in st.items() if "lin_l" in k})
    row, col = oppi.adjacency(ei, x.shape[0])
    logits, feat = oppi.forward(x, row, col, st, layers)
    loss_cls = oppi.loss(logits, y)[0]
    dummy = torch.zeros(x.shape[0], 2, dtype=dtype), torch.zeros(x.shape[0], dtype=torch.long)
    loss_aux = ocrit.lpw_criterion(*dummy, feat, T_FEAT.to(dtype), ei, kernel, GOLD["beta"])[2]
    loss = loss_cls + GOLD["beta"] * loss_aux
    loss.backward()
    named = {k: v for k, v in st.items() if "lin_r" not in k}
    grads = {k: v.grad for k, v in named.items()}
    after = {k: v.detach() - GOLD["lr"] * grads[k] / (grads[k].abs() + 1e-8) for k, v in named.items()}
    return torch.stack([loss, loss_cls, loss_aux]).detach(), grads, after


def test_designed_graph_has_the_edge_cases():
    ei = GOLD["edge_index"].long()
    n = GOLD["x"].shape[0]
    src, dst = ei
    assert ((src == 5) & (dst == 5)).sum() == 1                                 # a self-loop in the edge list
    assert ((src == 7) & (dst == 8)).sum() == 2                                 # a duplicate edge
    assert int(dst.max()) + 1 < n                                               # n_seg < n
    assert (torch.bincount(dst, minlength=n) == 0).any()                       # nodes with no in-edge
    assert int(torch.bincount(dst, minlength=n).max()) > 256                    # the hub


def test_teacher_features_match_the_reference():
    fp = oppi.fingerprint(T_FEAT)
    assert fp.keys() == GOLD["teacher_feat_fp"].keys()
    for part, v in GOLD["teacher_feat_fp"].items():
        assert (fp[part] - v.double()).abs().max() <= 5e-6 * v.double().abs().max(), part


@pytest.mark.parametrize("kernel", KERNELS)
def test_oracle_reproduces_the_reference_lpw_step(kernel):
    case = GOLD["cases"][kernel]
    losses, grads, after = oracle_lsp_step(kernel)
    ref = case["loss"]
    assert abs(losses[0] - ref[0]) <= 1e-5 * abs(ref[0]) and abs(losses[1] - ref[1]) <= 1e-5 * abs(ref[1])
    # the KL is a mean of per-edge terms that cancel to a small sum: its rounding is relative to the terms, not the result
    assert abs(losses[2] - ref[2]) <= 1e-5 * abs(ref[2]) + 1e-8
    assert set(case["grads"]) == set(grads)
    for k, fp_gold in case["grads"].items():
        fp = oppi.fingerprint(grads[k])
        for part, v in fp_gold.items():
            a, b = fp[part].double(), v.double()
            assert (a - b).abs().max() <= 1e-4 * max(b.abs().max().item(), 1e-30), (k, part)
    for k, ref in case["after"].items():
        # Adam's first step moves a parameter by lr * g / (|g| + eps): compared where the gradient is clearly nonzero
        idx = after_entries(grads[k].numel())
        g = grads[k].reshape(-1)
        keep = g[idx].abs() > 1e-2 * g.abs().max()
        assert (after[k].reshape(-1)[idx][keep] - ref[keep].double()).abs().max() <= 1e-5, k


def test_l2_self_loop_has_a_zero_subgradient_in_the_reference_and_the_oracle():
    """The l2 kernel on the self-loop 5 -> 5 is ||0||: torch's norm backward and the oracle both give it gradient 0, so the
    loss's gradient does not depend on how that edge's zero distance is differentiated."""
    f = torch.randn(10, 6, dtype=torch.float64, requires_grad=True)
    (f[5] - f[5]).norm(p=2, dim=-1).backward()
    assert torch.equal(f.grad, torch.zeros_like(f))
    f.grad = None
    ocrit._edge_similarity(f, torch.tensor([5]), torch.tensor([5]), "l2").sum().backward()
    assert torch.equal(f.grad, torch.zeros_like(f))


def inputs(k=2):
    gen = torch.Generator().manual_seed(0)
    t = [torch.randn(n, 16, generator=gen) for n in (40, 55)[:k]]
    ei = [torch.randint(0, n, (2, 3 * n), generator=gen) for n in (40, 55)[:k]]
    return t, ei


def test_per_graph_plans_refuse_malformed_inputs():
    t, ei = inputs()
    bad_edges = [
        [ei[0], ei[1][:, :0]],                                                   # a graph with no edges
        [ei[0], torch.cat([ei[1], torch.tensor([[0], [55]])], 1)],               # an index outside its graph
        [torch.cat([ei[0], torch.tensor([[40], [0]])], 1), ei[1]],
        [ei[0], torch.cat([ei[1], torch.tensor([[-1], [0]])], 1)],
        [ei[0], ei[1][0]],                                                       # not [2, E]
    ]
    for e in bad_edges:
        with pytest.raises(ValueError):
            PerGraphLSP(t, e, 136, device="cpu")
    with pytest.raises(ValueError):
        PerGraphLSP(t, ei[:1], 136, device="cpu")                               # counts differ
    with pytest.raises(ValueError):
        PerGraphLSP([], [], 136, device="cpu")
    with pytest.raises(ValueError):
        PerGraphLSP(t, ei, lib.LSP_MAX_F + 4, device="cpu")                     # wider than the kernel holds
    with pytest.raises(ValueError):
        PerGraphLSP(t, ei, 0, device="cpu")
    with pytest.raises(ValueError):
        PerGraphLSP(t, ei, 136, criterion="mse", device="cpu")                  # the fused kernel is the kld form
    with pytest.raises(ValueError):
        PerGraphLSP(t, ei, 136, kernel="gaussian", device="cpu")
