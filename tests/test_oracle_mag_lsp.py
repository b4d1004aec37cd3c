"""LSP on MAG without a GPU: the fp64 restatement oracle/mag_lsp.py reproduces one step of the reference's own MAG train()
with --training lpw (tests/golden/mag_lsp.pt, make_golden_mag_lsp.py), including a batch whose train rows induce no edge,
and BatchLSP / the induced-edge entry points refuse bad arguments before any device work."""
from pathlib import Path

import pytest
import torch

from efficient_gnns_b200 import lib
from efficient_gnns_b200.lsp import BatchLSP
from oracle import mag_lsp as om

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "mag_lsp.pt")
KERNELS = ["cosine", "poly", "l2", "rbf"]


class Batch:
    def __init__(self, **kw):
        self.__dict__.update(kw)


def batch(name):
    return Batch(edge_index=GOLD["edge_index"], edge_attr=GOLD["edge_type"], node_type=GOLD["node_type"],
                 local_node_idx=GOLD["local_node_idx"], y=GOLD["y"], train_mask=GOLD["train_mask"][name])


def oracle_step(name, kernel):
    st = {k: v.double().clone().requires_grad_(True) for k, v in GOLD["student_state"].items()}
    te = {k: v.double() for k, v in GOLD["teacher_state"].items()}
    loss, cls, aux = om.lpw_step_loss(st, te, {0: GOLD["x"].double()}, batch(name), [GOLD["keep"]], kernel, GOLD["beta"],
                                      alpha=GOLD["alpha"], kd_T=GOLD["kd_T"])
    total = loss if torch.isfinite(loss) else loss - GOLD["beta"] * aux + GOLD["beta"] * aux.detach().nan_to_num(0.0)
    total.backward()
    grads = {k: v.grad.clone() for k, v in st.items()}
    om.adam(st, {k: torch.zeros_like(v) for k, v in st.items()}, {k: torch.zeros_like(v) for k, v in st.items()}, 1, GOLD["lr"])
    return torch.stack([loss, cls, aux]).detach(), grads, {k: v.detach() for k, v in st.items()}


def test_designed_batches_have_the_edge_cases():
    ei, et = GOLD["edge_index"], GOLD["edge_type"]
    nt = GOLD["node_type"]
    assert len({r for r, (s, d) in enumerate(GOLD["relations"]) if d == 0}) >= 2      # two relations into papers
    assert set(GOLD["num_nodes"]) - {0}                                                # embedding-only types
    main = GOLD["train_mask"]["main"]
    assert bool((nt[main] == 0).all()) and bool(((nt == 0) & ~main).any())           # train and non-train papers
    sub = om.train_induced_edges(main, ei)
    rank7 = int(main[:7].sum())
    assert sub.shape[1] > 0 and not bool((sub == rank7).any())                       # paper 7: a train row, no induced edge
    assert om.train_induced_edges(GOLD["train_mask"]["no_edge"], ei).shape[1] == 0
    cites = ei[:, et == 1]
    assert bool(((cites[0] == 2) & (cites[1] == 2)).any())                            # a self-loop
    assert int(((cites[0] == 0) & (cites[1] == 1)).sum()) == 2                        # a duplicate edge


@pytest.mark.parametrize("kernel", KERNELS)
def test_oracle_reproduces_the_reference_lpw_step(kernel):
    case = GOLD["cases"][f"main/{kernel}"]
    losses, grads, after = oracle_step("main", kernel)
    for got, ref in zip(losses, case["loss"]):
        assert abs(got - ref) <= 1e-5 * abs(ref) + 1e-8, (kernel, losses, case["loss"])
    assert set(grads) == set(case["grads"])
    for k, ref in case["grads"].items():
        assert (grads[k] - ref.double()).abs().max() <= 1e-4 * max(ref.abs().max().item(), 1e-30), k
    for k, ref in case["after"].items():
        g = case["grads"][k]
        keep = g.abs() > 1e-2 * g.abs().max()          # Adam's first step is lr * g / (|g| + eps): compared where g is clear
        if bool(keep.any()):
            assert (after[k][keep] - ref[keep].double()).abs().max() <= 1e-5, k
        assert torch.equal(ref[g == 0], GOLD["student_state"][k][g == 0]), k     # no gradient, no move


def test_a_batch_without_induced_edge_has_a_nan_loss_and_no_lsp_gradient():
    """The reference's kl_div(reduction='mean') over no term is NaN: loss and loss_aux are NaN, loss_cls is finite, and the
    gradients (hence the step) are those of the KD loss alone."""
    case = GOLD["cases"]["no_edge/rbf"]
    ref = case["loss"]
    assert torch.isnan(ref[0]) and torch.isnan(ref[2]) and torch.isfinite(ref[1])
    losses, grads, after = oracle_step("no_edge", "rbf")
    assert torch.isnan(losses[0]) and torch.isnan(losses[2]) and abs(losses[1] - ref[1]) <= 1e-5 * abs(ref[1])
    for k, r in case["grads"].items():
        assert bool(torch.isfinite(r).all()), k
        assert (grads[k] - r.double()).abs().max() <= 1e-4 * max(r.abs().max().item(), 1e-30), k


def test_batch_lsp_refuses_bad_arguments():
    with pytest.raises(ValueError, match="kernel"):
        BatchLSP(32, kernel="gauss", device="cpu")
    with pytest.raises(ValueError, match="hidden width"):
        BatchLSP(lib.LSP_MAX_F + 4, device="cpu")
    with pytest.raises(ValueError, match="criterion"):
        BatchLSP(32, criterion="mse", device="cpu")


def test_induced_edges_argument_validation_without_gpu():
    L = lib.load()
    assert L.b200gnn_induced_edges_tiles(0) == 0 and L.b200gnn_induced_edges_tiles(1024) == 1
    assert L.b200gnn_induced_edges_tiles(1025) == 2 and L.b200gnn_induced_edges_tiles(-1) == -1
    # null pointers, negative sizes and a row pitch shorter than the edge count are rejected before any launch
    assert L.b200gnn_induced_edges_count_i64(None, 4, 4, None, 8, None, None, None, None) == -1
    assert L.b200gnn_induced_edges_count_i64(None, 0, -1, 1, 8, 1, 1, 1, None) == -1
    assert L.b200gnn_induced_edges_count_i64(1, 4, 4, 1, -8, 1, 1, 1, None) == -1
    assert L.b200gnn_induced_edges_count_i64(1, 2, 4, 1, 8, 1, 1, 1, None) == -1
    assert L.b200gnn_induced_edges_count_i64(1, 4, 4, 1, 8, 1, None, 1, None) == -1
    assert L.b200gnn_induced_edges_fill_i64(None, 4, 4, 1, 8, 1, 1, 1, 4, None) == -1
    assert L.b200gnn_induced_edges_fill_i64(1, 4, 4, None, 8, 1, 1, 1, 4, None) == -1
    assert L.b200gnn_induced_edges_fill_i64(1, 4, -4, 1, 8, 1, 1, 1, 4, None) == -1
    assert L.b200gnn_induced_edges_fill_i64(1, 4, 4, 1, 8, 1, 1, 1, -1, None) == -1
    # an empty edge list needs no fill
    assert L.b200gnn_induced_edges_fill_i64(None, 0, 0, 1, 8, 1, None, None, 0, None) == 0
