"""Generate tests/golden/ppi_lsp.pt by running the REFERENCE's own ``train()`` of ppi_pyg/gnn.py (:185-265) with
``--training lpw`` for one step: ``StudentNet`` learning from ``TeacherNet``'s ``out_feat`` through
``lpw_criterion(out, labels, model.out_feat, teacher_model.out_feat, batch.edge_index, kernel, beta)`` (BCE + beta * LSP).

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_ppi_lsp.py   (not run by the suite)

The stubs, the stand-in GATConv and the designed graph are make_golden_ppi.py's: n = 300, a hub above the engine's
HUB_THRESHOLD, node 299 with no edge, the self-loop 5 -> 5 already in edge_index (an LSP edge of similarity k(x, x); for
the l2 kernel the norm of a zero vector) and the duplicate 7 -> 8 (two LSP terms).  Both models start from
``oracle.ppi.seeded_state`` (student seed 101, teacher seed 202, the seeds of ppi_model.pt).  The teacher's 1024-wide
out_feat is a function of that state and the graph, so only its ``oracle.ppi.fingerprint`` is stored: a test restates it
and checks the restatement against the fingerprint.  Per kernel (cosine, poly, l2, rbf at the scripts' beta 100, Adam at
gnn.py's lr 0.005): the three losses train() returns, every gradient (``oracle.ppi.fingerprint``: whole up to 8192 entries)
and every parameter after the optimizer step at the AFTER_SAMPLES entries ``after_entries`` draws."""
from __future__ import annotations

import argparse
import importlib
import sys
from pathlib import Path

import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; the sklearn stub has no __spec__ to scan)

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402
import make_golden_ppi as mgp  # noqa: E402

from oracle import ppi as oppi  # noqa: E402

KERNELS = ("cosine", "poly", "l2", "rbf")
BETA, LR = 100.0, 0.005
SEEDS = dict(student=101, teacher=202)
AFTER_SAMPLES = 256


def after_entries(numel: int) -> torch.Tensor:
    """Flat entries of a parameter recorded after the step: the first AFTER_SAMPLES of the permutation oracle.ppi.fingerprint
    samples a large gradient with, so that they are also entries of the gradient's sample."""
    return torch.randperm(numel, generator=torch.Generator().manual_seed(0))[:AFTER_SAMPLES]


class Batch:
    """The fields train() reads from a PyG Batch of one graph."""

    def __init__(self, x, y, edge_index):
        self.x, self.y, self.edge_index = x, y, edge_index

    def to(self, device):
        return self


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mgp.install_stubs()
    sys.path.insert(0, str(mg.REF / "ppi_pyg"))
    gnn = importlib.import_module("gnn")
    ei = mgp.designed_edges()
    g = torch.Generator().manual_seed(41)                                    # make_golden_ppi's draws: the same x and y
    x = torch.randn(mgp.N, mgp.F_IN, generator=g)
    y = (torch.rand(mgp.N, mgp.C, generator=g) < 0.3).float()
    teacher = gnn.TeacherNet(mgp.F_IN, mgp.C)
    teacher.load_state_dict(oppi.seeded_state(oppi.layers_of("teacher", mgp.C), mgp.F_IN, SEEDS["teacher"]))
    teacher.eval()
    with torch.no_grad():
        teacher(x, ei)
    out = dict(edge_index=ei.to(torch.int32), x=x, y=y.to(torch.uint8), teacher_feat_fp=oppi.fingerprint(teacher.out_feat),
               in_channels=mgp.F_IN, out_channels=mgp.C, seeds=SEEDS, beta=BETA, lr=LR, cases={})
    for kernel in KERNELS:
        m = gnn.StudentNet(mgp.F_IN, mgp.C)
        m.load_state_dict(oppi.seeded_state(oppi.layers_of("student", mgp.C), mgp.F_IN, SEEDS["student"]))
        opt = torch.optim.Adam(m.parameters(), lr=LR)
        args = argparse.Namespace(training="lpw", kernel=kernel, beta=BETA)
        loss, loss_cls, loss_aux = gnn.train(m, teacher, None, [Batch(x, y, ei)], opt, args, "cpu")
        out["cases"][kernel] = dict(
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={k: oppi.fingerprint(p.grad) for k, p in m.named_parameters()},
            after={k: p.detach().reshape(-1)[after_entries(p.numel())].clone() for k, p in m.named_parameters()})
    torch.save(out, mg.OUT / "ppi_lsp.pt")
    print("wrote ppi_lsp.pt", (mg.OUT / "ppi_lsp.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
