"""Generate tests/golden/mag_lsp.pt by running the REFERENCE's own ``train()`` of mag_pyg/gnn_kd_and_aux.py (:174-268) with
``--training lpw`` for one step: the RGCN student (2 layers) learning from an RGCN teacher (3 layers, eval) through
``kd_criterion + beta * lpw_criterion(out, labels, model.out_feat[mask], teacher_model.out_feat[mask], subgraph(...))``.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_mag_lsp.py   (not run by the suite)

Stubs: make_golden.install_mag_stubs(), with torch_geometric.utils.softmax given PyG's size rule for an empty index
(maybe_num_nodes: 0 segments), so that a batch without train-induced edge runs as in the reference.  The reference's
forward hard-codes F.dropout(p=0.5); the module's ``F`` is replaced by one whose dropout multiplies by the recorded keep
mask of the fixture (``masks``) and divides by 1 - p; everything else is torch.nn.functional.

The designed batch (the whole tiny graph is the batch): papers 0-9 with features, authors 10-15 and fields 16-19 from
embedding tables; relations writes (author -> paper), cites (paper -> paper, with the self-loop 2 -> 2 and the duplicate
0 -> 1), has_topic (field -> paper) and to (paper -> author).  Batch ``main`` trains papers {0, 1, 2, 4, 5, 7}: paper 7
is a train row without induced edge.  Batch ``no_edge`` trains papers {3, 7}, which share no edge: the KL runs over no
term.  Per case: the three losses train() returns, every gradient and every parameter after Adam (lr 0.005)."""
from __future__ import annotations

import argparse
import importlib
import importlib.util
import sys
from pathlib import Path

import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; the stub modules have no __spec__ to scan)

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402

from oracle import ops as oo  # noqa: E402

KERNELS = ("cosine", "poly", "l2", "rbf")
BETA, LR, ALPHA, KD_T = 1.0, 0.005, 0.9, 4.0            # scripts/run_kd_and_aux.sh: lpw with beta 1; argparse defaults
F_IN, H, C, H_T = 8, 8, 5, 12
NUM_NODES = {0: 10, 1: 6, 2: 4}
OFF = {0: 0, 1: 10, 2: 16}
CITES = [(0, 1), (0, 1), (1, 0), (2, 2), (1, 4), (4, 5), (5, 0), (3, 0), (6, 1), (8, 7), (7, 9), (9, 3), (2, 6), (5, 2), (4, 0)]
TRAIN = {"main": [0, 1, 2, 4, 5, 7], "no_edge": [3, 7]}


class Batch:
    """The fields train() reads from a GraphSAINT batch."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def to(self, device):
        return self


def designed_graph():
    g = torch.Generator().manual_seed(5)
    writes = torch.stack([torch.randint(0, 6, (12,), generator=g), torch.randint(0, 10, (12,), generator=g)])
    topic = torch.stack([torch.randint(0, 4, (8,), generator=g), torch.randint(0, 10, (8,), generator=g)])
    cites = torch.tensor(CITES).t()
    rels = [(1, 0, writes), (0, 0, cites), (2, 0, topic), (0, 1, writes.flip(0))]
    eis, ets = [], []
    for r, (s, d, ei) in enumerate(rels):
        eis.append(torch.stack([ei[0] + OFF[s], ei[1] + OFF[d]]))
        ets.append(torch.full((ei.shape[1],), r, dtype=torch.long))
    n = sum(NUM_NODES.values())
    node_type = torch.cat([torch.full((NUM_NODES[t],), t, dtype=torch.long) for t in range(3)])
    local = torch.cat([torch.arange(NUM_NODES[t]) for t in range(3)])
    x = torch.randn(NUM_NODES[0], F_IN, generator=g)
    y = torch.full((n, 1), -1, dtype=torch.long)
    y[:10, 0] = torch.randint(0, C, (10,), generator=g)
    masks = {}
    for name, train in TRAIN.items():
        m = torch.zeros(n, dtype=torch.bool)
        m[train] = True
        masks[name] = m
    keep = (torch.rand(n, H, generator=g) < 0.5)
    return dict(edge_index=torch.cat(eis, 1), edge_type=torch.cat(ets), node_type=node_type, local_node_idx=local, x=x, y=y,
                train_mask=masks, keep=keep, relations=[(s, d) for s, d, _ in rels])


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_mag_stubs()
    tg = sys.modules["torch_geometric"]
    tg.utils.softmax = lambda src, index, num_nodes=None: oo.segment_softmax(
        src, index, num_nodes if num_nodes is not None else (int(index.max()) + 1 if index.numel() else 0))
    sys.path.insert(0, str(mg.REF / "mag_pyg"))
    spec = importlib.util.spec_from_file_location("mag_kd", mg.REF / "mag_pyg" / "gnn_kd_and_aux.py")
    mag = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mag)

    G = designed_graph()
    keep = {"mask": None}

    class _F:
        def __getattr__(self, k):
            return getattr(torch.nn.functional, k)

        @staticmethod
        def dropout(x, p=0.5, training=True):
            return x * keep["mask"].to(x.dtype) / (1 - p) if training else x

    mag.F = _F()
    torch.manual_seed(7)
    student0 = mag.RGCN(F_IN, H, C, 2, 0.5, NUM_NODES, [0], len(G["relations"]))
    teacher = mag.RGCN(F_IN, H_T, C, 3, 0.5, NUM_NODES, [0], len(G["relations"]))
    teacher.eval()
    out = dict(G, num_nodes=NUM_NODES, in_channels=F_IN, hidden=H, teacher_hidden=H_T, out_channels=C, beta=BETA, lr=LR,
               alpha=ALPHA, kd_T=KD_T, student_state={k: v.detach().clone() for k, v in student0.state_dict().items()},
               teacher_state={k: v.detach().clone() for k, v in teacher.state_dict().items()}, cases={})
    keep["mask"] = G["keep"]
    runs = [("main", k) for k in KERNELS] + [("no_edge", "rbf")]
    for batch_name, kernel in runs:
        m = mag.RGCN(F_IN, H, C, 2, 0.5, NUM_NODES, [0], len(G["relations"]))
        m.load_state_dict(out["student_state"])
        opt = torch.optim.Adam(m.parameters(), lr=LR)
        b = Batch(edge_index=G["edge_index"], edge_attr=G["edge_type"], node_type=G["node_type"],
                  local_node_idx=G["local_node_idx"], y=G["y"], train_mask=G["train_mask"][batch_name])
        args = argparse.Namespace(training="lpw", kernel=kernel, beta=BETA, alpha=ALPHA, kd_T=KD_T, num_steps=1, batch_size=1)
        loss, loss_cls, loss_aux = mag.train(m, [b], {0: G["x"]}, opt, args, "cpu", teacher)
        out["cases"][f"{batch_name}/{kernel}"] = dict(
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={k: p.grad.detach().clone() for k, p in m.named_parameters()},
            after={k: p.detach().clone() for k, p in m.named_parameters()})
    torch.save(out, mg.OUT / "mag_lsp.pt")
    print("wrote mag_lsp.pt", (mg.OUT / "mag_lsp.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
