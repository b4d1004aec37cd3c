"""Generate tests/golden/gat_model_arxiv.pt by running the REFERENCE's own ``GAT`` class (arxiv_dgl/models.py:239-313),
unmodified, on the ``dgl`` stand-in of make_golden.py (graph primitives restated with plain torch index ops).

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_gat_model.py   (not run by the test suite)

3 layers, 3 heads of width 10 (a head width the engine stores padded), use_symmetric_norm=True, use_attn_dst both ways, all
dropouts 0 (the draws are the only thing that cannot be shared): state, eval logits and ``feat``, and one train-mode
cross-entropy forward / backward with every parameter gradient.  On a designed graph: symmetric + self-loops, one hub above
the engine's hub threshold, degree-1 rows (self-loop only)."""
from __future__ import annotations

import importlib
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402

from oracle import graph as og  # noqa: E402


def designed_graph(n=700, e=2400, hub_deg=600, n_isolated=12, seed=5):
    """Symmetric graph + self-loops: node 0 is joined to hub_deg others, the last n_isolated nodes have the self-loop only."""
    from efficient_gnns_b200.synthetic import skewed_edges
    m = n - n_isolated
    ei = skewed_edges(m, e, seed).numpy()
    hub = np.stack([np.zeros(hub_deg, dtype=ei.dtype), np.arange(1, hub_deg + 1, dtype=ei.dtype)])
    ei = np.concatenate([ei, hub], axis=1)
    row, col, _ = og.to_sparse_adj_t(ei, n)
    r, c = og.to_symmetric(row, col, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    return torch.from_numpy(rs), torch.from_numpy(cs)                          # row = destination, col = source


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_stubs()
    mg.install_dgl_stubs()
    sys.path.insert(0, str(mg.REF / "arxiv_dgl"))
    models = importlib.import_module("models")
    n, F_in, C, D, H, L = 700, 16, 8, 10, 3, 3
    row, col = designed_graph(n)
    graph = mg._DGLGraph(col, row, n)
    g = torch.Generator().manual_seed(17)
    x = torch.randn(n, F_in, generator=g)
    y = torch.randint(0, C, (n,), generator=g)
    train_idx = torch.randperm(n, generator=g)[:400].sort().values
    out = {}
    for name, dst in (("attn_dst", True), ("no_attn_dst", False)):
        torch.manual_seed(7)
        m = models.GAT(F_in, C, D, L, H, torch.nn.functional.relu, dropout=0.0, input_drop=0.0, attn_drop=0.0, edge_drop=0.0,
                       use_attn_dst=dst, use_symmetric_norm=True)
        with torch.no_grad():                                                   # non-trivial BatchNorm / bias parameters
            for k, v in m.state_dict().items():
                if k.startswith("norms") and k.endswith(("weight", "bias")) or k == "bias_last.bias":
                    v.add_(0.3 * torch.randn(v.shape, generator=g))
        state = {k: v.detach().clone() for k, v in m.state_dict().items() if v is not None and "num_batches" not in k}
        m.train()
        logits = m(graph, x)
        loss = torch.nn.functional.cross_entropy(logits[train_idx], y[train_idx])
        loss.backward()
        case = dict(state=state, logits_train=logits.detach().clone(), feat_train=m.feat.detach().clone(), loss=loss.detach(),
                    grads={k: p.grad.detach().clone() for k, p in m.named_parameters()},
                    state_after={k: v.detach().clone() for k, v in m.state_dict().items() if "running" in k})
        m.load_state_dict({**m.state_dict(), **state})
        m.eval()
        with torch.no_grad():
            case["logits_eval"] = m(graph, x).clone()
            case["feat_eval"] = m.feat.clone()
        out[name] = case
    torch.save(dict(row=row, col=col, x=x, y=y, train_idx=train_idx, n_layers=L, n_heads=H, n_hidden=D, n_classes=C, cases=out),
               mg.OUT / "gat_model_arxiv.pt")
    print("wrote gat_model_arxiv.pt")


if __name__ == "__main__":
    main()
