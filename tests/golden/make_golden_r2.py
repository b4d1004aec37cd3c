"""Round-2 golden fixtures: the reference's OWN files at sizes that cross the engine's special paths (hub rows split
across CTAs, the pipelined K=256 kernel, the 750-wide teacher features) and the PPI criterion file.

    python tests/golden/make_golden_r2.py        REFERENCE=<checkout of the reference repository>   (not run by the test suite)

Same method as make_golden.py (whose stand-in modules are reused): the reference file computes, the third-party
primitives underneath come from oracle/.  Large outputs are stored for a fixed subset of rows (`rows`) plus their full
Frobenius norms, so the files stay small while every parameter gradient (a reduction over ALL rows) is stored whole.
  * criterion_ppi.pt    — ppi_pyg/criterion.py: kd / fitnet / lpw / nce with the binary cross-entropy term.
  * model_arxiv_hub.pt  — arxiv_pyg/gnn.py `GCN` and `SAGE`, 16-256-256-8, on a 3,000-node graph whose heaviest rows
                          have > 1,000 neighbours (hub path) — K=256 aggregations forward and backward.
  * lsp_wide.pt         — arxiv_pyg/criterion.py lpw_criterion (cosine, rbf) with F_s=256, F_t=750 on the train-induced
                          subgraph of the same graph (destination segments up to > 1,000 edges).
  * gat_wide.pt         — arxiv_dgl/models.py `GATConv`, 3 heads x 250 (the reference teacher's shape, K=750), hub graph.
"""
from __future__ import annotations

import importlib
import sys
from pathlib import Path

import numpy as np
import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
import make_golden as mg  # noqa: E402
import inputs_r2 as R2  # noqa: E402

REF, OUT = mg.REF, mg.OUT
og = mg.og


def main():
    assert REF.exists()
    mg.install_stubs()
    # ------------------------------------------------------------------ ppi_pyg/criterion.py
    sys.path.insert(0, str(REF / "ppi_pyg"))
    spec = importlib.util.spec_from_file_location("ppi_criterion", REF / "ppi_pyg" / "criterion.py")
    pc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(pc)
    g = torch.Generator().manual_seed(31)
    n, C, F = 300, 121, 32
    logits = torch.randn(n, C, generator=g)
    labels = (torch.rand(n, C, generator=g) < 0.3).float()
    t_logits = torch.randn(n, C, generator=g) * 3
    feat, t_feat = torch.randn(n, F, generator=g), torch.randn(n, F, generator=g)
    _, r, c, _ = R2.hub_graph(n, 1500, 2)
    ei = torch.from_numpy(np.stack([r, c]))
    cases = {}

    def run(name, fn, with_feat=True):
        z = logits.clone().requires_grad_(True)
        f = feat.clone().requires_grad_(with_feat)
        out = fn(z, f)
        gr = torch.autograd.grad(out[0], [z] + ([f] if with_feat else []))
        cases[name] = dict(loss=out[0].detach(), loss_cls=out[1].detach(), loss_aux=out[2].detach(), d_logits=gr[0],
                           d_feat=gr[1] if with_feat else None)
    run("kd", lambda z, f: pc.kd_criterion(z, labels, t_logits), False)
    run("fitnet", lambda z, f: pc.fitnet_criterion(z, labels, f, t_feat))
    run("lpw_cosine", lambda z, f: pc.lpw_criterion(z, labels, f, t_feat, ei, "cosine", 100))
    run("nce_full", lambda z, f: pc.nce_criterion(z, labels, f, t_feat, 0.5, 0.075, 10 ** 9))
    torch.save(dict(inputs=dict(logits=logits, labels=labels, t_logits=t_logits, feat=feat, t_feat=t_feat, edge_index=ei),
                    cases=cases), OUT / "criterion_ppi.pt")

    # ------------------------------------------------------------------ arxiv_pyg/gnn.py GCN / SAGE on a hub graph
    sys.path.insert(0, str(REF / "arxiv_pyg"))
    for m in ("criterion", "gnn"):
        sys.modules.pop(m, None)
    crit = importlib.import_module("criterion")
    gnn = importlib.import_module("gnn")
    hm = R2.hub_model()
    n, (Fin, Hd, C) = hm["n"], hm["dims"]
    deg = np.diff(hm["rowptr"])
    assert deg.max() > 1000, deg.max()          # hub threshold of the engine is 256
    x, y, train_idx, rows = hm["x"], hm["y"], hm["train_idx"], hm["rows"]
    adj = mg._AdjT(torch.from_numpy(hm["rowptr"]), torch.from_numpy(hm["c"]), n)
    models = {}
    for name, cls in (("gcn", gnn.GCN), ("sage", gnn.SAGE)):
        torch.manual_seed(5)
        m = cls(Fin, Hd, C, 3, 0.0)
        m.train()
        out = m(x, adj)
        loss = torch.nn.functional.cross_entropy(out[train_idx], y[train_idx])
        loss.backward()
        models[name] = dict(state={k: v.detach().clone() for k, v in m.state_dict().items()},
                            logits_rows=out.detach()[rows].clone(), logits_norm=out.detach().double().norm(),
                            out_feat_rows=m.out_feat.detach()[rows].clone(), out_feat_norm=m.out_feat.detach().double().norm(),
                            loss=loss.detach(), grads={k: p.grad.detach().clone() for k, p in m.named_parameters()})
    torch.save(dict(input_checksum=R2.checksum(x, y, train_idx, torch.from_numpy(hm["c"])), max_degree=int(deg.max()),
                    models=models), OUT / "model_arxiv_hub.pt")

    # ------------------------------------------------------------------ LSP with the real widths (256 vs 750)
    lw = R2.lsp_wide()
    sub_ei, rows_l = lw["sub_edge_index"], lw["rows"]
    seg = torch.bincount(sub_ei[1], minlength=lw["feat"].shape[0])
    lsp = {}
    for k, (sf, st) in lw["scales"].items():
        f = (lw["feat"] * sf).clone().requires_grad_(True)
        out = crit.lpw_criterion(lw["logits"], lw["labels"], f, lw["t_feat"] * st, sub_ei, k, 100)
        (gf,) = torch.autograd.grad(out[0], [f])
        lsp[k] = dict(loss=out[0].detach(), loss_cls=out[1].detach(), loss_aux=out[2].detach(), d_feat_rows=gf[rows_l].clone(),
                      d_feat_norm=gf.double().norm())
    torch.save(dict(input_checksum=R2.checksum(lw["feat"], lw["t_feat"], sub_ei), max_segment=int(seg.max()), cases=lsp),
               OUT / "lsp_wide.pt")

    # ------------------------------------------------------------------ the reference's DGL GATConv at the teacher's shape
    mg.install_dgl_stubs()
    sys.path.insert(0, str(REF / "arxiv_dgl"))
    dgl_models = importlib.import_module("models")
    gw = R2.gat_wide()
    graph = mg._DGLGraph(gw["col"], gw["row"], gw["n"])
    torch.manual_seed(6)
    layer = dgl_models.GATConv(32, 250, num_heads=3, residual=True, use_symmetric_norm=True, use_attn_dst=True)
    layer.train()
    xin = gw["x"].clone().requires_grad_(True)
    out = layer(graph, xin)
    (out * gw["w"]).sum().backward()
    torch.save(dict(input_checksum=R2.checksum(gw["x"], gw["w"], gw["col"]), max_degree=gw["max_degree"],
                    state={k: v.detach().clone() for k, v in layer.state_dict().items()},
                    out_rows=out.detach()[gw["rows"]].clone(), out_norm=out.detach().double().norm(),
                    d_x=xin.grad.detach().clone(), grads={k: p.grad.detach().clone() for k, p in layer.named_parameters()}),
               OUT / "gat_wide.pt")
    print("wrote", sorted(p.name for p in OUT.glob("*.pt")))


if __name__ == "__main__":
    main()
