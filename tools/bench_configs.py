"""Secondary measurements for BASELINE configs 3-5 through the module / criterion path (not the contract benchmark):
   config 3  3-layer GraphSAGE student + G-CRD (S=8192 / 16384, proj 256) on the ARXIV-shape graph: full training step
   config 4  one GAT layer (H=8, D=32) forward+backward and the LSP-cosine loss on the train-induced subgraph
   config 5  R-GCN style aggregation on the MAG-shape graph: 7 rectangular mean-SpMMs (K=128), forward+backward
Each line is JSON; timings are CUDA events, median of `iters` after warm-up."""
import json
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import criterion as C, nn as bnn, sparse, synthetic  # noqa: E402


def med_time(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


class Student(torch.nn.Module):
    def __init__(self, conv, dims, dropout=0.5):
        super().__init__()
        self.convs = torch.nn.ModuleList([conv(dims[i], dims[i + 1]) for i in range(len(dims) - 1)])
        self.bns = torch.nn.ModuleList([torch.nn.BatchNorm1d(d) for d in dims[1:-1]])
        self.dropout = dropout

    def forward(self, x, adj):
        for conv, bn in zip(self.convs[:-1], self.bns):
            x = F.dropout(F.relu(bn(conv(x, adj))), p=self.dropout, training=self.training)
            self.out_feat = x
        return self.convs[-1](x, adj)


def main():
    only = int(sys.argv[sys.argv.index("--only") + 1]) if "--only" in sys.argv else None
    dev = "cuda"
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.to(dev)
    perm = (ei[1] * n + ei[0]).argsort()
    adj = sparse.SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    x, y = ds.x.to(dev), ds.y.squeeze(1).to(dev)
    idx = ds.split_idx["train"].to(dev)
    t_feat = ds.teacher_feat.to(dev)
    nnz = adj.nnz()

    # ---- config 3: SAGE + G-CRD
    for S in (8192, 16384) if only in (None, 3) else ():
        torch.manual_seed(0)
        model = Student(bnn.SAGEConv, [128, 256, 256, 40]).to(dev)
        sproj = torch.nn.Sequential(bnn.Linear(256, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).to(dev)
        tproj = torch.nn.Sequential(bnn.Linear(750 + 2, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).to(dev)
        tf = F.pad(t_feat, (0, 2))            # 750 -> 752: row pitch multiple of 16 bytes for the TMA GEMM
        opt = torch.optim.Adam(list(model.parameters()) + list(sproj.parameters()) + list(tproj.parameters()), lr=0.01)

        def step():
            out = model(x, adj)[idx]
            loss, _, _ = C.nce_criterion(out, y[idx], sproj(model.out_feat[idx]), tproj(tf[idx]), 0.1, 0.075, S)
            opt.zero_grad(); loss.backward(); opt.step()
        ms = med_time(step, 8, 3)
        print(json.dumps(dict(config=3, what="3-layer SAGE + G-CRD full step (module path, autograd, torch Adam/BN)", S=S,
                              nnz_sym=nnz, ms_per_step=ms, edges_per_s=6 * nnz / ms * 1e3)), flush=True)

    # ---- config 3 on the fused engine (engine_sage.SAGEStudentTrainer): no autograd tape, no torch BN/Adam on the student
    if only in (None, 3):
        from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
        tl = ds.teacher_logits.to(dev)
        for S in (8192, 16384):
            torch.manual_seed(0)
            tr = SAGEStudentTrainer(adj, [128, 256, 256, 40], dropout=0.5, lr=0.01, seed=0)
            sproj = torch.nn.Sequential(bnn.Linear(256, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).to(dev)
            tproj = torch.nn.Sequential(bnn.Linear(752, 256), torch.nn.BatchNorm1d(256), torch.nn.ReLU()).to(dev)
            tf = F.pad(t_feat, (0, 2))
            opt = torch.optim.Adam(list(sproj.parameters()) + list(tproj.parameters()), lr=0.01)

            def aux(f):
                return C.nce_criterion(tr.Y[-1][idx], y[idx], sproj(f[idx]), tproj(tf[idx]), 1.0, 0.075, S)[2]

            def step():
                opt.zero_grad()
                tr.train_step(x, y, idx, tl, aux=aux, beta=0.1)
                opt.step()
            ms = med_time(step, 8, 3)
            print(json.dumps(dict(config=3, what="3-layer SAGE + kd + G-CRD full step on the FUSED engine (student: b200gnn kernels only; "
                                                 "projection heads + their Adam on the module path), chunked InfoNCE without the SxS logits", S=S,
                                  nnz_sym=nnz, ms_per_step=ms, edges_per_s=6 * nnz / ms * 1e3)), flush=True)
        tr = SAGEStudentTrainer(adj, [128, 256, 256, 40], dropout=0.5, lr=0.01, seed=0)
        tr.capture(x, y, idx, tl, warmup=2)
        ms = med_time(lambda: tr.replay(), 20, 5)
        print(json.dumps(dict(config=3, what="3-layer SAGE + logit-KD, fused engine, CUDA graph (the configs[1] step with SAGEConv)",
                              nnz_sym=nnz, ms_per_step=ms, edges_per_s=6 * nnz / ms * 1e3)), flush=True)
        del tr
        torch.cuda.empty_cache()

    # ---- config 4: GAT layer + LSP
    adj_sl = bnn._fill_diag_pattern(adj)
    if only not in (None, 4, 5):
        return
    for H, D in ((8, 32), (3, 250)) if only in (None, 4) else ():
        torch.manual_seed(0)
        layer = bnn.DGLGATConv(128, D, num_heads=H, use_symmetric_norm=True).to(dev)

        def gat_step():
            out = layer(adj_sl, x)
            layer.zero_grad(); out.sum().backward()
        ms = med_time(gat_step, 8, 3)
        print(json.dumps(dict(config=4, what="DGL-style GATConv layer fwd+bwd (fc + edge softmax + multi-head aggregation)",
                              heads=H, head_dim=D, nnz=adj_sl.nnz(), ms=ms, edges_per_s=2 * adj_sl.nnz() / ms * 1e3)), flush=True)
    r, c, _ = adj.coo()
    sub, _ = bnn.subgraph(idx, torch.stack([r, c]), relabel_nodes=True)
    feat = torch.randn(idx.numel(), 256, device=dev, requires_grad=True)
    tsub = t_feat[idx].contiguous()
    z = torch.randn(idx.numel(), 40, device=dev, requires_grad=True)

    def lsp_step():
        loss, _, _ = C.lpw_criterion(z, y[idx], feat, tsub, sub, "cosine", 100)
        feat.grad = None; loss.backward()
    ms = med_time(lsp_step, 8, 3) if only in (None, 4) else 0.0
    if only in (None, 4):
        print(json.dumps(dict(config=4, what="LSP cosine (student 256-d, teacher 750-d) fwd+bwd on the train-induced subgraph",
                              E_sub=int(sub.shape[1]), ms=ms,
                              reference_materialised_bytes=int(sub.shape[1]) * (256 + 750) * 2 * 4)), flush=True)
    if only not in (None, 5):
        return

    # ---- config 5: MAG-shape per-relation mean aggregation (RGCN.inference formulation, mag_pyg/gnn.py:153-169)
    rels = []
    for i, ((s, _, d), e) in enumerate(synthetic.MAG_RELATIONS.items()):
        eidx = synthetic.mag_relation_edges(s, d, e, seed=i)
        rels.append((s, d, eidx))
        if s != d:
            rels.append((d, s, eidx.flip(0)))
        else:
            rels[-1] = (s, d, torch.cat([eidx, eidx.flip(0)], 1))       # cites made undirected
    feats = {k: torch.randn(v, 128, device=dev, requires_grad=True) for k, v in synthetic.MAG_NODES.items()}
    adjs = []
    tot = 0
    for s, d, eidx in rels:
        a = sparse.SparseTensor(row=eidx[1].to(dev), col=eidx[0].to(dev),
                                sparse_sizes=(synthetic.MAG_NODES[d], synthetic.MAG_NODES[s]), is_sorted=False).coalesce()
        a.storage.engine_csr_unweighted(); a.storage.engine_csc("mean")
        adjs.append((s, d, a)); tot += a.nnz()

    def mag_step():
        outs = {k: 0 for k in feats}
        total = 0
        for s, d, a in adjs:
            total = total + a.matmul(feats[s], reduce="mean").sum()
        for f in feats.values():
            f.grad = None
        total.backward()
    ms = med_time(mag_step, 5, 2)
    print(json.dumps(dict(config=5, what="MAG-shape: 7 relation-wise rectangular mean-SpMMs K=128, fwd+bwd (one R-GCN layer's aggregation)",
                          relations=len(adjs), nnz_total=tot, ms=ms, edges_per_s=2 * tot / ms * 1e3)), flush=True)

    # ---- config 5b: the full-batch R-GCN engine (rgcn.RGCNInference = RGCN.inference, mag_pyg/gnn.py:140-171), 2 layers
    from efficient_gnns_b200.rgcn import RGCNInference
    del feats, adjs
    torch.cuda.empty_cache()
    types = list(synthetic.MAG_NODES)
    key2int = {k: i for i, k in enumerate(types)}
    eid = {}
    for i, (s_, d_, eidx) in enumerate(rels):
        key = (s_, f"rel{i}", d_)
        eid[key] = eidx
        key2int[key] = i
    g = torch.Generator().manual_seed(0)
    for hidden in (64, 512):
        state = {}
        for t in types[1:]:
            state[f"emb_dict.{key2int[t]}"] = torch.randn(synthetic.MAG_NODES[t], 128, generator=g) * 0.1
        for li, (a, b) in enumerate(((128, hidden), (hidden, 349))):
            for r in range(len(rels)):
                state[f"convs.{li}.rel_lins.{r}.weight"] = torch.randn(b, a, generator=g) * 0.05
            for t in range(len(types)):
                state[f"convs.{li}.root_lins.{t}.weight"] = torch.randn(b, a, generator=g) * 0.05
                state[f"convs.{li}.root_lins.{t}.bias"] = torch.zeros(b)
        eng = RGCNInference(state, {key2int[t]: n_ for t, n_ in synthetic.MAG_NODES.items()}, eid, key2int)
        xp = torch.randn(synthetic.MAG_NODES[types[0]], 128, generator=g).to(dev)
        ms = med_time(lambda: eng({0: xp}), 5, 2)
        print(json.dumps(dict(config=5, what=f"MAG-shape full-batch R-GCN inference, 2 layers 128->{hidden}->349: 14 rectangular mean-SpMMs + "
                                             "22 wgmma GEMMs (relation GEMMs accumulate in the epilogue), CSRs built once",
                              relations=len(rels), nnz_total=eng.nnz, ms=ms, edges_per_s=2 * eng.nnz / ms * 1e3)), flush=True)
        del eng, state
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
