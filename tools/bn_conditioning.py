"""How well conditioned are the BatchNorm statistics of the training engines?  (DESIGN.md §4.3)

bn_finalize forms var = Σy²/n - mean² in fp64 from fp32 slot sums, so the relative error of invstd grows like
gamma(L)·(1 + 3 (mean/std)²) / 2 (tests/test_batchnorm_gpu.py, stage C), L the longest fp32 addition chain of the slot
producer.  This script trains the GCN engine in the bench.py configuration, the SAGE student and the arxiv GAT engine on
the synthetic ARXIV-shape graph, reads mean and invstd out of every hidden layer's bn buffer every --every steps, and
prints per layer the maximum and the 99th percentile of (mean/std)² over columns and samples, with the invstd bound they
give at L = 336 (16 rows x 21 tiles: the 3xTF32 GEMM epilogue at 169,343 x 256 on 132 SMs, the longest chain of the
producers at this shape).  Columns with zero variance (the GAT head padding) are left out.

    python tools/bn_conditioning.py [--steps 200] [--every 10]
"""
from __future__ import annotations

import argparse
import math
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import sparse  # noqa: E402
from efficient_gnns_b200.engine import GCNStudentTrainer  # noqa: E402
from efficient_gnns_b200.engine_gat import GATTrainer  # noqa: E402
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer  # noqa: E402
from efficient_gnns_b200.synthetic import ARXIV, make_node_dataset  # noqa: E402
from oracle import graph as og  # noqa: E402

U = 2.0 ** -24
L_CHAIN = 336
EPS = 1e-5


def invstd_bound(r2: float) -> float:
    g = L_CHAIN * U / (1 - L_CHAIN * U)
    return g * (1 + 3 * r2) / 2


def sample(tr, acc):
    for l, bn in enumerate(tr.bn):
        mean, inv = bn[0].double(), bn[1].double()
        var = 1.0 / (inv * inv) - EPS
        live = var > 1e-3 * EPS                       # zero-variance columns (padding) carry no conditioning
        acc.setdefault(l, []).append(((mean[live] ** 2) / var[live]).cpu().numpy())


def run(name, tr, inputs, steps, every):
    tr.capture(*inputs, warmup=2)
    acc = {}
    for s in range(1, steps + 1):
        tr.replay()
        if s % every == 0:
            sample(tr, acc)
    torch.cuda.synchronize()
    for l, xs in sorted(acc.items()):
        r2 = np.concatenate(xs)
        mx, p99 = float(r2.max()), float(np.percentile(r2, 99))
        print(f"{name:5s} layer {l}: (mean/std)^2 max {mx:9.3g} (mean/std {math.sqrt(mx):7.3g}), p99 {p99:9.3g};  "
              f"invstd bound at the max {invstd_bound(mx):.2e}, at p99 {invstd_bound(p99):.2e}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--every", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bn_conditioning reads the engines' statistics on a GPU"
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True)
    print("gpu:", smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else torch.cuda.get_device_name(0))
    ds = make_node_dataset(ARXIV, seed=0)
    n = ds.num_nodes
    x, y = ds.x.to(dev), ds.y.view(-1).to(dev)
    t, idx = ds.teacher_logits.to(dev), ds.split_idx["train"].to(dev)

    ei = ds.edge_index.to(dev)
    perm = (ei[1] * n + ei[0]).argsort()
    adj = sparse.SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    run("GCN", GCNStudentTrainer(adj, [128, 256, 256, 40], dropout=0.5, lr=0.01, seed=0), (x, y, idx, t), args.steps,
        args.every)
    run("SAGE", SAGEStudentTrainer(adj, [128, 256, 256, 40], dropout=0.5, lr=0.01, seed=0), (x, y, idx, t), args.steps,
        args.every)

    r, c, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(r, c, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    adj_gat = sparse.SparseTensor(row=torch.from_numpy(rs).to(dev), col=torch.from_numpy(cs).to(dev), sparse_sizes=(n, n),
                                  is_sorted=True)
    run("GAT", GATTrainer(adj_gat, x.shape[1], ds.num_classes, 250, 3, 3, dropout=0.75, input_drop=0.1,
                          use_attn_dst=False, use_symmetric_norm=True, lr=2e-3), (x, y, idx, t), args.steps, args.every)


if __name__ == "__main__":
    main()
