"""Time one epoch of the arxiv GAT teacher (engine_gat_teacher.GATTeacherTrainer, one CUDA-graph replay) against the module
path: gat.py's ``train`` + ``evaluate`` written on this package's nn.DGLGATConv, torch BatchNorm1d / dropout, autograd and
torch.optim.RMSprop, on the same graph and GPU.

    python tools/bench_gat_teacher.py [--epochs 5] [--warmup 2] [--rounds 3] [--profile DIR] [--out result.json]

Input: the ARXIV-shape synthetic graph made bidirected with self-loops (SparseTensor.to_symmetric().fill_diag), the teacher
preset (use_labels, one label iteration, mask rate 0.5, no attn_dst, symmetric normalisation, 3 layers of 3 heads x 250,
dropout 0.75, input_drop 0.25, edge_drop 0.3, lr 0.002 with the 50-epoch warm-up).  An epoch is two training forwards,
one backward, the RMSprop step and two eval forwards (gat.py:116-183), plus the best-epoch snapshot on the engine side.
The arms are alternated round by round in one process after a warm-up; the result is the median epoch time of each arm
with the range over the rounds and the card name and power limit read in the same run, as one JSON line.  --profile DIR
runs torch.profiler over a few replays instead (a run of its own: tracing slows the host) and writes a per-kernel table.
Needs a GPU; reads nothing outside the repository.
"""
from __future__ import annotations

import argparse
import json
import math
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import lib, nn as enn, sparse  # noqa: E402
from efficient_gnns_b200.engine_gat_teacher import GATTeacherTrainer  # noqa: E402
from efficient_gnns_b200.synthetic import ARXIV, make_node_dataset  # noqa: E402
from oracle import graph as og  # noqa: E402

P, P_IN, P_EDGE, LAYERS, HEADS, HIDDEN, LR, MASK_RATE = 0.75, 0.25, 0.3, 3, 3, 250, 0.002, 0.5
EPSILON = 1 - math.log(2)


class ModuleGAT(torch.nn.Module):
    """The reference's GAT (arxiv_dgl/models.py:239-313) composed of this package's DGLGATConv module, no attn_dst."""

    def __init__(self, in_feats, n_classes):
        super().__init__()
        self.convs, self.norms = torch.nn.ModuleList(), torch.nn.ModuleList()
        for i in range(LAYERS):
            last = i == LAYERS - 1
            conv = enn.DGLGATConv(HEADS * HIDDEN if i else in_feats, n_classes if last else HIDDEN, num_heads=1 if last else HEADS,
                                  edge_drop=P_EDGE, residual=True, use_symmetric_norm=True)
            conv.attn_r = None
            self.convs.append(conv)
            if not last:
                self.norms.append(torch.nn.BatchNorm1d(HEADS * HIDDEN))
        self.bias_last = torch.nn.Parameter(torch.zeros(n_classes))

    def forward(self, adj, x):
        h = F.dropout(x, P_IN, self.training)
        for i, conv in enumerate(self.convs):
            h = conv(adj, h)
            if i < LAYERS - 1:
                h = F.dropout(torch.relu(self.norms[i](h.flatten(1))), P, self.training)
                self.feat = h
        return h.mean(1) + self.bias_last


def custom_loss(x, labels):
    return torch.mean(torch.log(EPSILON + F.cross_entropy(x, labels, reduction="none")) - math.log(EPSILON))


def timed(fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / n * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", default=None, help="directory for the per-kernel table (torch.profiler; no end-to-end timing)")
    ap.add_argument("--out", default=None, help="also write the JSON result line to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gat_teacher measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    result = {"metric": "gat_teacher_epoch_ms", "gpu": smi.stdout.strip().splitlines()[0] if smi.returncode == 0
              else torch.cuda.get_device_name(0), "epochs": args.epochs, "rounds": args.rounds}

    ds = make_node_dataset(ARXIV, seed=0)
    n, C = ds.num_nodes, ds.num_classes
    r, c, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(r, c, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    adj = sparse.SparseTensor(row=torch.from_numpy(rs).to(dev), col=torch.from_numpy(cs).to(dev), sparse_sizes=(n, n), is_sorted=True)
    x, y = ds.x.to(dev), ds.y.view(-1).to(dev)
    tri, vai, tei = (ds.split_idx[k].to(dev) for k in ("train", "valid", "test"))
    result["graph"] = {"nodes": n, "nnz": int(rs.shape[0])}

    tr = GATTeacherTrainer(adj, x, y, ds.split_idx, n_classes=C)
    for _ in range(args.warmup):
        tr.epoch()
    tr.capture()
    if args.profile:
        profile(tr, Path(args.profile))
        return

    model = ModuleGAT(x.shape[1] + C, C).to(dev)
    opt = torch.optim.RMSprop(model.parameters(), lr=LR)
    state = {"epoch": 0}

    def add_labels(idx):
        onehot = torch.zeros(n, C, device=dev)
        onehot[idx, y[idx]] = 1
        return torch.cat([x, onehot], dim=-1)

    def module_epoch():
        state["epoch"] += 1
        for g in opt.param_groups:                                           # adjust_learning_rate
            g["lr"] = LR * min(state["epoch"], 50) / 50
        model.train()                                                        # train(), gat.py:116-148
        mask = torch.rand(tri.shape, device=dev) < MASK_RATE
        pred_idx = tri[~mask]
        feat = add_labels(tri[mask])
        opt.zero_grad(set_to_none=True)
        pred = model(adj, feat)
        unlabel = torch.cat([pred_idx, vai, tei])
        pred = pred.detach()
        feat[unlabel, -C:] = F.softmax(pred[unlabel], dim=-1)
        pred = model(adj, feat)
        custom_loss(pred[pred_idx], y[pred_idx]).backward()
        opt.step()
        model.eval()                                                         # evaluate(), gat.py:151-183
        with torch.no_grad():
            feat = add_labels(tri)
            pred = model(adj, feat)
            unlabel = torch.cat([vai, tei])
            feat[unlabel, -C:] = F.softmax(pred[unlabel], dim=-1)
            pred = model(adj, feat)
            for i in (tri, vai, tei):
                custom_loss(pred[i], y[i])
                (pred[i].argmax(-1) == y[i]).float().mean()

    for _ in range(args.warmup):
        module_epoch()
    eng, mod = [], []
    for _ in range(args.rounds):
        eng.append(timed(tr.replay, args.epochs))
        mod.append(timed(module_epoch, args.epochs))
    before = lib.launch_count()
    tr.epoch()
    result.update({
        "engine_ms_median": statistics.median(eng), "engine_ms_range": [min(eng), max(eng)],
        "module_ms_median": statistics.median(mod), "module_ms_range": [min(mod), max(mod)],
        "speedup": statistics.median(mod) / statistics.median(eng), "launches_per_epoch": lib.launch_count() - before,
        "parameters": tr.n_parameters(), "val_loss": float(tr.row[6])})
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


def profile(tr: GATTeacherTrainer, out_dir: Path, epochs: int = 3):
    """Per-kernel device time of `epochs` graph replays."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    out_dir.mkdir(parents=True, exist_ok=True)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(epochs):
            tr.replay()
        torch.cuda.synchronize()
    rows = sorted(((e.key, e.count, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0),
                  key=lambda t: -t[2])
    total = sum(t for _, _, t in rows)
    lines = [f"# GAT teacher epoch: {epochs} replays, {total / epochs / 1e3:.3f} ms of kernels per epoch",
             "kernel | calls/epoch | us/call | share"]
    for k, cnt, t in rows[:24]:
        lines.append(f"{k[:90]} | {cnt / epochs:.1f} | {t / cnt:.1f} | {t / total:.1%}")
    (out_dir / "gat_teacher_kernels.txt").write_text("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
