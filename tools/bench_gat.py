"""Time the fused GAT training step (engine_gat.GATTrainer, CUDA-graph replay) against the module path: the same model
composed of nn.DGLGATConv, torch BatchNorm1d / dropout, autograd and torch.optim.Adam on the same graph and GPU.

    python tools/bench_gat.py [--steps 10] [--warmup 3] [--rounds 3] [--profile DIR] [--out result.json]

Input: the ARXIV-shape synthetic graph made bidirected with self-loops (arxiv_dgl/gat.py:61,66), 128 -> 2 hidden layers -> 40,
dropout 0.75, input_drop 0.1, edge_drop 0.1, symmetric normalisation, at 8 heads of 32 and at 3 heads of 250 (the teacher
shape), supervised and with logit KD.  The arms are alternated round by round in one process after a warm-up; the result is
the median step time of each arm with the range over the rounds, the card name and power limit read in the same run, and
the launches per step, as one JSON line.  --profile DIR runs torch.profiler over a few replays instead (a run of its own:
tracing slows the host) and writes a per-kernel table with the algorithmic bytes over kernel time as a share of the H100
SXM's 3.35 TB/s HBM3 figure for the HBM-bound sparse kernels.  Needs a GPU; reads nothing outside the repository.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import nn as enn, sparse  # noqa: E402
from efficient_gnns_b200.engine_gat import GATTrainer  # noqa: E402
from efficient_gnns_b200.synthetic import ARXIV, make_node_dataset  # noqa: E402
from oracle import graph as og  # noqa: E402

HBM_PEAK = 3.35e12
P, P_IN, P_EDGE, LAYERS = 0.75, 0.1, 0.1, 3


class ModuleGAT(torch.nn.Module):
    """The reference's GAT (arxiv_dgl/models.py:239-313) composed of this package's DGLGATConv module."""

    def __init__(self, in_feats, n_classes, n_hidden, n_heads):
        super().__init__()
        self.convs, self.norms = torch.nn.ModuleList(), torch.nn.ModuleList()
        for i in range(LAYERS):
            last = i == LAYERS - 1
            self.convs.append(enn.DGLGATConv(n_heads * n_hidden if i else in_feats, n_classes if last else n_hidden,
                                             num_heads=1 if last else n_heads, edge_drop=P_EDGE, residual=True, use_symmetric_norm=True))
            if not last:
                self.norms.append(torch.nn.BatchNorm1d(n_heads * n_hidden))
        self.bias_last = torch.nn.Parameter(torch.zeros(n_classes))

    def forward(self, adj, x):
        h = torch.nn.functional.dropout(x, P_IN, self.training)
        for i, conv in enumerate(self.convs):
            h = conv(adj, h)
            if i < LAYERS - 1:
                h = torch.nn.functional.dropout(torch.relu(self.norms[i](h.flatten(1))), P, self.training)
        return h.mean(1) + self.bias_last


def timed(fn, steps):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile", default=None, help="directory for the per-kernel table (torch.profiler; no end-to-end timing)")
    ap.add_argument("--out", default=None, help="also write the JSON result line to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_gat measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    result = {"metric": "gat_train_step_ms", "gpu": smi.stdout.strip().splitlines()[0] if smi.returncode == 0
              else torch.cuda.get_device_name(0), "steps": args.steps, "rounds": args.rounds, "shapes": {}}

    ds = make_node_dataset(ARXIV, seed=0)
    n = ds.num_nodes
    r, c, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(r, c, n)
    rs, cs, _ = og.fill_diag(r, c, np.ones(r.shape[0], dtype=np.float32), n)
    adj = sparse.SparseTensor(row=torch.from_numpy(rs).to(dev), col=torch.from_numpy(cs).to(dev), sparse_sizes=(n, n), is_sorted=True)
    x, y = ds.x.to(dev), ds.y.view(-1).to(dev)
    teacher, idx = ds.teacher_logits.to(dev), ds.split_idx["train"].to(dev)
    result["graph"] = {"nodes": n, "nnz": int(rs.shape[0])}

    for H, D in ((8, 32), (3, 250)):
        for kd in (False, True):
            name = f"H{H}_D{D}_{'kd' if kd else 'supervised'}"
            t = teacher if kd else None
            tr = GATTrainer(adj, x.shape[1], ds.num_classes, D, LAYERS, H, dropout=P, input_drop=P_IN, edge_drop=P_EDGE,
                            use_attn_dst=False, use_symmetric_norm=True, lr=2e-3)
            tr.capture(x, y, idx, t, warmup=args.warmup)
            if args.profile:
                profile(tr, name, Path(args.profile))
                del tr
                torch.cuda.empty_cache()
                continue
            model = ModuleGAT(x.shape[1], ds.num_classes, D, H).to(dev)
            for conv in model.convs:
                conv.attn_r = None                                   # use_attn_dst=False, as the engine arm
            opt = torch.optim.Adam(model.parameters(), lr=2e-3)

            def module_step():
                model.train()
                opt.zero_grad(set_to_none=True)
                z = model(adj, x)[idx]
                loss = torch.nn.functional.cross_entropy(z, y[idx])
                if kd:
                    kl = torch.nn.functional.kl_div(torch.log_softmax(z / 4.0, 1), torch.softmax(t[idx] / 4.0, 1))
                    loss = kl * (0.9 * 16.0) + loss * 0.1
                loss.backward()
                opt.step()
            for _ in range(args.warmup):
                module_step()
            eng, mod = [], []
            for _ in range(args.rounds):
                eng.append(timed(tr.replay, args.steps))
                mod.append(timed(module_step, args.steps))
            result["shapes"][name] = {
                "engine_ms_median": statistics.median(eng), "engine_ms_range": [min(eng), max(eng)],
                "module_ms_median": statistics.median(mod), "module_ms_range": [min(mod), max(mod)],
                "speedup": statistics.median(mod) / statistics.median(eng), "launches_per_step": tr.launches_per_step(),
                "stored_head_width": tr.Dp[0], "useful_gemm_flop": tr.useful_flop(), "loss": float(tr.loss_out[0])}
            del tr, model, opt
            torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


def profile(tr: GATTrainer, name: str, out_dir: Path, steps: int = 5):
    """Per-kernel device time of `steps` graph replays; algorithmic bytes (from shapes) over time for the sparse kernels."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    out_dir.mkdir(parents=True, exist_ok=True)
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            tr.replay()
        torch.cuda.synchronize()
    rows = sorted(((e.key, e.count, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0),
                  key=lambda t: -t[2])
    total = sum(t for _, _, t in rows)
    nbytes = tr.algorithmic_bytes()
    key = {"gat_aggregate_epi_kernel": "gat_aggregate_epi", "gat_scores_kernel": "gat_scores", "gat_scores_bwd_kernel": "gat_scores_bwd",
           "gat_edge_softmax_kernel": "gat_edge_softmax"}
    lines = [f"# {name}: {steps} replays, {total / steps / 1e3:.3f} ms of kernels per step", "kernel | calls/step | us/call | share | bytes/time of 3.35 TB/s"]
    for k, cnt, t in rows[:24]:
        share = ""
        for frag, b in key.items():
            if frag in k and "finalize" not in k:
                share = f"{nbytes[b] / (t / cnt * 1e-6) / HBM_PEAK:.1%} (hidden-width bytes; HBM-bound)"
        lines.append(f"{k[:90]} | {cnt / steps:.1f} | {t / cnt:.1f} | {t / total:.1%} | {share}")
    (out_dir / f"gat_kernels_{name}.txt").write_text("\n".join(lines) + "\n")
    print("\n".join(lines))


if __name__ == "__main__":
    main()
