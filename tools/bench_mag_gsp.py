"""Time GSP in the R-GCN student step (the reference's MAG ``--training gpw``, mag_pyg/gnn_kd_and_aux.py:174-268) on
GraphSAINT batches of the MAG-shaped synthetic at scale 1, built as tools/bench_rgcn.py builds it: 20,000 roots, walk_length
2, the student 2 x 32 against a 3 x 512 teacher that runs on the student's batch, the MAG script's settings (beta 1,
lr 0.005) for each --kernels and --max-samples.

Arms, on the same batches, each step ending in a device synchronise:
  gsp_fused_<kernel>_<S>   RGCNTrainer(..., gsp=BatchGSP(32, 512, kernel, 1, S)).train_step(b, x, teacher=t)
  gsp_eager_<kernel>_<S>   the route without gsp=: t.forward(b, x, training=False) (its own plan), then train_step(b, x,
                           teacher_logits=..., aux=lambda f: criterion.gpw_criterion(...)[2]) with host autograd; numpy
                           draws the sample, as the reference does
  kd_teacher               the KD-only step with teacher=t
The arms run in turn for --rounds rounds, so the spread between rounds shows the noise.  Prints one JSON line: ms/step and
b200gnn launches/step per arm, the mean train rows per batch, and the GPU's name and power limit.

--profile adds a separate torch.profiler pass of one fused step per (kernel, S) and reports the GPU time of the GSP parts
in that step: the student and the teacher Gram GEMMs (per chunk, the two GEMMs launched before the pair pass: student
first), the pair pass, the contraction (both launches), and the contraction's share of its fp32 FMA bound 2 S^2 H / 67
TFLOP/s (the H100 SXM data sheet's FP32 rate).

    python tools/bench_mag_gsp.py [--steps 10] [--warmup 3] [--rounds 2] [--kernels poly cosine]
                                  [--max-samples 24576 16384] [--profile]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

FP32_PEAK = 67e12          # H100 SXM data sheet, dense FP32


def gsp_kernel_times(trace_path: str) -> dict:
    """GPU time (ms) of the GSP parts of a profiled step from its chrome trace: the GEMM launches right before each pair pass
    are the chunk's student (first) and teacher (second) Gram GEMMs."""
    with open(trace_path) as fh:
        events = json.load(fh)["traceEvents"]
    kernels = sorted((e for e in events if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    out = dict(student_gram=0.0, teacher_gram=0.0, pair=0.0, contraction=0.0, chunks=0)
    for i, e in enumerate(kernels):
        name = e["name"]
        if "gsp_pair_kernel" in name:
            out["pair"] += e["dur"]
            out["chunks"] += 1
            out["teacher_gram"] += kernels[i - 1]["dur"]
            out["student_gram"] += kernels[i - 2]["dur"]
            assert "gemm" in kernels[i - 1]["name"] and "gemm" in kernels[i - 2]["name"], (kernels[i - 2]["name"],
                                                                                          kernels[i - 1]["name"])
        elif "gsp_contract" in name:
            out["contraction"] += e["dur"]
    return {k: (round(v / 1e3, 3) if k != "chunks" else v) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--batch-size", type=int, default=20000)
    ap.add_argument("--kernels", nargs="+", default=["poly", "cosine"])
    ap.add_argument("--max-samples", type=int, nargs="+", default=[24576, 16384])
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mag_gsp needs a CUDA device")
    import efficient_gnns_b200  # noqa: F401
    from bench_rgcn import mag_graph
    from efficient_gnns_b200 import criterion, lib, sampling
    from efficient_gnns_b200.gsp import BatchGSP
    from efficient_gnns_b200.rgcn import RGCNTrainer
    torch.cuda.set_device(0)
    data, x, num_nodes, relations, C = mag_graph(args.scale)
    x = {k: v.cuda() for k, v in x.items()}
    R = len(relations)
    n_batches = args.steps + args.warmup
    bs = list(sampling.GraphSAINTRandomWalkSampler(data, batch_size=args.batch_size, walk_length=2, num_steps=n_batches, seed=0))
    lr, beta, H = 0.005, 1.0, 32

    def trainer(hidden, L, seed, gsp=None):
        return RGCNTrainer(128, hidden, C, L, 0.5, num_nodes, list(x), R, relations, lr=lr, seed=seed, gsp=gsp)

    teacher = trainer(512, 3, 0)
    kd_t = trainer(H, 2, 1)
    np.random.seed(0)

    def eager_arm(kernel, S):
        tr = trainer(H, 2, 1)

        def step(b):
            tm = b.train_mask
            tl = teacher.forward(b, x, training=False)[tm]
            t_feat = teacher.out_feat()
            n = tl.shape[0]
            dummy = torch.zeros(n, 2, device="cuda"), torch.zeros(n, dtype=torch.long, device="cuda")
            tr.train_step(b, x, teacher_logits=tl, beta=beta, aux=lambda f: criterion.gpw_criterion(
                *dummy, f[tm], t_feat[tm], kernel, 1, S)[2])
        return step

    def timed(fn):
        for b in bs[:args.warmup]:
            fn(b)
        torch.cuda.synchronize()
        lib.reset_launch_count()
        total = 0.0
        for b in bs[args.warmup:]:
            t0 = time.perf_counter()
            fn(b)
            torch.cuda.synchronize()
            total += time.perf_counter() - t0
        return total * 1e3 / args.steps, lib.launch_count() / args.steps

    result = {"metric": "mag_gsp_step", "batch_size": args.batch_size, "scale": args.scale, "steps": args.steps, "beta": beta}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name(0)
    rows = [int(b.train_mask.sum()) for b in bs[args.warmup:]]
    result["batch_nodes"] = round(sum(b.num_nodes for b in bs) / len(bs))
    result["train_rows"] = round(sum(rows) / len(rows))
    result["train_rows_min_max"] = [min(rows), max(rows)]
    arms = {"kd_teacher": lambda b: kd_t.train_step(b, x, teacher=teacher)}
    fused_of = {}
    for kernel in args.kernels:
        for S in args.max_samples:
            result[f"drawn_fraction_{S}"] = round(sum(n > S for n in rows) / len(rows), 3)
            fused = fused_of[kernel, S] = trainer(H, 2, 1, BatchGSP(H, 512, kernel, beta, S))
            arms[f"gsp_fused_{kernel}_{S}"] = lambda b, fused=fused: fused.train_step(b, x, teacher=teacher)
            arms[f"gsp_eager_{kernel}_{S}"] = eager_arm(kernel, S)
    for r in range(args.rounds):
        for name, fn in arms.items():
            ms, launches = timed(fn)
            result.setdefault(f"{name}_ms", []).append(round(ms, 3))
            result[f"{name}_launches"] = launches
    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        b = bs[args.warmup]
        S_b = int(b.train_mask.sum())
        prof_out = {}
        with tempfile.TemporaryDirectory() as tmp:
            for (kernel, S), fused in fused_of.items():
                fused.train_step(b, x, teacher=teacher)
                torch.cuda.synchronize()
                with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                    fused.train_step(b, x, teacher=teacher)
                    torch.cuda.synchronize()
                path = os.path.join(tmp, f"{kernel}_{S}.json")
                prof.export_chrome_trace(path)
                t = gsp_kernel_times(path)
                s = min(S, S_b)
                t["S"] = s
                t["contraction_fp32_bound_ms"] = round(2.0 * s * s * H / FP32_PEAK * 1e3, 3)
                t["contraction_share_of_bound"] = round(t["contraction_fp32_bound_ms"] / max(t["contraction"], 1e-9), 3)
                prof_out[f"{kernel}_{S}"] = t
        result["profile_ms"] = prof_out
    print(json.dumps(result))


if __name__ == "__main__":
    main()
