"""Per-kernel time of the benchmarked training step (bench.py's workload: 3-layer GCN 128-256-256-40 with logit-KD on
the ARXIV-shape synthetic graph, one CUDA-graph replay per step).

Builds the workload as bench.py does, captures the step, replays it under torch.profiler with CUDA activities and prints
one JSON line per kernel name, sorted by device time per step: {"kernel", "ms_per_step", "launches_per_step", "share"}.
The first line names the GPU and its power limit.  Kernels on the side stream overlap the critical path, so the shares
add up to more than the step time.  Tracing slows the host; take step times from bench.py, not from this tool.

    python tools/profile_step.py [--steps 20] [--warmup 10] [--trace DIR]
"""
import argparse
import json
import subprocess
import sys
from collections import defaultdict
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import lib, sparse, synthetic  # noqa: E402
from efficient_gnns_b200.engine import GCNStudentTrainer  # noqa: E402

DIMS = [128, 256, 256, 40]                   # bench.py's student


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = (f.strip() for f in out[torch.cuda.current_device()].split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {"gpu": torch.cuda.get_device_name(), "power_limit": "unknown"}


def build_trainer():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    lib.load()
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.to(dev)
    perm = (ei[1] * n + ei[0]).argsort()
    adj = sparse.SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    tr = GCNStudentTrainer(adj, DIMS, dropout=0.5, lr=0.01, seed=0)
    d = {"x": ds.x, "y": ds.y.squeeze(1).contiguous(), "t": ds.teacher_logits, "idx": ds.split_idx["train"]}
    d = {k: v.to(dev) for k, v in d.items()}
    tr.capture(d["x"], d["y"], d["idx"], d["t"], warmup=2)
    return tr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--trace", metavar="DIR", default=None, help="also write a Chrome trace there")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device")

    tr = build_trainer()
    for _ in range(args.warmup):
        tr.replay()
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(args.steps):
            tr.replay()
        torch.cuda.synchronize()

    us, count = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            us[ev.name] += ev.device_time
            count[ev.name] += 1
    total = sum(us.values())
    print(json.dumps({**gpu_info(), "steps": args.steps, "kernel_ms_per_step_sum": total / args.steps / 1e3}), flush=True)
    for name in sorted(us, key=us.get, reverse=True):
        print(json.dumps({"kernel": name, "ms_per_step": us[name] / args.steps / 1e3,
                          "launches_per_step": count[name] / args.steps, "share": us[name] / total}), flush=True)
    if args.trace:
        Path(args.trace).mkdir(parents=True, exist_ok=True)
        prof.export_chrome_trace(str(Path(args.trace) / "step.pt.trace.json"))


if __name__ == "__main__":
    main()
