"""Time LSP in the R-GCN student step (the reference's MAG ``--training lpw``, mag_pyg/gnn_kd_and_aux.py:174-268) on GraphSAINT
batches of the MAG-shaped synthetic at scale 1, built as tools/bench_rgcn.py builds it: 20,000 roots, walk_length 2, the
student 2 x 32 against a 3 x 512 teacher that runs on the student's batch.

Arms, on the same batches, each step ending in a device synchronise:
  lsp_fused     RGCNTrainer(..., lsp=BatchLSP(32, kernel, beta)).train_step(b, x, teacher=t)
  lsp_eager     today's route: t.forward(b, x, training=False) (its own plan), nn.subgraph, then
                train_step(b, x, teacher_logits=..., aux=lambda f: criterion.lpw_criterion(...)[2], beta=beta)
  kd_teacher    the KD-only step with teacher=t (one plan per batch, teacher logits read in place)
  kd_logits     the KD-only step after a separate t.forward (a second plan, the logits scattered into an [N, C] buffer)
The arms run in turn for --rounds rounds, so the spread between rounds shows the noise.  Prints one JSON line: ms/step and
b200gnn launches/step per arm, the mean train rows and train-induced edges per batch, and the GPU's name and power limit.

    python tools/bench_mag_lsp.py [--steps 10] [--warmup 3] [--rounds 2] [--kernel rbf] [--beta 1]
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--batch-size", type=int, default=20000)
    ap.add_argument("--kernel", default="rbf")
    ap.add_argument("--beta", type=float, default=1.0)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mag_lsp needs a CUDA device")
    import efficient_gnns_b200  # noqa: F401
    from bench_rgcn import mag_graph
    from efficient_gnns_b200 import criterion, lib, nn, sampling
    from efficient_gnns_b200.lsp import BatchLSP
    from efficient_gnns_b200.rgcn import RGCNTrainer
    torch.cuda.set_device(0)
    data, x, num_nodes, relations, C = mag_graph(args.scale)
    x = {k: v.cuda() for k, v in x.items()}
    R = len(relations)
    n_batches = args.steps + args.warmup
    bs = list(sampling.GraphSAINTRandomWalkSampler(data, batch_size=args.batch_size, walk_length=2, num_steps=n_batches, seed=0))

    def trainer(H, L, seed, lsp=None):
        return RGCNTrainer(128, H, C, L, 0.5, num_nodes, list(x), R, relations, lr=0.005, seed=seed, lsp=lsp)

    teacher = trainer(512, 3, 0)
    fused = trainer(32, 2, 1, BatchLSP(32, args.kernel, args.beta))
    eager, kd_t, kd_l = trainer(32, 2, 1), trainer(32, 2, 1), trainer(32, 2, 1)

    def eager_step(b):
        tm = b.train_mask
        tl = teacher.forward(b, x, training=False)[tm]
        t_feat = teacher.out_feat()
        ei = nn.subgraph(tm, b.edge_index, relabel_nodes=True)[0]
        n = tl.shape[0]
        dummy = torch.zeros(n, 2, device="cuda"), torch.zeros(n, dtype=torch.long, device="cuda")
        eager.train_step(b, x, teacher_logits=tl, beta=args.beta, aux=lambda f: criterion.lpw_criterion(
            *dummy, f[tm], t_feat[tm], ei, args.kernel, 1)[2])

    arms = {
        "lsp_fused": lambda b: fused.train_step(b, x, teacher=teacher),
        "lsp_eager": eager_step,
        "kd_teacher": lambda b: kd_t.train_step(b, x, teacher=teacher),
        "kd_logits": lambda b: kd_l.train_step(b, x, teacher_logits=teacher.forward(b, x, training=False)[b.train_mask]),
    }

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

    result = {"metric": "mag_lsp_step", "batch_size": args.batch_size, "scale": args.scale, "steps": args.steps,
              "kernel": args.kernel, "beta": args.beta}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name(0)
    result["batch_nodes"] = round(sum(b.num_nodes for b in bs) / len(bs))
    result["train_rows"] = round(sum(int(b.train_mask.sum()) for b in bs) / len(bs))
    result["induced_edges"] = round(sum(sampling.induced_edges(b.edge_index, b.train_mask).shape[1] for b in bs) / len(bs))
    for r in range(args.rounds):
        for name, fn in arms.items():
            ms, launches = timed(fn)
            result.setdefault(f"{name}_ms", []).append(round(ms, 3))
            result[f"{name}_launches"] = launches
    print(json.dumps(result))


if __name__ == "__main__":
    main()
