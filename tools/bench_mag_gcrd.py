"""Time G-CRD in the R-GCN student step (the reference's MAG ``--training nce``, mag_pyg/gnn_kd_and_aux.py:174-277) on
GraphSAINT batches of the MAG-shaped synthetic at scale 1, built as tools/bench_rgcn.py builds it: 20,000 roots, walk_length
2, the student 2 x 32 against a 3 x 512 teacher that runs on the student's batch, the MAG script's settings (proj_dim 128,
nce_T 0.075, beta 0.1, lr 0.005) at each --max-samples.

Arms, on the same batches, each step ending in a device synchronise:
  gcrd_fused    RGCNTrainer(..., gcrd=BatchGCRD(32, 512, max_samples=S)).train_step(b, x, teacher=t)
  gcrd_eager    the route without gcrd=: t.forward(b, x, training=False) (its own plan), torch heads (nn.Sequential(Linear,
                BatchNorm1d, ReLU)) through train_step(b, x, teacher_logits=..., aux=lambda f: criterion.nce_criterion(...)[2])
                and a torch Adam on the heads; numpy draws the sample, as the reference does
  kd_teacher    the KD-only step with teacher=t
The arms run in turn for --rounds rounds, so the spread between rounds shows the noise.  Prints one JSON line: ms/step and
b200gnn launches/step per arm and max_samples, the mean train rows per batch, the fraction of batches that draw a sample
(n_train > max_samples), and the GPU's name and power limit.

    python tools/bench_mag_gcrd.py [--steps 10] [--warmup 3] [--rounds 2] [--max-samples 24576 16384]
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
    ap.add_argument("--max-samples", type=int, nargs="+", default=[24576, 16384])
    ap.add_argument("--proj-dim", type=int, default=128)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mag_gcrd needs a CUDA device")
    import efficient_gnns_b200  # noqa: F401
    from bench_rgcn import mag_graph
    from efficient_gnns_b200 import criterion, lib, sampling
    from efficient_gnns_b200.gcrd import BatchGCRD
    from efficient_gnns_b200.rgcn import RGCNTrainer
    torch.cuda.set_device(0)
    data, x, num_nodes, relations, C = mag_graph(args.scale)
    x = {k: v.cuda() for k, v in x.items()}
    R = len(relations)
    n_batches = args.steps + args.warmup
    bs = list(sampling.GraphSAINTRandomWalkSampler(data, batch_size=args.batch_size, walk_length=2, num_steps=n_batches, seed=0))
    lr, beta, nce_T, P = 0.005, 0.1, 0.075, args.proj_dim

    def trainer(H, L, seed, gcrd=None):
        return RGCNTrainer(128, H, C, L, 0.5, num_nodes, list(x), R, relations, lr=lr, seed=seed, gcrd=gcrd)

    teacher = trainer(512, 3, 0)
    kd_t = trainer(32, 2, 1)
    np.random.seed(0)

    def eager_arm(S):
        tr = trainer(32, 2, 1)
        sp = torch.nn.Sequential(torch.nn.Linear(32, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).cuda()
        tp = torch.nn.Sequential(torch.nn.Linear(512, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).cuda()
        opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=lr)

        def step(b):
            tm = b.train_mask
            tl = teacher.forward(b, x, training=False)[tm]
            t_feat = teacher.out_feat()
            n = tl.shape[0]
            dummy = torch.zeros(n, 2, device="cuda"), torch.zeros(n, dtype=torch.long, device="cuda")
            opt.zero_grad()
            tr.train_step(b, x, teacher_logits=tl, beta=beta, aux=lambda f: criterion.nce_criterion(
                *dummy, sp(f[tm]), tp(t_feat[tm]), 1.0, nce_T, S)[2])
            opt.step()
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

    result = {"metric": "mag_gcrd_step", "batch_size": args.batch_size, "scale": args.scale, "steps": args.steps,
              "proj_dim": P, "nce_T": nce_T, "beta": beta}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 and smi.stdout.strip() else torch.cuda.get_device_name(0)
    rows = [int(b.train_mask.sum()) for b in bs[args.warmup:]]
    result["batch_nodes"] = round(sum(b.num_nodes for b in bs) / len(bs))
    result["train_rows"] = round(sum(rows) / len(rows))
    result["train_rows_min_max"] = [min(rows), max(rows)]
    arms = {"kd_teacher": lambda b: kd_t.train_step(b, x, teacher=teacher)}
    for S in args.max_samples:
        result[f"drawn_fraction_{S}"] = round(sum(n > S for n in rows) / len(rows), 3)
        fused = trainer(32, 2, 1, BatchGCRD(32, 512, P, max_samples=S, nce_T=nce_T, beta=beta))
        arms[f"gcrd_fused_{S}"] = lambda b, fused=fused: fused.train_step(b, x, teacher=teacher)
        arms[f"gcrd_eager_{S}"] = eager_arm(S)
    for r in range(args.rounds):
        for name, fn in arms.items():
            ms, launches = timed(fn)
            result.setdefault(f"{name}_ms", []).append(round(ms, 3))
            result[f"{name}_launches"] = launches
    print(json.dumps(result))


if __name__ == "__main__":
    main()
