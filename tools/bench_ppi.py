"""Time the fused PPI GAT step (engine_ppi) against the module path on the PPI-shaped synthetic.

    python tools/bench_ppi.py [--epochs 5] [--scale 1.0] [--json out.json]

Arms, on the 20 training graphs of synthetic.make_ppi_graphs(scale):
  * student kd   : engine_ppi.student with fixed teacher logits, one CUDA graph replay per training graph;
  * teacher sup  : engine_ppi.teacher, supervised, graph replays;
  * module path  : the same models composed here from nn.GATConv + torch.nn.Linear + F.elu with torch.optim.Adam and
                   kd_criterion / BCE under autograd, one graph per step as gnn.py's train() runs them.
Reports the median ms per step and per epoch (CUDA events around each epoch), the b200gnn launches per fused step, and the
GPU name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import engine_ppi, lib, synthetic  # noqa: E402
from efficient_gnns_b200 import nn as enn  # noqa: E402


class ModuleNet(torch.nn.Module):
    def __init__(self, layers, fin):
        super().__init__()
        for i, (H, D, concat) in enumerate(layers, start=1):
            out = H * D if concat else D
            setattr(self, f"conv{i}", enn.GATConv(fin, D, heads=H, concat=concat))
            setattr(self, f"lin{i}", torch.nn.Linear(fin, out))
            fin = out
        self.L = len(layers)

    def forward(self, x, ei):
        for i in range(1, self.L + 1):
            z = getattr(self, f"conv{i}")(x, ei) + getattr(self, f"lin{i}")(x)
            x = F.elu(z) if i < self.L else z
        return x


def timed_epochs(run_epoch, epochs: int):
    run_epoch(-1)                                      # warm-up epoch: every shape, plans, allocator
    torch.cuda.synchronize()
    out = []
    for e in range(epochs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run_epoch(e)
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return out


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_ppi measures on a CUDA device"
    graphs = synthetic.make_ppi_graphs("train", 0, args.scale)
    n_g = len(graphs)
    dev = torch.device("cuda")
    gen = torch.Generator().manual_seed(1)
    teach = [torch.randn(g[0].shape[0], 121, generator=gen) * 2 for g in graphs]
    dgr = [(x.to(dev), y.to(dev), ei.to(dev)) for x, y, ei in graphs]
    teach_d = [t.to(dev) for t in teach]
    res = dict(gpu=gpu_info(), scale=args.scale, n_graphs=n_g, nodes=[int(g[0].shape[0]) for g in graphs], epochs=args.epochs)
    for name, make, kd in (("student_kd", engine_ppi.student, True), ("teacher_sup", engine_ppi.teacher, False)):
        tr = make(graphs, teacher_logits=teach if kd else None)
        res[f"{name}_launches_per_step"] = tr.launches_per_step(0)
        tr.capture()
        fused = timed_epochs(lambda e: tr.train_epoch(max(e, 0)), args.epochs)
        layers = tr.layers
        m = ModuleNet(layers, 50).to(dev)
        m.load_state_dict({k: v for k, v in tr.state_dict().items()})
        opt = torch.optim.Adam(m.parameters(), lr=0.005)

        def module_epoch(e):
            order = tr.epoch_order(max(e, 0))
            for i in order:
                x, y, ei = dgr[i]
                out = m(x, ei)
                if kd:
                    t = teach_d[i]
                    loss = F.binary_cross_entropy_with_logits(out, torch.sigmoid(t)) * 0.5 + \
                        F.binary_cross_entropy_with_logits(out, y) * 0.5
                else:
                    loss = F.binary_cross_entropy_with_logits(out, y)
                opt.zero_grad()
                loss.backward()
                opt.step()
        before = lib.launch_count()
        module_epoch(0)
        torch.cuda.synchronize()
        res[f"{name}_module_launches_per_step"] = (lib.launch_count() - before) / n_g
        module = timed_epochs(module_epoch, args.epochs)
        for arm, ts in (("fused", fused), ("module", module)):
            med = statistics.median(ts)
            res[f"{name}_{arm}_ms_per_epoch"] = round(med, 3)
            res[f"{name}_{arm}_ms_per_step"] = round(med / n_g, 4)
            res[f"{name}_{arm}_ms_per_epoch_range"] = [round(min(ts), 3), round(max(ts), 3)]
        res[f"{name}_speedup"] = round(statistics.median(module) / statistics.median(fused), 3)
        del tr, m, opt
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
