"""Time an epoch of the PPI student with G-CRD (ppi_pyg/gnn.py --training nce: BCE + beta * InfoNCE between the projected
student and teacher features of each graph) on the 20 training graphs of synthetic.make_ppi_graphs(scale), three arms
alternated epoch by epoch in one process:

    captured   engine_ppi.student with gcrd.PerGraphGCRD, one CUDA graph replay per training graph
    eager_aux  the same fused student with train_step(i, aux=lambda f: criterion_ppi.nce_criterion(..., sp(f), tp(t), ...)[2],
               beta), torch projection heads and a torch Adam over them
    module     the module path: StudentNet composed of nn.GATConv + torch.nn.Linear + F.elu under autograd, torch heads,
               criterion_ppi.nce_criterion and one torch.optim.Adam over the model and both heads, one graph per step as
               gnn.py's train() runs it

The teacher features are TeacherNet's out_feat [n, 1024] (engine_ppi.teacher(...).predict(..., return_feat=True)).  The
defaults are the scripts' (scripts/run.sh): beta 0.1, nce_T 0.075, max_samples 16384 (every node of a graph), proj_dim 256.

    python tools/bench_ppi_gcrd.py [--epochs 7] [--scale 1.0] [--max-samples 16384] [--json out.json]

One warm-up epoch per arm, then --epochs timed rounds (CUDA events around each epoch, profiler off).  Prints one JSON line:
median ms per epoch with range for each arm, b200gnn launches per captured step, and the card's name and power limit read
in the same run."""
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
sys.path.insert(0, str(Path(__file__).resolve().parent))
import efficient_gnns_b200  # noqa: E402,F401
from bench_ppi import ModuleNet  # noqa: E402
from efficient_gnns_b200 import criterion_ppi, engine_ppi, synthetic  # noqa: E402
from efficient_gnns_b200.gcrd import PerGraphGCRD  # noqa: E402


class StudentModule(ModuleNet):
    """bench_ppi's module-path StudentNet, keeping the last hidden activation as ``out_feat`` as gnn.py's classes do."""

    def forward(self, x, ei):
        for i in range(1, self.L + 1):
            z = getattr(self, f"conv{i}")(x, ei) + getattr(self, f"lin{i}")(x)
            if i < self.L:
                x = self.out_feat = F.elu(z)
            else:
                x = z
        return x


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=7)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--beta", type=float, default=0.1)
    ap.add_argument("--nce-T", type=float, default=0.075)
    ap.add_argument("--max-samples", type=int, default=16384)
    ap.add_argument("--proj-dim", type=int, default=256)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ppi_gcrd.py measures on a CUDA device; none found")
    dev = torch.device("cuda")
    graphs = synthetic.make_ppi_graphs("train", 0, args.scale)
    n_g = len(graphs)
    dgr = [(x.to(dev), y.to(dev), ei.to(dev)) for x, y, ei in graphs]
    teacher = engine_ppi.teacher(graphs, seed=1)
    feats = [teacher.predict(x, ei, return_feat=True)[1].clone() for x, _, ei in dgr]
    del teacher
    beta, nce_T, S, P = args.beta, args.nce_T, args.max_samples, args.proj_dim

    obj = PerGraphGCRD(feats, 136, proj_dim=P, max_samples=S, nce_T=nce_T, beta=beta)
    cap = engine_ppi.student(graphs, seed=0, gcrd=obj)
    launches = cap.launches_per_step(0)
    cap.capture()

    def torch_heads():
        sp = torch.nn.Sequential(torch.nn.Linear(136, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).to(dev)
        tp = torch.nn.Sequential(torch.nn.Linear(1024, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).to(dev)
        sp.load_state_dict({k: v.to(dev) for k, v in obj.student_proj_state_dict().items()})
        tp.load_state_dict({k: v.to(dev) for k, v in obj.teacher_proj_state_dict().items()})
        return sp, tp

    eager = engine_ppi.student(graphs, seed=0)
    e_sp, e_tp = torch_heads()
    e_opt = torch.optim.Adam(list(e_sp.parameters()) + list(e_tp.parameters()), lr=0.005)
    m = StudentModule(eager.layers, 50).to(dev)
    m.load_state_dict(eager.state_dict())
    m_sp, m_tp = torch_heads()
    opt = torch.optim.Adam([{"params": m.parameters()}, {"params": m_sp.parameters()}, {"params": m_tp.parameters()}],
                           lr=0.005)

    def eager_epoch(e):
        for i in eager.epoch_order(e):
            e_opt.zero_grad()
            eager.train_step(i, beta=beta, aux=lambda f: criterion_ppi.nce_criterion(
                eager.logits().detach(), eager.y[i], e_sp(f), e_tp(feats[i]), 1.0, nce_T, S)[2])
            e_opt.step()

    def module_epoch(e):
        for i in eager.epoch_order(e):
            x, y, ei = dgr[i]
            out = m(x, ei)
            loss = criterion_ppi.nce_criterion(out, y, m_sp(m.out_feat), m_tp(feats[i]), beta, nce_T, S)[0]
            opt.zero_grad()
            loss.backward()
            opt.step()

    arms = {"captured": lambda e: cap.train_epoch(e), "eager_aux": eager_epoch, "module": module_epoch}
    for fn in arms.values():                                  # warm-up epoch: every graph's shapes, plans, allocator
        fn(0)
    torch.cuda.synchronize()
    ts = {k: [] for k in arms}
    for e in range(1, args.epochs + 1):
        for k, fn in arms.items():
            ts[k].append(timed(lambda: fn(e)))
    res = dict(gpu=card(), scale=args.scale, n_graphs=n_g, beta=beta, nce_T=nce_T, max_samples=S, proj_dim=P,
               epochs=args.epochs, launches_per_step_captured=launches, n=[int(f.shape[0]) for f in feats])
    for k, v in ts.items():
        res[f"{k}_ms_per_epoch"] = round(statistics.median(v), 3)
        res[f"{k}_ms_per_epoch_range"] = [round(min(v), 3), round(max(v), 3)]
        res[f"{k}_ms_per_step"] = round(statistics.median(v) / n_g, 4)
    line = json.dumps(res)
    print(line)
    if args.json:
        Path(args.json).write_text(line + "\n")


if __name__ == "__main__":
    main()
