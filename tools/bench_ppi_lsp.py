"""Time an epoch of the PPI student with LSP (ppi_pyg/gnn.py --training lpw: BCE + beta * lpw on each graph's edge list) on
the 20 training graphs of synthetic.make_ppi_graphs(scale), three arms alternated epoch by epoch in one process:

    captured   engine_ppi.student with lsp.PerGraphLSP, one CUDA graph replay per training graph
    eager_aux  the same fused student with train_step(i, aux=lambda f: criterion_ppi.lpw_criterion(..., f, ...)[2], beta)
    module     the module path: StudentNet composed of nn.GATConv + torch.nn.Linear + F.elu under autograd,
               criterion_ppi.lpw_criterion and torch.optim.Adam, one graph per step as gnn.py's train() runs it

The teacher features are TeacherNet's out_feat [n, 1024] (engine_ppi.teacher(...).predict(..., return_feat=True)).

    python tools/bench_ppi_lsp.py [--epochs 7] [--scale 1.0] [--kernel cosine] [--beta 100] [--json out.json]

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
from efficient_gnns_b200.lsp import PerGraphLSP  # noqa: E402


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
    ap.add_argument("--kernel", default="cosine")
    ap.add_argument("--beta", type=float, default=100.0)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_ppi_lsp.py measures on a CUDA device; none found")
    dev = torch.device("cuda")
    graphs = synthetic.make_ppi_graphs("train", 0, args.scale)
    n_g = len(graphs)
    dgr = [(x.to(dev), y.to(dev), ei.to(dev)) for x, y, ei in graphs]
    teacher = engine_ppi.teacher(graphs, seed=1)
    feats = [teacher.predict(x, ei, return_feat=True)[1].clone() for x, _, ei in dgr]
    edges = [ei for _, _, ei in dgr]
    del teacher
    kernel, beta = args.kernel, args.beta

    cap = engine_ppi.student(graphs, seed=0, lsp=PerGraphLSP(feats, edges, 136, kernel=kernel, beta=beta))
    launches = cap.launches_per_step(0)
    cap.capture()
    eager = engine_ppi.student(graphs, seed=0)
    m = StudentModule(eager.layers, 50).to(dev)
    m.load_state_dict(eager.state_dict())
    opt = torch.optim.Adam(m.parameters(), lr=0.005)

    def eager_epoch(e):
        for i in eager.epoch_order(e):
            eager.train_step(i, beta=beta, aux=lambda f: criterion_ppi.lpw_criterion(
                eager.logits().detach(), eager.y[i], f, feats[i], edges[i], kernel, 1)[2])

    def module_epoch(e):
        for i in eager.epoch_order(e):
            x, y, ei = dgr[i]
            out = m(x, ei)
            loss = criterion_ppi.lpw_criterion(out, y, m.out_feat, feats[i], ei, kernel, beta)[0]
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
    res = dict(gpu=card(), scale=args.scale, n_graphs=n_g, kernel=kernel, beta=beta, epochs=args.epochs,
               launches_per_step_captured=launches, E=[int(ei.shape[1]) for ei in edges])
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
