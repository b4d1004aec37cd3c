"""Times one LSP training step (kd + beta * lpw, arxiv_pyg/gnn_kd_and_aux.py:149-155) on the ARXIV-shape graph, three arms
alternated in one process, for GCN and SAGE students [128, 256, 256, 40] with (cosine, beta 100), the scripts' setting, and
(rbf, beta 0.5), the reference's default kernel:

    captured   GCNStudentTrainer / SAGEStudentTrainer with lsp.LSP, the whole step one CUDA graph replay
    eager_aux  the same fused student with train_step(aux=lambda f: criterion.lpw_criterion(..., f[idx], t[idx], ...)[2])
    module     the module path: torch model of efficient_gnns_b200.nn convs, torch Adam, autograd, criterion.lpw_criterion

The edge list is the reference's train-induced subgraph (gnn_kd_and_aux.py:240-243).  Prints one JSON line per (model, kernel)
with medians and ranges in ms, launches per step of the captured arm, and the card name and power limit read in the same run.
--profile DIR writes the per-kernel table of the captured step (torch.profiler) and adds lsp_student_kernel's algorithmic
bytes over its time to the JSON line."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import efficient_gnns_b200  # noqa: E402,F401
from bench_configs import Student  # noqa: E402
from efficient_gnns_b200 import criterion as C, nn as bnn, sparse, synthetic  # noqa: E402
from efficient_gnns_b200.engine import GCNStudentTrainer  # noqa: E402
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer  # noqa: E402
from efficient_gnns_b200.lsp import LSP  # noqa: E402
from oracle import graph as og  # noqa: E402

DIMS = [128, 256, 256, 40]
SETTINGS = {"cosine": 100.0, "rbf": 0.5}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


def student_bytes(obj: LSP) -> int:
    """Compulsory HBM bytes of one lsp_student_kernel launch: every edge's source row and each non-empty segment's destination
    row (4H each), and per edge src, sim_t, sim_s, pos_dst / pos_src, the two val / selfc pairs and the c / ra scratch."""
    H, E = obj.H, obj.E
    segments = int((torch.diff(obj.plan.rowptr.long()) > 0).sum())
    return 4 * H * (E + segments) + E * (4 + 4 + 4 + 8 + 16 + 8) + 4 * (obj.plan.n_seg + 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--models", nargs="+", default=["gcn", "sage"])
    ap.add_argument("--kernels", nargs="+", default=list(SETTINGS))
    ap.add_argument("--profile", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_lsp.py measures on a CUDA device; none found")
    dev = "cuda"
    gpu = card()
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.to(dev)
    perm = (ei[1] * n + ei[0]).argsort()
    adj = sparse.SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    x, y = ds.x.to(dev), ds.y.squeeze(1).to(dev)
    idx = ds.split_idx["train"].to(dev)
    t_feat, tl = ds.teacher_feat.to(dev), ds.teacher_logits.to(dev)
    r, c, _ = adj.coo()
    sub = torch.from_numpy(og.subgraph(idx.cpu().numpy(), np.stack([r.cpu().numpy(), c.cpu().numpy()]), True)[0]).to(dev)
    for model in args.models:
        Eng, conv = ((GCNStudentTrainer, lambda i, o: bnn.GCNConv(i, o, cached=True)) if model == "gcn"
                     else (SAGEStudentTrainer, bnn.SAGEConv))
        for kernel in args.kernels:
            beta = SETTINGS[kernel]
            torch.manual_seed(0)
            obj = LSP(t_feat, idx, sub, DIMS[-2], kernel=kernel, beta=beta)
            cap = Eng(adj, DIMS, dropout=0.5, lr=0.01, seed=0, lsp=obj)
            cap.capture(x, y, idx, tl, warmup=2)
            before = efficient_gnns_b200.lib.launch_count()
            cap._step_impl(x, y, idx, tl)
            launches = efficient_gnns_b200.lib.launch_count() - before

            ea = Eng(adj, DIMS, dropout=0.5, lr=0.01, seed=0)

            def eager_step():
                ea.train_step(x, y, idx, tl, beta=beta,
                              aux=lambda f: C.lpw_criterion(ea.Y[-1][idx], y[idx], f[idx], t_feat[idx], sub, kernel, 1)[2])

            mod = Student(conv, DIMS).to(dev)
            mopt = torch.optim.Adam(mod.parameters(), lr=0.01)

            def module_step():
                out = mod(x, adj)[idx]
                _, _, la = C.lpw_criterion(out, y[idx], mod.out_feat[idx], t_feat[idx], sub, kernel, 1)
                lk, _, _ = C.kd_criterion(out, y[idx], tl[idx], 0.9, 4.0)
                loss = lk + beta * la
                mopt.zero_grad(); loss.backward(); mopt.step()

            arms = {"captured": cap.replay, "eager_aux": eager_step, "module": module_step}
            for fn in arms.values():
                for _ in range(args.warmup):
                    fn()
            torch.cuda.synchronize()
            ts = {k: [] for k in arms}
            for _ in range(args.iters):
                for k, fn in arms.items():
                    ts[k].append(timed(fn))
            res = dict(model=model, kernel=kernel, beta=beta, E=obj.E, gpu=gpu, launches_per_step_captured=launches)
            for k, v in ts.items():
                v = sorted(v)
                res[f"{k}_ms_median"] = round(v[len(v) // 2], 3)
                res[f"{k}_ms_range"] = [round(v[0], 3), round(v[-1], 3)]
            if args.profile:
                from torch.profiler import ProfilerActivity, profile
                reps = 5
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(reps):
                        cap.replay()
                    torch.cuda.synchronize()
                out = Path(args.profile)
                out.mkdir(parents=True, exist_ok=True)
                avg = prof.key_averages()
                (out / f"lsp_{model}_{kernel}.txt").write_text(avg.table(sort_by="cuda_time_total", row_limit=40))
                us = sum(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) for e in avg
                         if "lsp_student_kernel" in e.key) / reps
                if us > 0:
                    res["lsp_student_us"] = round(us, 1)
                    res["lsp_student_algorithmic_GBps"] = round(student_bytes(obj) / (us * 1e-6) / 1e9, 1)
            print(json.dumps(res), flush=True)
            del cap, obj, ea, mod
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
