"""Times one GSP training step (kd + beta * GSP, arxiv_pyg/gnn_kd_and_aux.py:138-148) on the ARXIV-shape graph, three arms
alternated in one process for GCN and SAGE students [128, 256, 256, 40] at S = 4096, 8192 and 16384 and proj_dim 128 and
256, with the scripts' cosine kernel at beta 10 (run_kd_and_aux.sh; --kernel / --beta change it):

    captured   GCNStudentTrainer / SAGEStudentTrainer with gsp.GSP, the whole step one CUDA graph replay
    eager_aux  the same fused student with train_step(aux=...): torch projection heads + torch Adam, criterion.gpw_criterion
    module     the module path: torch model of efficient_gnns_b200.nn convs, torch heads, torch Adam, autograd

Prints one JSON line per (model, S, proj_dim) with medians and ranges in ms, launches per step of the captured arm, the bytes
the GSP object allocates (all of its step's buffers), and the card name and power limit read in the same run.
--profile DIR, in a separate pass after the timing, writes the per-kernel table of the captured step (torch.profiler)."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
sys.path.insert(0, str(Path(__file__).resolve().parent))
import efficient_gnns_b200  # noqa: E402,F401
from bench_configs import Student  # noqa: E402
from efficient_gnns_b200 import criterion as C, nn as bnn, sparse, synthetic  # noqa: E402
from efficient_gnns_b200.engine import GCNStudentTrainer  # noqa: E402
from efficient_gnns_b200.engine_sage import SAGEStudentTrainer  # noqa: E402
from efficient_gnns_b200.gsp import GSP  # noqa: E402

DIMS = [128, 256, 256, 40]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b)


def heads(dev, P):
    sp = torch.nn.Sequential(bnn.Linear(256, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).to(dev)
    tp = torch.nn.Sequential(bnn.Linear(752, P), torch.nn.BatchNorm1d(P), torch.nn.ReLU()).to(dev)
    return sp, tp


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--samples", type=int, nargs="+", default=[4096, 8192, 16384])
    ap.add_argument("--proj", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--kernel", default="cosine")
    ap.add_argument("--beta", type=float, default=10.0)
    ap.add_argument("--models", nargs="+", default=["gcn", "sage"])
    ap.add_argument("--profile", type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_gsp.py measures on a CUDA device; none found")
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
    tf = F.pad(t_feat, (0, 2))                      # 750 -> 752: 16-byte row pitch for the tensor-core GEMM
    for model in args.models:
        Eng, conv = ((GCNStudentTrainer, lambda i, o: bnn.GCNConv(i, o, cached=True)) if model == "gcn"
                     else (SAGEStudentTrainer, bnn.SAGEConv))
        for S in args.samples:
            for P in args.proj:
                K, B = args.kernel, args.beta
                torch.manual_seed(0)
                torch.cuda.synchronize()
                before = torch.cuda.memory_allocated()
                g = GSP(t_feat, idx, 256, proj_dim=P, max_samples=S, kernel=K, beta=B, seed=1)
                gsp_bytes = torch.cuda.memory_allocated() - before
                cap = Eng(adj, DIMS, dropout=0.5, lr=0.01, seed=0, gsp=g)
                cap.capture(x, y, idx, tl, warmup=2)
                launches = g.launches_per_step(x, y, idx, tl)

                ea = Eng(adj, DIMS, dropout=0.5, lr=0.01, seed=0)
                esp, etp = heads(dev, P)
                eopt = torch.optim.Adam(list(esp.parameters()) + list(etp.parameters()), lr=0.01)

                def eager_step():
                    def aux(f):
                        return C.gpw_criterion(ea.Y[-1][idx], y[idx], esp(f[idx]), etp(tf[idx]), K, 1.0, S)[2]
                    eopt.zero_grad()
                    ea.train_step(x, y, idx, tl, aux=aux, beta=B)
                    eopt.step()

                mod = Student(conv, DIMS).to(dev)
                msp, mtp = heads(dev, P)
                mopt = torch.optim.Adam(list(mod.parameters()) + list(msp.parameters()) + list(mtp.parameters()), lr=0.01)

                def module_step():
                    out = mod(x, adj)[idx]
                    _, _, la = C.gpw_criterion(out, y[idx], msp(mod.out_feat[idx]), mtp(tf[idx]), K, 1.0, S)
                    lk, _, _ = C.kd_criterion(out, y[idx], tl[idx], 0.9, 4.0)
                    loss = lk + B * la
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
                res = dict(model=model, S=S, proj_dim=P, kernel=K, beta=B, gpu=gpu, launches_per_step_captured=launches,
                           gsp_object_MB=round(gsp_bytes / 2 ** 20, 1))
                for k, v in ts.items():
                    v = sorted(v)
                    res[f"{k}_ms_median"] = round(v[len(v) // 2], 3)
                    res[f"{k}_ms_range"] = [round(v[0], 3), round(v[-1], 3)]
                print(json.dumps(res), flush=True)
                if args.profile and model == "gcn":
                    from torch.profiler import ProfilerActivity, profile
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        for _ in range(3):
                            cap.replay()
                        torch.cuda.synchronize()
                    out = Path(args.profile)
                    out.mkdir(parents=True, exist_ok=True)
                    (out / f"gsp_{model}_S{S}_P{P}.txt").write_text(prof.key_averages().table(sort_by="cuda_time_total",
                                                                                             row_limit=40))
                del cap, g, ea, mod
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
