"""Time G-CRD in the SIGN student step (gcrd.SIGNGCRD, SIGNStudentTrainer(..., gcrd=)) over whole epochs at the ARXIV shape
with the SIGN script's settings (scripts/run_all_kd_and_aux.sh: R 5, hidden 512, ff_layer 2, batch 50,000, proj_dim 256,
max_samples 16384, nce_T 0.075, beta 0.1), epochs of three arms alternated on the same GPU:

    gcrd     the captured G-CRD step: one CUDA graph per batch size, heads on the un-stored dropout(prelu(cat))
    kd       the captured KD-only step (what the G-CRD step adds to)
    aux      the eager aux= step: out_feat materialised, torch heads (Linear, BatchNorm1d, ReLU), criterion.nce_criterion
             with its own row draw, autograd, and the heads in a torch Adam of their own

    python tools/bench_sign_gcrd.py [--epochs 5] [--out result.json]

Input: the ARXIV-shape synthetic graph and features (90,941 training nodes: batches of 50,000 and 40,941), hop features
from nn.neighbor_average_features(5), and 750-wide synthetic teacher features (the GAT teacher's width).  Prints one JSON
line with the GPU's name, power limit and maximum SM clock beside the per-arm epoch and step times.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import criterion, nn as enn, sparse  # noqa: E402
from efficient_gnns_b200.engine_sign import SIGNStudentTrainer  # noqa: E402
from efficient_gnns_b200.gcrd import SIGNGCRD  # noqa: E402
from efficient_gnns_b200.synthetic import ARXIV, make_node_dataset  # noqa: E402
from oracle import graph as og  # noqa: E402

R, HIDDEN, FF, BATCH, PROJ, MAX_SAMPLES, NCE_T, BETA, F_T = 5, 512, 2, 50000, 256, 16384, 0.075, 0.1, 750


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result line to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sign_gcrd measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    result = {"metric": "sign_gcrd_train_epoch", "hops": R + 1, "hidden": HIDDEN, "ff_layer": FF, "batch_size": BATCH,
              "proj_dim": PROJ, "max_samples": MAX_SAMPLES, "epochs": args.epochs}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else torch.cuda.get_device_name(0)

    ds = make_node_dataset(ARXIV, seed=0)
    n = ds.num_nodes
    row, col, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    adj_t = sparse.SparseTensor(row=torch.from_numpy(row).to(dev), col=torch.from_numpy(col).to(dev), sparse_sizes=(n, n),
                                is_sorted=True)
    feats = [f.contiguous() for f in enn.neighbor_average_features(adj_t, ds.x.to(dev), R)]
    y = ds.y.view(-1).to(dev)
    teacher = ds.teacher_logits.to(dev)
    t_feat = torch.randn(n, F_T, device=dev, generator=torch.Generator(device=dev).manual_seed(1)).relu_()
    train_idx = ds.split_idx["train"].to(dev)
    n_train = train_idx.numel()
    sizes = [min(BATCH, n_train - s) for s in range(0, n_train, BATCH)]
    result["batches"] = sizes
    width = (R + 1) * HIDDEN

    mk = lambda gcrd=None: SIGNStudentTrainer(feats, ds.num_classes, hidden=HIDDEN, ff_layer=FF, batch_size=BATCH,  # noqa: E731
                                              gcrd=gcrd)
    heads = SIGNGCRD(t_feat, width, proj_dim=PROJ, max_samples=MAX_SAMPLES, nce_T=NCE_T, beta=BETA)
    tr_gcrd = mk(heads).capture(sizes, y, teacher)
    tr_kd = mk().capture(sizes, y, teacher)
    tr_aux = mk()
    sp = torch.nn.Sequential(torch.nn.Linear(width, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU()).to(dev)
    tp = torch.nn.Sequential(torch.nn.Linear(F_T, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU()).to(dev)
    sp.load_state_dict(heads.student_proj_state_dict())
    tp.load_state_dict(heads.teacher_proj_state_dict())
    opt = torch.optim.Adam(list(sp.parameters()) + list(tp.parameters()), lr=tr_aux.lr)

    def aux_epoch(e):
        order = tr_aux.epoch_order(train_idx, e)
        for s in range(0, n_train, BATCH):
            b = order[s:s + BATCH]
            yb, tb = y[b], t_feat[b]
            aux = lambda f: criterion.nce_criterion(tr_aux.logits().detach(), yb, sp(f), tp(tb), BETA, NCE_T,  # noqa: E731
                                                    MAX_SAMPLES)[2]
            opt.zero_grad()
            tr_aux.train_step(b, y, teacher, aux=aux, beta=BETA)
            opt.step()

    arms = {"gcrd": lambda e: tr_gcrd.train_epoch(train_idx, y, teacher, epoch=e),
            "kd": lambda e: tr_kd.train_epoch(train_idx, y, teacher, epoch=e),
            "aux": aux_epoch}

    def timed(fn, e):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(e)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    for fn in arms.values():                                       # warm-up of every shape
        timed(fn, 0)
    times = {k: [] for k in arms}
    for e in range(1, args.epochs + 1):
        for k, fn in arms.items():
            times[k].append(timed(fn, e))
    steps = len(sizes)
    for k, t in times.items():
        med = statistics.median(t)
        result[f"{k}_epoch_ms"] = [round(v, 2) for v in t]
        result[f"{k}_step_ms"] = round(med / steps, 2)
    result["gcrd_over_kd_ms_per_step"] = round(result["gcrd_step_ms"] - result["kd_step_ms"], 2)
    result["aux_over_gcrd"] = round(statistics.median(times["aux"]) / statistics.median(times["gcrd"]), 3)
    result["gcrd_last_loss"] = [round(v, 5) for v in tr_gcrd.loss_out.tolist()]
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
