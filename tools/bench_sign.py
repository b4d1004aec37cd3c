"""Time the fused SIGN student training step (engine_sign.SIGNStudentTrainer, KD, CUDA-graph replay) over whole epochs
against the same model as a plain torch module in fp32 (oracle/sign.py's forward, autograd, torch.optim.Adam;
allow_tf32=False) on the same GPU, epochs of the two alternated.

    python tools/bench_sign.py [--epochs 5] [--ff 2] [--hidden 512] [--R 5] [--batch-size 50000] [--out result.json]

Input: the ARXIV-shape synthetic graph and features, hop features from nn.neighbor_average_features(R).  Per step it
reports milliseconds, the useful FLOP of the dense contractions (forward, input and weight gradients, computed from the
shapes by SIGNStudentTrainer.useful_flop) and the tensor rate 3 x useful FLOP/s (3xTF32 issues three TF32 products per
fp32 product) as a share of the 495 TF/s dense TF32 data-sheet figure of the H100 SXM.
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
from efficient_gnns_b200 import nn as enn, sparse  # noqa: E402
from efficient_gnns_b200.engine_sign import SIGNStudentTrainer  # noqa: E402
from efficient_gnns_b200.synthetic import ARXIV, make_node_dataset  # noqa: E402
from oracle import criterion as oc, graph as og, sign as osign  # noqa: E402

TF32_PEAK = 495e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=5)
    ap.add_argument("--ff", type=int, default=2)
    ap.add_argument("--hidden", type=int, default=512)
    ap.add_argument("--R", type=int, default=5)
    ap.add_argument("--batch-size", type=int, default=50000)
    ap.add_argument("--out", default=None, help="also write the JSON result line to this file")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sign measures on a GPU"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    dev = torch.device("cuda")
    result = {"metric": "sign_kd_train_step", "ff_layer": args.ff, "hidden": args.hidden, "hops": args.R + 1,
              "batch_size": args.batch_size, "epochs": args.epochs}
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    result["gpu"] = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else torch.cuda.get_device_name(0)

    ds = make_node_dataset(ARXIV, seed=0)
    n = ds.num_nodes
    row, col, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)          # row = destination, col = source
    adj_t = sparse.SparseTensor(row=torch.from_numpy(row).to(dev), col=torch.from_numpy(col).to(dev), sparse_sizes=(n, n),
                                is_sorted=True)
    feats = [f.contiguous() for f in enn.neighbor_average_features(adj_t, ds.x.to(dev), args.R)]
    y = ds.y.view(-1).to(dev)
    teacher = ds.teacher_logits.to(dev)
    train_idx = ds.split_idx["train"].to(dev)
    n_train = train_idx.numel()
    sizes = [min(args.batch_size, n_train - s) for s in range(0, n_train, args.batch_size)]
    result["batches"] = sizes

    tr = SIGNStudentTrainer(feats, ds.num_classes, hidden=args.hidden, ff_layer=args.ff, batch_size=args.batch_size)
    tr.capture(sizes, y, teacher)
    flop = sum(tr.useful_flop(b) for b in sizes)

    # the torch arm: the same model as an fp32 torch module (the oracle's functional forward on leaf parameters)
    sd = {k: v.detach().clone().requires_grad_(True) for k, v in tr.state_dict().items()}
    opt = torch.optim.Adam(list(sd.values()), lr=tr.lr)
    H, hid, p, p_in = tr.H, tr.hidden, tr.p, tr.p_in

    def torch_epoch(epoch):
        order = tr.epoch_order(train_idx, epoch)
        for s in range(0, n_train, args.batch_size):
            b = order[s:s + args.batch_size]
            B = b.numel()
            keep = lambda *shape, q=p: torch.rand(*shape, device=dev) >= q  # noqa: E731
            masks = dict(input=[keep(B, tr.F, q=p_in) for _ in range(H)], hidden=[[keep(B, hid) for _ in range(tr.ff - 1)]
                                                                                for _ in range(H)],
                         cat=keep(B, H * hid), project=[keep(B, hid) for _ in range(tr.ff - 1)])
            logits, _ = osign.sign_forward([f[b] for f in feats], sd, tr.ff, masks, p, p_in)
            loss = oc.kd_criterion(logits, y[b], teacher[b], tr.alpha, tr.kd_T)[0]
            opt.zero_grad()
            loss.backward()
            opt.step()

    def timed(fn, e):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(e)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    eng = lambda e: tr.train_epoch(train_idx, y, teacher, epoch=e)  # noqa: E731
    timed(eng, 0); timed(torch_epoch, 0)                           # warm-up of every shape
    t_eng, t_torch = [], []
    for e in range(1, args.epochs + 1):
        t_eng.append(timed(eng, e))
        t_torch.append(timed(torch_epoch, e))
    steps = len(sizes)
    me, mt = statistics.median(t_eng), statistics.median(t_torch)
    result.update(
        engine_epoch_ms=[round(v, 3) for v in t_eng], torch_epoch_ms=[round(v, 3) for v in t_torch],
        engine_step_ms=round(me / steps, 3), torch_step_ms=round(mt / steps, 3), speedup=round(mt / me, 3),
        useful_gflop_per_step=round(flop / steps / 1e9, 1),
        engine_useful_tflops=round(flop / (me * 1e-3) / 1e12, 1),
        engine_tensor_rate_share_of_tf32_peak=round(3 * flop / (me * 1e-3) / TF32_PEAK, 3),
        torch_useful_tflops=round(flop / (mt * 1e-3) / 1e12, 1))
    loss = tr.loss_out.tolist()
    result["engine_last_loss"] = [round(v, 5) for v in loss]
    line = json.dumps(result)
    print(line)
    if args.out:
        Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        Path(args.out).write_text(line + "\n")


if __name__ == "__main__":
    main()
