"""Time the fused R-GCN training step (efficient_gnns_b200.rgcn.RGCNTrainer) on GraphSAINT batches of the MAG-shaped synthetic
(scale 1), built the way the reference's main() builds its graph (mag_pyg/gnn.py:308-366): reverse relations, undirected
cites, group_hetero_graph, batch_size 20000 roots, walk_length = num_layers.

Arms (same batches): the student KD step (2 x 32, teacher logits from the engine's eval forward of a 3 x 512 teacher), the
teacher's supervised step (3 x 512), and the module path (RelConv/RelNet of tests/test_rgcn_gpu.py on the mirrored PyG
surface + torch Adam) for both.  Prints one JSON line: ms/step, b200gnn launches/step, the weight-gradient and embedding-Adam
shares of the engine step (CUDA events around those calls in a separate, synchronised pass), and the first-step loss of the
engine vs the module path from the same weights (no dropout, so the two compute the same function).

    python tools/bench_rgcn.py [--steps 10] [--warmup 3] [--scale 1.0]
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
sys.path.insert(0, str(ROOT / "tests"))


def mag_graph(scale: float):
    import torch
    import efficient_gnns_b200
    from efficient_gnns_b200 import synthetic
    from efficient_gnns_b200.graphdata import Data
    from efficient_gnns_b200.nn import to_undirected
    sys.path.insert(0, str(Path(efficient_gnns_b200.__file__).resolve().parent / "shim"))
    from torch_geometric.utils.hetero import group_hetero_graph
    m = synthetic.make_mag_dataset(scale)
    eid = dict(m["edge_index_dict"])
    r, c = eid[("author", "affiliated_with", "institution")]
    eid[("institution", "to", "author")] = torch.stack([c, r])
    r, c = eid[("author", "writes", "paper")]
    eid[("paper", "to", "author")] = torch.stack([c, r])
    r, c = eid[("paper", "has_topic", "field_of_study")]
    eid[("field_of_study", "to", "paper")] = torch.stack([c, r])
    eid[("paper", "cites", "paper")] = to_undirected(eid[("paper", "cites", "paper")])
    edge_index, edge_type, node_type, local_node_idx, local2global, key2int = group_hetero_graph(eid, m["num_nodes_dict"])
    n = node_type.numel()
    data = Data(edge_index=edge_index, edge_attr=edge_type, node_type=node_type, local_node_idx=local_node_idx)
    data.num_nodes = n
    data.y = node_type.new_full((n, 1), -1)
    data.y[local2global["paper"]] = m["y_dict"]["paper"]
    data.train_mask = torch.zeros(n, dtype=torch.bool)
    data.train_mask[local2global["paper"][m["split_idx"]["train"]["paper"]]] = True
    x_dict = {key2int[k]: v for k, v in m["x_dict"].items()}
    num_nodes = {key2int[k]: v for k, v in m["num_nodes_dict"].items()}
    relations = {int(key2int[k]): (int(key2int[k[0]]), int(key2int[k[-1]])) for k in eid}
    return data, x_dict, num_nodes, relations, m["num_classes"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--batch-size", type=int, default=20000)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        raise SystemExit("bench_rgcn needs a CUDA device")
    import efficient_gnns_b200  # noqa: F401
    from efficient_gnns_b200 import lib, ops, sampling
    from efficient_gnns_b200.rgcn import RGCNTrainer
    from test_rgcn_gpu import RelConv
    torch.cuda.set_device(0)
    data, x_dict, num_nodes, relations, C = mag_graph(args.scale)
    x_dict = {k: v.cuda() for k, v in x_dict.items()}
    R = len(relations)
    n_batches = args.steps + args.warmup

    def sampled(layers):
        loader = sampling.GraphSAINTRandomWalkSampler(data, batch_size=args.batch_size, walk_length=layers, num_steps=n_batches,
                                                      seed=0)
        return list(loader)

    class Net(torch.nn.Module):                      # the module path: RelConv x L, relu between layers (mag_pyg/gnn.py:127-137)
        def __init__(self, H, L, p):
            super().__init__()
            from efficient_gnns_b200 import nn as bnn
            self.bnn, self.p = bnn, p
            dims = [128] + [H] * (L - 1) + [C]
            self.emb_dict = torch.nn.ParameterDict({str(t): torch.nn.Parameter(torch.empty(n, 128)) for t, n in num_nodes.items()
                                                    if t not in x_dict})
            self.convs = torch.nn.ModuleList([RelConv(dims[i], dims[i + 1], len(num_nodes), R) for i in range(L)])

        def forward(self, b):
            h = self.bnn.group_input(x_dict, self.emb_dict, b.node_type, b.local_node_idx, 128)
            for i, conv in enumerate(self.convs):
                h = conv(h, b.edge_index, b.edge_attr, b.node_type)
                if i != len(self.convs) - 1:
                    h = F.dropout(F.relu(h), p=self.p, training=True)
            return h

    def timed(fn, batches):
        for b in batches[:args.warmup]:
            fn(b)
        torch.cuda.synchronize()
        lib.reset_launch_count()
        t0 = time.perf_counter()
        for b in batches[args.warmup:]:
            fn(b)
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3 / args.steps, lib.launch_count() / args.steps

    def shares(tr, batches, teacher=None):
        """Fraction of a synchronised engine step spent in the weight-gradient GEMMs and in the embedding Adam."""
        acc = {"wgrad": 0.0, "emb_adam": 0.0}
        orig = {"wgrad": ops.gemm_wgrad_tf32x3, "emb_adam": ops.embedding_adam}

        def wrap(key):
            def f(*a, **k):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); r = orig[key](*a, **k); e1.record(); e1.synchronize()
                acc[key] += e0.elapsed_time(e1)
                return r
            return f
        import efficient_gnns_b200.rgcn as rg
        rg.ops.gemm_wgrad_tf32x3, rg.ops.embedding_adam = wrap("wgrad"), wrap("emb_adam")
        try:
            total = 0.0
            for b in batches[args.warmup:]:
                tl = teacher.forward(b, x_dict, training=False)[b.train_mask] if teacher else None
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(); tr.train_step(b, x_dict, teacher_logits=tl); e1.record(); e1.synchronize()
                total += e0.elapsed_time(e1)
        finally:
            rg.ops.gemm_wgrad_tf32x3, rg.ops.embedding_adam = orig["wgrad"], orig["emb_adam"]
        return {k: round(v / total, 4) for k, v in acc.items()}

    result = {"metric": "rgcn_train_step", "batch_size": args.batch_size, "scale": args.scale, "steps": args.steps}
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        result["gpu"] = smi.stdout.strip().splitlines()[0]
    except Exception:
        result["gpu"] = torch.cuda.get_device_name(0)

    # ---- teacher (3 x 512), supervised
    b3 = sampled(3)
    result["teacher_batch_nodes"] = int(sum(b.num_nodes for b in b3) / len(b3))
    teacher = RGCNTrainer(128, 512, C, 3, 0.5, num_nodes, list(x_dict), R, relations, seed=0)
    ms, la = timed(lambda b: teacher.train_step(b, x_dict), b3)
    result["teacher_engine_ms"], result["teacher_engine_launches"] = round(ms, 3), la
    result["teacher_engine_shares"] = shares(teacher, b3)
    net = Net(512, 3, 0.5).cuda()
    net.load_state_dict(teacher.state_dict())
    opt = torch.optim.Adam(net.parameters(), lr=0.01)

    def module_step(b, model=net, o=opt, tl=None):
        out = model(b)[b.train_mask]
        loss = F.cross_entropy(out, b.y[b.train_mask].view(-1))
        o.zero_grad(); loss.backward(); o.step()
    ms, la = timed(module_step, b3)
    result["teacher_module_ms"] = round(ms, 3)
    del net, opt
    torch.cuda.empty_cache()

    # ---- student (2 x 32), KD against the teacher's eval forward
    b2 = sampled(2)
    result["student_batch_nodes"] = int(sum(b.num_nodes for b in b2) / len(b2))
    student = RGCNTrainer(128, 32, C, 2, 0.5, num_nodes, list(x_dict), R, relations, seed=1)
    tls = [teacher.forward(b, x_dict, training=False)[b.train_mask].clone() for b in b2]
    it = iter(range(n_batches))
    ms, la = timed(lambda b: student.train_step(b, x_dict, teacher_logits=tls[next(it)]), b2)
    result["student_kd_engine_ms"], result["student_kd_engine_launches"] = round(ms, 3), la
    result["student_kd_engine_shares"] = shares(student, b2, teacher)
    net = Net(32, 2, 0.5).cuda()
    net.load_state_dict(student.state_dict())
    opt = torch.optim.Adam(net.parameters(), lr=0.01)
    it = iter(range(n_batches))

    def module_kd(b):
        out = net(b)[b.train_mask]
        tl = tls[next(it)]
        loss = (F.kl_div(F.log_softmax(out / 4.0, 1), F.softmax(tl / 4.0, 1)) * (0.9 * 16)
                + F.cross_entropy(out, b.y[b.train_mask].view(-1)) * 0.1)
        opt.zero_grad(); loss.backward(); opt.step()
    ms, la = timed(module_kd, b2)
    result["student_kd_module_ms"] = round(ms, 3)

    # ---- parity: fresh student, no dropout, same weights, one supervised step on the same batch
    eng = RGCNTrainer(128, 32, C, 2, 0.0, num_nodes, list(x_dict), R, relations, seed=5)
    ref = Net(32, 2, 0.0).cuda()
    ref.load_state_dict(eng.state_dict())
    b = b2[0]
    l_eng = float(eng.train_step(b, x_dict)[0])
    l_mod = float(F.cross_entropy(ref(b)[b.train_mask], b.y[b.train_mask].view(-1)))
    result["parity_loss_engine"], result["parity_loss_module"] = l_eng, l_mod
    result["parity_rel_diff"] = abs(l_eng - l_mod) / abs(l_mod)
    result["teacher_speedup"] = round(result["teacher_module_ms"] / result["teacher_engine_ms"], 3)
    result["student_kd_speedup"] = round(result["student_kd_module_ms"] / result["student_kd_engine_ms"], 3)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
