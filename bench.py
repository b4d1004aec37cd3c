#!/usr/bin/env python
"""Benchmark of the hot path: one full training step (fwd + loss + bwd + Adam) of the 3-layer GCN student with
logit-KD on the ARXIV-shape synthetic graph (BASELINE.json configs[1]).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--impl ours|reference] [--dump-outputs DIR]

Prints ONE JSON line (see README/DESIGN.md for the keys).  metric = edges aggregated per second,
edges/s = 2 * L * nnz(Â) / t_step  (L=3 aggregations forward + 3 backward, nnz of the matrix the SpMM walks).
"""
from __future__ import annotations

import argparse
import json
import os

import subprocess
import sys

# stdout carries exactly ONE JSON line: park the real stdout and point fd 1 at stderr before torch / NCCL load, so that
# library chatter (NCCL's version banner, warnings from C++ code) cannot land in front of it.
if not hasattr(sys, "_b200gnn_json_fd"):          # once per process (dist_bench re-imports this file as a module)
    sys.stdout.flush()
    sys._b200gnn_json_fd = os.dup(1)
    os.dup2(2, 1)
_JSON_FD = sys._b200gnn_json_fd


def emit_json_line(line: dict):
    os.write(_JSON_FD, (json.dumps(line) + "\n").encode())

import threading
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent
sys.path.insert(0, str(ROOT))

METRIC = "edges aggregated/s (fwd+bwd), 3-layer GCN student + logit-KD, ARXIV-shape"
UNIT = "edges/s"
DIMS = [128, 256, 256, 40]


def workload_config(ds, nnz_hat, extra=None):
    cfg = {"workload": "configs[1]: 3-layer GCN 128-256-256-40 + logit-KD, synthetic ARXIV-shape "
                       f"(N={ds.num_nodes}, E_in={ds.edge_index.shape[1]}, nnz(A_hat)={nnz_hat}), fp32, full batch",
           "edges_per_step": 6 * nnz_hat, "nnz_walked": nnz_hat,
           "l2_policy": "per-step working set (~7 GB of activations) is far larger than the 50 MB L2; no flush needed"}
    if extra:
        cfg.update(extra)
    return cfg


def peaks():
    p = ROOT / "MEASURED_PEAKS.json"
    if p.exists():
        d = json.loads(p.read_text())
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s)"


class ClockSampler:
    """SM clock / throttle reasons sampled DURING the timed region: NVML polled every ~2 ms from a thread (the timed region of
    the default run is ~0.1 s, too short for `nvidia-smi -lms`), `nvidia-smi` as the fallback when NVML is unavailable."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index=0):
        self.rows, self.proc, self.index = [], None, index
        self.sm, self.max_mhz, self.reasons, self._stop, self._nvml = [], None, set(), False, None

    def _nvml_loop(self):
        nv, h = self._nvml
        names = {"hw_slowdown": getattr(nv, "nvmlClocksEventReasonHwSlowdown", 0x8),
                 "hw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonHwThermalSlowdown", 0x40),
                 "sw_thermal_slowdown": getattr(nv, "nvmlClocksEventReasonSwThermalSlowdown", 0x20),
                 "sw_power_cap": getattr(nv, "nvmlClocksEventReasonSwPowerCap", 0x4)}
        get_reasons = getattr(nv, "nvmlDeviceGetCurrentClocksEventReasons", None) or nv.nvmlDeviceGetCurrentClocksThrottleReasons
        while not self._stop:
            try:
                self.sm.append(int(nv.nvmlDeviceGetClockInfo(h, nv.NVML_CLOCK_SM)))
                r = int(get_reasons(h))
                self.reasons.update(n for n, bit in names.items() if r & bit)
            except Exception:  # noqa: BLE001
                pass
            time.sleep(0.002)

    def __enter__(self):
        try:
            import pynvml as nv
            nv.nvmlInit()
            vis = os.environ.get("CUDA_VISIBLE_DEVICES")
            phys = self.index
            if vis:
                ids = [v for v in vis.split(",") if v.strip() != ""]
                if self.index < len(ids) and ids[self.index].strip().isdigit():
                    phys = int(ids[self.index])
            h = nv.nvmlDeviceGetHandleByIndex(phys)
            self.max_mhz = int(nv.nvmlDeviceGetMaxClockInfo(h, nv.NVML_CLOCK_SM))
            self._nvml = (nv, h)
            self.t = threading.Thread(target=self._nvml_loop, daemon=True)
            self.t.start()
            return self
        except Exception:  # noqa: BLE001
            self._nvml = None
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), f"--query-gpu={self.Q}",
                                          "--format=csv,noheader,nounits", "-lms", "20"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except OSError:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def __exit__(self, *a):
        self._stop = True
        if self._nvml is not None:
            self.t.join(timeout=1)
        if self.proc:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except subprocess.TimeoutExpired:
                self.proc.kill()

    def summary(self):
        if self._nvml is not None:
            sm = sorted(self.sm)
            return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": self.max_mhz, "reasons": sorted(self.reasons),
                    "samples": len(sm), "source": "nvml"}
        sm = sorted(int(r[0]) for r in self.rows if r and r[0].isdigit())
        mx = max((int(r[1]) for r in self.rows if len(r) > 1 and r[1].isdigit()), default=None)
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = sorted({n for r in self.rows if len(r) >= 6 for n, v in zip(names, r[2:6]) if v.lower().startswith("active")})
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": reasons, "samples": len(sm),
                "source": "nvidia-smi"}


# ----------------------------------------------------------------------------------------------- reference / CPU arm
class CpuStep:
    """The reference's own CPU implementation of the path, restated (oracle/): GCN.forward + kd_criterion + backward
    through torch autograd + Adam on the host cores.  form='csr' -> torch.sparse_csr @ (what SparseTensor.matmul's
    spmm_cpu corresponds to, the path arxiv_pyg/gnn.py takes); form='scatter' -> index_select + scatter_add_
    (what torch_scatter.scatter_sum executes)."""

    def __init__(self, ds):
        from oracle import graph as og
        self.ds, n = ds, ds.num_nodes
        row, col, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
        r, c = og.to_symmetric(row, col, n)
        r, c, v = og.gcn_norm(r, c, n)
        self.ptr, self.c, self.v = torch.from_numpy(og.ind2ptr(r, n)), torch.from_numpy(c), torch.from_numpy(v)
        g = torch.Generator().manual_seed(0)
        self.W = [((torch.rand(DIMS[i], DIMS[i + 1], generator=g) * 2 - 1) * (6.0 / (DIMS[i] + DIMS[i + 1])) ** 0.5)
                  .requires_grad_(True) for i in range(3)]
        self.B = [torch.zeros(DIMS[i + 1], requires_grad=True) for i in range(3)]
        self.ga = [torch.ones(DIMS[i + 1], requires_grad=True) for i in range(2)]
        self.be = [torch.zeros(DIMS[i + 1], requires_grad=True) for i in range(2)]
        self.opt = torch.optim.Adam(self.W + self.B + self.ga + self.be, lr=0.01)
        self.nnz = int(self.c.numel())

    def step(self, form: str) -> float:
        from oracle import criterion as oc, nn as onn
        ds, n = self.ds, self.ds.num_nodes
        idx, y = ds.split_idx["train"], ds.y.squeeze(1)
        t0 = time.perf_counter()
        masks = [torch.rand(n, DIMS[i + 1]) >= 0.5 for i in range(2)]
        logits, _ = onn.gcn_forward(ds.x, self.ptr, self.c, self.v, self.W, self.B, self.ga, self.be, masks, 0.5, form=form)
        loss, _, _ = oc.kd_criterion(logits[idx], y[idx], ds.teacher_logits[idx], 0.9, 4.0)
        self.opt.zero_grad(); loss.backward(); self.opt.step()
        loss.item()
        return time.perf_counter() - t0

    def pick_threads(self, form: str = "csr"):
        """torch's CPU sparse kernels do not scale to every core of a large host (128 threads ran the step 4x slower than
        8 on the round-1 boxes): time one step per candidate count and keep the fastest, so the CPU arm is the host at
        its best rather than at its widest."""
        ncpu = os.cpu_count() or 1
        cands = sorted({c for c in (8, 16, 32, 64, ncpu) if c <= ncpu} | {min(ncpu, 8)})
        tried = {}
        torch.set_num_threads(cands[0])
        self.step(form)                                   # first-touch / allocator warm-up, not timed
        for c in cands:
            torch.set_num_threads(c)
            tried[c] = self.step(form)
            if tried[c] > 2.0 * min(tried.values()):      # clearly past the knee: stop widening
                break
        best = min(tried, key=tried.get)
        torch.set_num_threads(best)
        return best, {str(k): round(v, 3) for k, v in tried.items()}


def cpu_reference_step_time(ds, steps: int, warmup: int, form: str, cpu: "CpuStep" = None):
    """Mean seconds per step of the CPU arm at the current torch thread count."""
    cpu = cpu or CpuStep(ds)
    times = [cpu.step(form) for _ in range(warmup + steps)][warmup:]
    return sum(times) / len(times), cpu.nnz


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    from efficient_gnns_b200 import synthetic
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    cpu = CpuStep(ds)
    cores, tried = cpu.pick_threads("csr")
    # each step is one FULL training step of the workload on the host (seconds each): --steps / --warmup set the count
    warmup = args.warmup
    for _ in range(warmup):
        cpu.step("csr")
    times = [cpu.step("csr") for _ in range(args.steps)]
    steps, t_csr, nnz = len(times), sum(times) / len(times), cpu.nnz
    t_sc, _ = cpu_reference_step_time(ds, 1, 0, "scatter", cpu)
    val = 6 * nnz / t_csr
    sample = (f"{steps} full training steps (fwd+KD loss+bwd+Adam) of the same workload on the host, CSR SpMM form, "
              f"{cores} of {os.cpu_count()} host threads (fastest of s/step {tried}); --warmup {warmup}; "
              f"scatter_add form timed once: {6 * nnz / t_sc:.3e} edges/s")
    line = {"impl": "reference", "metric": METRIC, "value": val, "unit": UNIT, "n_gpus": args.gpus, "steps": steps,
            "warmup": warmup, "ms_per_step": t_csr * 1e3, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": workload_config(ds, nnz),
            "cpu_baseline": {"value": val, "unit": UNIT, "cores": cores, "kind": "port", "sample": sample,
                             "scatter_add_value": 6 * nnz / t_sc},
            "e2e": {"value": val, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    emit_json_line(line)


def parity_check(tr, ds, d):
    """One eager training step of the benchmarked engine compared with oracle/check.py (fp64) on identical inputs,
    parameters and dropout masks: the numbers tests/test_fullscale_gpu.py asserts on."""
    from efficient_gnns_b200 import ops
    from oracle import check, graph as og
    n = ds.num_nodes
    row, col, _ = og.to_sparse_adj_t(ds.edge_index.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    rn, cn, vn = og.gcn_norm(r, c, n)
    ptr, cc, vv = torch.from_numpy(og.ind2ptr(rn, n)), torch.from_numpy(cn), torch.from_numpy(vn).double()
    torch.cuda.synchronize()
    state = {k: v.cpu() for k, v in tr.state_dict().items()}
    step = int(tr.step_count.item())
    masks = [ops.dropout_mask(n, tr.dims[l + 1], tr.p, tr.seed, tr.dropout_offset(l, step)).cpu().bool()
             for l in range(tr.L - 1)]
    tr.train_step(d["x"], d["y"], d["idx"], d["t"])
    torch.cuda.synchronize()
    res = check.compare_engine_step(tr, ds.x, ds.y.squeeze(1), ds.teacher_logits, ds.split_idx["train"], ptr, cc, vv, masks, state)
    free, pat = res["free"], res["pattern"]
    return {"against": "oracle/check.py fp64 restatement of arxiv_pyg/gnn.py:45-53,102-195 + criterion.py:8-21, full size",
            "training_step_index": step,
            "logits_max_rel": free["logits_max"], "out_feat_max_rel": free["hidden_max"], "loss_rel": max(free["loss_rel"]),
            "relu_pattern_flips": free["flips"], "elements": free["elements"],
            "flip_worst_preactivation_rel": max(free["flip_worst_pre_rel"]),
            "grad_max_rel_same_pattern": max(pat["grad_max"]), "grad_fro_rel_same_pattern": max(pat["grad_fro"]),
            "grad_fro_rel_free": max(free["grad_fro"]), "grad_max_rel_free": max(free["grad_max"]),
            "pass": bool(free["logits_max"] <= 1e-5 and max(free["loss_rel"]) <= 1e-5 and max(pat["grad_max"]) <= 1e-5
                         and max(free["flip_worst_pre_rel"]) <= 1e-5)}


DUMP_LIMIT_BYTES = 64 << 20


def dump_outputs(out_dir, tr):
    """What the timed step hands back to its caller, after the last timed step: the three losses, the logits, the
    gradients and the updated parameters, as <name>.npy in float32 (about 28 MB at ARXIV shape).  Inputs, parameters and
    dropout masks are seeded, so two builds run with the same arguments can be compared output for output."""
    import numpy as np
    d = Path(out_dir)
    d.mkdir(parents=True, exist_ok=True)
    arrays = {"loss": tr.loss_out, "logits": tr.Y[-1], "grads": tr.grads}
    arrays.update({"param." + k: v for k, v in tr.state_dict().items()})
    arrays = {k: v.detach().float().cpu().numpy() for k, v in arrays.items()}
    total = sum(a.nbytes for a in arrays.values())
    if total > DUMP_LIMIT_BYTES:
        raise RuntimeError(f"--dump-outputs: {total} bytes exceed the {DUMP_LIMIT_BYTES}-byte limit")
    for name, a in arrays.items():
        np.save(d / f"{name}.npy", a)


# ----------------------------------------------------------------------------------------------- our arm (1 GPU)
def run_single(args):
    import efficient_gnns_b200  # noqa: F401
    from efficient_gnns_b200 import lib, ops, sparse, synthetic
    from efficient_gnns_b200.engine import GCNStudentTrainer

    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", "0")))
    torch.cuda.set_device(dev)
    lib.load()
    ds = synthetic.make_node_dataset(synthetic.ARXIV, seed=0)
    n = ds.num_nodes
    ei = ds.edge_index.to(dev)
    perm = (ei[1] * n + ei[0]).argsort()
    adj = sparse.SparseTensor(row=ei[1][perm], col=ei[0][perm], sparse_sizes=(n, n), is_sorted=True).to_symmetric()
    tr = GCNStudentTrainer(adj, DIMS, dropout=0.5, lr=0.01, seed=0)
    nnz = tr.nnz

    # pinned host copies of the step's inputs (e2e) and their resident device twins (kernel-only timing)
    host = {"x": ds.x.pin_memory(), "y": ds.y.squeeze(1).contiguous().pin_memory(),
            "t": ds.teacher_logits.pin_memory(), "idx": ds.split_idx["train"].pin_memory()}
    d = {k: torch.empty_like(v, device=dev) for k, v in host.items()}
    for k in d:
        d[k].copy_(host[k], non_blocking=True)
    torch.cuda.synchronize()
    tr.capture(d["x"], d["y"], d["idx"], d["t"], warmup=2)
    launches = tr.launches_per_step()          # counted on one eager step
    torch.cuda.synchronize()

    # ---- phase 1: device-resident throughput (CUDA-graph replays), clocks sampled during the region
    for _ in range(args.warmup):
        tr.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ClockSampler(dev.index or 0) as clk:
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            tr.replay()
        e1.record()
        torch.cuda.synchronize()
    ms_step = e0.elapsed_time(e1) / args.steps
    clocks = clk.summary()
    losses = tr.loss_out.tolist()
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, tr)

    # ---- phase 2: end to end — every step copies ITS inputs from pinned host memory and its losses are read back.
    # Two device input sets + two captured graphs: the upload of step k+1 (copy stream) overlaps the compute of step k.
    h2d = sum(v.numel() * v.element_size() for v in host.values())
    d2 = {k: torch.empty_like(v) for k, v in d.items()}
    for k in d2:
        d2[k].copy_(d[k])
    tr.capture(d2["x"], d2["y"], d2["idx"], d2["t"], warmup=1, key=1)
    sets = [d, d2]
    loss_host = torch.empty(3).pin_memory()
    copy_stream = torch.cuda.Stream()
    main = torch.cuda.current_stream()
    uploaded = [torch.cuda.Event(), torch.cuda.Event()]
    consumed = [torch.cuda.Event(), torch.cuda.Event()]

    def upload(i):
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[i])          # the step that last read this set has finished
            for k in sets[i]:
                sets[i][k].copy_(host[k], non_blocking=True)
            uploaded[i].record(copy_stream)

    def e2e_loop(n_steps):
        for i in (0, 1):
            consumed[i].record(main)
        upload(0)
        for step in range(n_steps):
            i = step & 1
            if step + 1 < n_steps:
                upload(1 - i)
            main.wait_event(uploaded[i])
            tr.replay(i)
            consumed[i].record(main)
            loss_host.copy_(tr.loss_out, non_blocking=True)

    e2e_loop(max(3, args.warmup // 2))
    torch.cuda.synchronize()
    e0.record()
    e2e_loop(args.steps)
    e1.record()
    torch.cuda.synchronize()
    ms_e2e = e0.elapsed_time(e1) / args.steps

    # ---- phase 3: roofline of the dominant kernel (K=256 aggregation), each launch bracketed by CUDA events
    #      on the launching stream, inside eager training steps
    evs = []
    orig = ops.spmm_csr

    def timed_spmm(g, x, *a, **k):
        if x.shape[1] != 256:
            return orig(g, x, *a, **k)
        a0, a1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a0.record(); out = orig(g, x, *a, **k); a1.record()
        evs.append((a0, a1))
        return out
    ops.spmm_csr = timed_spmm
    import efficient_gnns_b200.engine as eng
    eng.ops.spmm_csr = timed_spmm
    for it in range(6):
        if it == 2:
            evs.clear()
        tr.train_step(d["x"], d["y"], d["idx"], d["t"])
    torch.cuda.synchronize()
    ops.spmm_csr = orig
    k256_ms = sum(a.elapsed_time(b) for a, b in evs) / len(evs)
    alg = tr.spmm_algorithmic_bytes()[256]
    peak, peak_src = peaks()
    achieved = alg / (k256_ms * 1e-3) / 1e9

    # ---- parity of THIS run's engine against the fp64 CPU restatement, on the same inputs (one more eager step)
    parity = None
    if not args.no_parity:
        parity = parity_check(tr, ds, d)

    # ---- CPU baseline on this box's host cores (bounded sample)
    cpu = None
    if not args.no_cpu_baseline:
        cstep = CpuStep(ds)
        cores, tried = cstep.pick_threads("csr")
        t_csr, _ = cpu_reference_step_time(ds, 2, 0, "csr", cstep)
        cpu = {"value": 6 * nnz / t_csr, "unit": UNIT, "cores": cores, "kind": "port",
               "sample": f"2 full training steps of the same workload (oracle/, torch CPU, CSR SpMM form) on {cores} of "
                         f"{os.cpu_count()} host threads, the fastest of s/step {tried}"}

    line = {"metric": METRIC, "value": 6 * nnz / (ms_step * 1e-3), "unit": UNIT, "n_gpus": 1, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(ds, nnz),
            "engine": {"parallelism": "1 GPU", "cuda_graph": True, "hub_threshold": tr.G.hub_threshold,
                       "chunk_nnz": tr.G.chunk_nnz, "aggregations_executed": tr.aggregations_per_step(),
                       "edges_walked_per_s": sum(tr.aggregations_per_step().values()) * nnz / (ms_step * 1e-3),
                       "edges_note": "value counts the reference step's 6 aggregations (2*L*nnz); the engine executes "
                                     "layer 0 as (A_hat X) W, which needs 5 (edges_walked_per_s counts those)"},
            "parity_check": parity,
            "roofline": {"bound": "hbm", "kernel": "spmm_rows_bulk_kernel (cp.async.bulk ring), K=256 aggregation (2 of the 5 aggregations the engine runs per step; the reference runs 4 of 6 at this width)",
                         "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
                         "algorithmic_bytes_per_launch": alg, "ms_per_launch": k256_ms,
                         "launches_timed": len(evs), "peak_source": peak_src},
            "cpu_baseline": cpu,
            "e2e": {"value": 6 * nnz / (ms_e2e * 1e-3), "unit": UNIT, "ms_per_step": ms_e2e,
                    "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 12,
                    "note": "features, labels, teacher logits and train index re-uploaded from pinned host memory every "
                            "step (double-buffered, overlapping the previous step), 3 loss scalars read back"},
            "gpu_launches": launches * args.steps, "gpu_launches_per_step": launches,
            "clocks": clocks, "loss": losses}
    emit_json_line(line)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-graph", action="store_true")
    ap.add_argument("--no-parity", action="store_true", help="skip the fp64 CPU parity leg (~20 s of host time)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the last step's outputs as DIR/<name>.npy (1 GPU only)")
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be at least 1")
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if args.dump_outputs and (world > 1 or args.gpus > 1 or args.impl != "ours"):
        ap.error("--dump-outputs is implemented for the 1-GPU run of --impl ours")
    if args.impl == "reference":
        return run_reference(args)
    if world > 1 or args.gpus > 1:
        from efficient_gnns_b200 import dist_bench
        return dist_bench.run(args)
    return run_single(args)


if __name__ == "__main__":
    main()
