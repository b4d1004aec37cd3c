"""Micro-benchmark: wgmma 3xTF32 GEMM vs cuBLAS fp32 (torch.mm) on the layer shapes of the ARXIV-shape GCN."""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import ops  # noqa: E402


def timeit(fn, iters=20):
    for _ in range(3):
        fn()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    M = 169_343
    for (K, N) in [(128, 256), (256, 256), (256, 40), (40, 256)]:
        a = torch.randn(M, K, device="cuda")
        w = torch.randn(N, K, device="cuda") / K ** 0.5
        hi, lo = ops.split_tf32(w)
        out = torch.empty(M, N, device="cuda")
        t_tc = timeit(lambda: ops.gemm_tf32x3(a, hi, lo, out=out))
        wt = w.t().contiguous()
        t_cb = timeit(lambda: torch.mm(a, wt, out=out))
        ref = (a[:4096].double() @ w.double().t())
        err = ((out[:4096].double() - ref).abs().max() / ref.abs().max()).item()
        flops = 2.0 * M * N * K
        print(json.dumps(dict(M=M, N=N, K=K, ms_wgmma=t_tc, ms_cublas_fp32=t_cb, tflops_effective=flops / t_tc / 1e9,
                              hbm_GBps=(M * K + M * N) * 4 / t_tc / 1e6, rel_err=err)), flush=True)


def bnbwd():
    """Input-gradient GEMM with the BatchNorm-backward reduction in its epilogue vs GEMM + separate reduce pass."""
    from efficient_gnns_b200 import lib
    M, N = 169_343, 256
    y = torch.randn(M, N, device="cuda")
    x_out = torch.relu(torch.randn(M, N, device="cuda"))
    mean, invstd = y.mean(0), (y.var(0, unbiased=False) + 1e-5).rsqrt()
    out = torch.empty(M, N, device="cuda")
    part = torch.empty(ops.gemm_stat_slots(M, N), 2, N, device="cuda")
    part2 = torch.empty(ops.rows_slots(M), 2, N, device="cuda")
    for K in (40, 256):
        a = torch.randn(M, K, device="cuda")
        hi, lo = ops.split_tf32(torch.randn(N, K, device="cuda"))
        res = dict(kind="bnbwd", M=M, N=N, K=K)
        res["ms_gemm"] = timeit(lambda: ops.gemm_tf32x3(a, hi, lo, out=out))
        res["ms_reduce_pass"] = timeit(lambda: ops.bn_act_bwd_reduce(out, x_out, y, mean, invstd, 0.5, part2))
        for variant, name in ((0, "ms_fused_auto"), (1, "ms_fused_tma"), (2, "ms_fused_regs")):
            lib.load().b200gnn_gemm_set_bnbwd_variant(variant)
            res[name] = timeit(lambda: ops.gemm_tf32x3_bnbwd(a, hi, lo, out, x_out, y, mean, invstd, 0.5, part))
        lib.load().b200gnn_gemm_set_bnbwd_variant(0)
        res["GBps_fused_tma"] = (M * K + 3 * M * N) * 4 / res["ms_fused_tma"] / 1e6
        print(json.dumps(res), flush=True)


def wgrad():
    from efficient_gnns_b200 import lib
    M = 169_343
    for (K, N) in [(128, 256), (256, 256), (256, 40)]:
        x = torch.randn(M, K, device="cuda"); d = torch.randn(M, N, device="cuda")
        out = torch.empty(K, N, device="cuda")
        ws = torch.empty(int(lib.load().b200gnn_wgrad_workspace_floats(K, N)), device="cuda")
        t_tc = timeit(lambda: ops.gemm_wgrad_tf32x3(x, d, out=out, workspace=ws))
        t_cb = timeit(lambda: torch.mm(x.t(), d, out=out))
        ref = x.double().t() @ d.double()
        err = ((out.double() - ref).norm() / ref.norm()).item()
        print(json.dumps(dict(kind="wgrad", Nn=M, Kin=K, Nout=N, ms_wgmma=t_tc, ms_cublas_fp32=t_cb, fro_err=err,
                              hbm_GBps=(M * K + M * N) * 4 / t_tc / 1e6)), flush=True)


if __name__ == "__main__":
    wgrad()
    bnbwd()
    main()
