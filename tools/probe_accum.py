"""Does the tensor core's fp32 accumulate round to nearest or truncate, and what does that leave in the 3xTF32 kernels?

(a) tf32_mm: cuBLAS with TF32 enabled (wgmma on Hopper) on operands already rounded to tf32, so every product is exact in
    fp32 and the only error left is the accumulation.  With all-positive operands a round-to-nearest accumulator leaves a
    mean signed error near zero; a truncating one leaves a negative mean that grows with K.
(b) gemm / wgrad: signed error of this project's 3xTF32 kernels against fp64, random-sign and all-positive operands, next
    to torch.mm fp32 (TF32 off) on the same inputs.
One JSON line per case."""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import ops  # noqa: E402


def stats(c, ref):
    e = (c.double() - ref) / ref.abs().max()
    er = ((c.double() - ref) / ref.abs().clamp_min(1e-300))
    return dict(max_rel=float(e.abs().max()), fro_rel=float((c.double() - ref).norm() / ref.norm()),
                mean_signed_rel=float(er.mean()))


def tf32(x):
    return (x.view(torch.int32) + 0x1000 & -0x2000).view(torch.float32)      # round to nearest tf32, as the kernels do


def main():
    torch.manual_seed(0)
    dev = "cuda"
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(json.dumps(dict(device=torch.cuda.get_device_name(0), sms=sms)), flush=True)
    for K in (256, 4096, 65536):
        a, b = tf32(torch.rand(1024, K, device=dev)), tf32(torch.rand(256, K, device=dev))
        ref = a.double() @ b.double().t()
        torch.backends.cuda.matmul.allow_tf32 = True
        c = a @ b.t()
        torch.backends.cuda.matmul.allow_tf32 = False
        print(json.dumps(dict(op="tf32_mm", positive=True, K=K, cublas_tf32=stats(c, ref))), flush=True)
    for positive in (False, True):
        for K in (32, 128, 256, 1024):
            M, N = 4096, 256
            a = torch.randn(M, K, device=dev); b = torch.randn(N, K, device=dev)
            if positive:
                a, b = a.abs(), b.abs()
            ref = a.double() @ b.double().t()
            hi, lo = ops.split_tf32(b)
            c = ops.gemm_tf32x3(a, hi, lo)
            c32 = a @ b.t()
            print(json.dumps(dict(op="gemm", positive=positive, K=K, tf32x3=stats(c, ref), cublas_fp32=stats(c32, ref))), flush=True)
        for rows in (sms * 16, sms * 16 * 8, sms * 16 * 72):
            x = torch.randn(rows, 256, device=dev); g = torch.randn(rows, 256, device=dev)
            if positive:
                x, g = x.abs(), g.abs()
            ref = x.double().t() @ g.double()
            w = ops.gemm_wgrad_tf32x3(x, g)
            w32 = x.t() @ g
            print(json.dumps(dict(op="wgrad", positive=positive, rows=rows, tf32x3=stats(w, ref), cublas_fp32=stats(w32, ref))),
                  flush=True)


if __name__ == "__main__":
    main()
