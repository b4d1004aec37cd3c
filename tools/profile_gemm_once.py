"""A few launches of the two tensor-core kernels at the benchmark's largest shapes, for `ncu --set full` captures
(shared-memory traffic behind DESIGN §4.2's bound).  usage: python tools/profile_gemm_once.py {gemm|wgrad}"""
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import ops  # noqa: E402

M, K, N = 169_343, 256, 256
x = torch.randn(M, K, device="cuda")
if sys.argv[1] == "gemm":
    hi, lo = ops.split_tf32(torch.randn(N, K, device="cuda") / 16)
    out = torch.empty(M, N, device="cuda")
    for _ in range(4):
        ops.gemm_tf32x3(x, hi, lo, out=out)
else:
    g = torch.randn(M, N, device="cuda")
    out, ws = torch.empty(K, N, device="cuda"), torch.empty(ops.wgrad_workspace_floats(K, N), device="cuda")
    for _ in range(4):
        ops.gemm_wgrad_tf32x3(x, g, out=out, workspace=ws)
torch.cuda.synchronize()
