"""G-CRD (nce_criterion) forward + backward at the scripts' S = 16384, F = 256 for several logits-chunk sizes
(criterion.NCE_CHUNK_BYTES): the chunk and its transpose are meant to stay L2-resident between the chunk's three GEMMs.
    python tools/bench_nce_chunk.py [S]"""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
import efficient_gnns_b200  # noqa: E402,F401
from efficient_gnns_b200 import criterion  # noqa: E402


def main():
    S = int(sys.argv[1]) if len(sys.argv) > 1 else 16384
    g = torch.Generator(device="cuda").manual_seed(0)
    fs = torch.randn(S, 256, device="cuda", generator=g).requires_grad_(True)
    ft = torch.randn(S, 256, device="cuda", generator=g)
    logits, labels = torch.randn(S, 40, device="cuda", generator=g), torch.randint(0, 40, (S,), device="cuda", generator=g)
    default = criterion.NCE_CHUNK_BYTES
    for mb in (8, 16, 32, 64):
        criterion.NCE_CHUNK_BYTES = mb << 20

        def step():
            fs.grad = None
            _, _, aux = criterion.nce_criterion(logits, labels, fs, ft, max_samples=S)
            aux.backward()
        for _ in range(3):
            step()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(10):
            step()
        e1.record()
        torch.cuda.synchronize()
        print(json.dumps(dict(S=S, chunk_MB=mb, default=(mb << 20) == default, ms=e0.elapsed_time(e1) / 10)), flush=True)
    criterion.NCE_CHUNK_BYTES = default


if __name__ == "__main__":
    main()
