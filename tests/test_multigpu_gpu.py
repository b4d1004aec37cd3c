"""Multi-rank equivalence inside the GPU suite: spawns torchrun on 2 (and 4) GPUs of the machine when they are
visible and skips otherwise (single-GPU machines).  The scripts compare the P-GPU step with the
1-GPU engine on the same inputs (tests/hybrid_equiv.py, tests/dist_equiv.py)."""
import os
import socket
import subprocess
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _torchrun(nproc, script, *args, timeout=600):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", "--master-addr", "127.0.0.1",
           "--master-port", str(_free_port()), str(ROOT / "tests" / script), *args]
    env = dict(os.environ)
    r = subprocess.run(cmd, cwd=str(ROOT), env=env, capture_output=True, text=True, timeout=timeout)
    return r.returncode, r.stdout[-4000:] + r.stderr[-2000:]


@pytest.mark.parametrize("nproc", [2, 4])
@pytest.mark.parametrize("mode", ["peer", "nccl"])
def test_hybrid_layout_step_equals_single_gpu(nproc, mode):
    if torch.cuda.device_count() < nproc:
        pytest.skip(f"needs {nproc} GPUs")
    rc, out = _torchrun(nproc, "hybrid_equiv.py", mode)
    assert rc == 0 and f"HYBRID_EQUIV {mode} P={nproc} PASS" in out, out


def test_allgather_node_parallel_step_equals_single_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rc, out = _torchrun(2, "dist_equiv.py")
    assert rc == 0 and "DIST_EQUIV PASS" in out, out


@pytest.mark.parametrize("mode", ["peer", "nccl"])
def test_head_parallel_gat_layer_equals_single_gpu(mode):
    """BASELINE configs[3] (GAT teacher, 1->8 GPUs): the head-parallel layer of hybrid_gat.py vs nn.DGLGATConv on one GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rc, out = _torchrun(2, "hybrid_gat_equiv.py", mode)
    assert rc == 0 and f"HYBRID_GAT_EQUIV {mode} P=2 PASS" in out, out


@pytest.mark.parametrize("mode", ["peer", "nccl"])
def test_feature_parallel_rgcn_inference_equals_single_gpu(mode):
    """BASELINE configs[4] (R-GCN on MAG-shape, 2/4/8 GPUs): rgcn.RGCNInference with per-type R<->C exchanges vs one GPU."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    rc, out = _torchrun(2, "hybrid_rgcn_equiv.py", mode)
    assert rc == 0 and f"HYBRID_RGCN_EQUIV {mode} P=2 PASS" in out, out
