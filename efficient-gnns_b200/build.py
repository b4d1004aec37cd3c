"""In-tree build of libb200gnn.so (hand-written sm_90a CUDA for the H100, behind a C ABI).

Plain ``nvcc -shared``: no torch headers, no JIT cache: the library is built
once into the package directory and loaded from there.  Rebuilds only when a source or
header is newer than the library.
"""
from __future__ import annotations

import os
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
INCLUDE = PKG_DIR.parent / "include"
LIB_PATH = PKG_DIR / "libb200gnn.so"

def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _stale() -> bool:
    if not LIB_PATH.exists():
        return True
    t = LIB_PATH.stat().st_mtime
    deps = sources() + sorted(CSRC.glob("*.cuh")) + sorted(INCLUDE.glob("*.h")) + [Path(__file__)]
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    if not force and not _stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    obj_dir = PKG_DIR / "build"
    obj_dir.mkdir(exist_ok=True)
    procs = []
    for src in sources():
        obj = obj_dir / (src.stem + ".o")
        objs.append(obj)
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
               "-Xcompiler", "-fPIC", "-Xptxas=-v", "-I", str(INCLUDE), "-I", str(CSRC),
               "-c", str(src), "-o", str(obj)]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    log = []
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        log.append(f"== {src.name}\n{out}")
        failed |= p.returncode != 0
    (obj_dir / "ptxas.log").write_text("\n".join(log))
    if failed:
        sys.stderr.write("\n".join(log))
        raise RuntimeError("nvcc failed building libb200gnn.so")
    if verbose:
        print("\n".join(log))
    link = [nvcc, "-shared", "-o", str(LIB_PATH)] + [str(o) for o in objs] + ["-lcudart"]
    subprocess.run(link, check=True)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
