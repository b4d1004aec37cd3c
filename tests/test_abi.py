"""The C-ABI library loads and exports exactly what include/b200gnn.h declares (no compute calls)."""
import re
from pathlib import Path

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib

ROOT = Path(__file__).resolve().parents[1]


def header_functions():
    text = (ROOT / "include" / "b200gnn.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(b200gnn_[a-z0-9_]+)\s*\(", text)))


def test_library_loads_and_exports_every_declared_symbol():
    L = lib.load()
    names = header_functions()
    assert len(names) >= 9
    for n in names:
        assert hasattr(L, n), f"{n} declared in b200gnn.h but not exported"


def test_python_signature_table_matches_header():
    assert sorted(lib.SIGNATURES) == header_functions()


def test_abi_version_and_error_strings():
    L = lib.load()
    assert L.b200gnn_abi_version() == 2
    assert L.b200gnn_error_string(0) == b"ok"
    assert b"argument" in L.b200gnn_error_string(-1)
    assert L.b200gnn_spmm_stat_slots(17, 3) == 3 + 3
    assert L.b200gnn_csr_chunk_count(10, 100, 64, 4) == 3


def test_argument_validation_without_gpu():
    L = lib.load()
    # bad reduce / null pointers are rejected before any launch
    assert L.b200gnn_spmm_csr_f32(None, None, None, None, 4, None, 4, 5, 5, 4, 7, None, None, None, 1, 0, 1, None,
                                  None, 0, 0, None, None) == -1
    assert L.b200gnn_spmm_csr_f32(None, None, None, None, 4, None, 4, 5, 5, 4, 0, None, None, None, 1, 0, 1, None,
                                  None, 0, 0, None, None) == -1
    # empty problem is a no-op
    assert L.b200gnn_spmm_csr_f32(None, None, None, None, 4, None, 4, 0, 0, 4, 0, None, None, None, 0, 0, 1, None,
                                  None, 0, 0, None, None) == 0


def test_cpu_tensors_are_rejected_loudly():
    import pytest
    import torch
    from efficient_gnns_b200.sparse import SparseTensor
    adj = SparseTensor(row=torch.tensor([0, 1]), col=torch.tensor([1, 0]), sparse_sizes=(2, 2))
    with pytest.raises(lib.B200GnnError):
        adj.matmul(torch.ones(2, 4))
