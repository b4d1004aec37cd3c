import sys
from pathlib import Path

import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

GOLDEN = Path(__file__).resolve().parent / "golden"


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100)")


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def golden_criterion():
    return torch.load(GOLDEN / "criterion_arxiv.pt")


@pytest.fixture(scope="session")
def golden_model():
    return torch.load(GOLDEN / "model_arxiv.pt")


@pytest.fixture(scope="session")
def golden_gat():
    return torch.load(GOLDEN / "gat_arxiv.pt")


@pytest.fixture(scope="session")
def golden_rgcn():
    return torch.load(GOLDEN / "rgcn_mag.pt")


@pytest.fixture(scope="session")
def golden_sign():
    return torch.load(GOLDEN / "sign_arxiv.pt")


def rel_err(a: torch.Tensor, b: torch.Tensor) -> float:
    """max-norm relative error max|a-b| / max|b| (SURVEY.md §8c parity metric)."""
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    denom = b.abs().max().item()
    return (a - b).abs().max().item() / (denom if denom > 0 else 1.0)


def fro_err(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    denom = b.norm().item()
    return (a - b).norm().item() / (denom if denom > 0 else 1.0)
