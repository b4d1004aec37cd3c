"""Dense row passes, Adam and the KD row loss (through the C ABI) vs fp64 PyTorch-CPU references."""
import pytest
import torch
import torch.nn.functional as F

import efficient_gnns_b200  # noqa: F401
from conftest import rel_err
from efficient_gnns_b200 import ops
from oracle import criterion as oc

pytestmark = pytest.mark.gpu


def test_dropout_mask_is_replayable_and_unbiased():
    n, K, p = 4000, 256, 0.5
    y = torch.ones(n, K, device="cuda")
    a = ops.affine_relu_dropout(y, relu=False, p=p, seed=7, offset=3)
    m = ops.dropout_mask(n, K, p, 7, 3)
    assert torch.equal(a > 0, m.bool()) and torch.all(a[m.bool()] == 2.0)
    step = torch.tensor([5], dtype=torch.int32, device="cuda")
    b = ops.affine_relu_dropout(y, relu=False, p=p, seed=7, offset=1, step_dev=step, step_mul=3)
    assert torch.equal(b > 0, ops.dropout_mask(n, K, p, 7, 16).bool())
    assert not torch.equal(a, b)
    assert abs(float(m.float().mean()) - 0.5) < 5e-3
    # columns/rows are not correlated with the element index pattern
    assert float(m.float().mean(0).std()) < 0.02 and float(m.float().mean(1).std()) < 0.06


def test_col_sum():
    y = torch.randn(12345, 40, generator=torch.Generator().manual_seed(0))
    assert rel_err(ops.col_sum(y.cuda()), y.double().sum(0)) < 1e-5


def test_adam_matches_torch_optim():
    g = torch.Generator().manual_seed(0)
    p0 = torch.randn(10_007, generator=g)
    ref = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref], lr=0.01)
    pc, m, v = p0.cuda(), torch.zeros(10_007, device="cuda"), torch.zeros(10_007, device="cuda")
    step = torch.zeros(1, dtype=torch.int32, device="cuda")
    for it in range(5):
        gr = torch.randn(10_007, generator=g) * (10.0 ** (it - 3))
        ref.grad = gr.clone(); opt.step()
        ops.adam_step(pc, gr.cuda(), m, v, step, 0.01)
    assert int(step.item()) == 5
    assert (pc.cpu() - ref.detach()).abs().max().item() < 1e-6


@pytest.mark.parametrize("C", [8, 40, 47, 256])
@pytest.mark.parametrize("kd", [True, False])
def test_kd_loss_matches_oracle(C, kd):
    n, nt = 5000, 2600
    g = torch.Generator().manual_seed(C)
    z = torch.randn(n, C, generator=g) * 3
    t = torch.randn(n, C, generator=g) * 2
    y = torch.randint(0, C, (n,), generator=g)
    idx = torch.randperm(n, generator=g)[:nt].sort().values
    zr = z.double().requires_grad_(True)
    if kd:
        loss, lc, lk = oc.kd_criterion(zr[idx], y[idx], t.double()[idx], 0.9, 4.0)
    else:
        loss = lc = oc.cross_entropy(zr[idx], y[idx]); lk = loss * 0
    loss.backward()
    out, dz = ops.kd_loss_fwd_bwd(z.cuda(), y.cuda(), idx.cuda(), t.cuda() if kd else None, 0.9, 4.0)
    out = out.cpu()
    assert abs(out[0] - loss.item()) < 1e-5 * abs(loss.item())
    assert abs(out[1] - lc.item()) < 1e-5 * abs(lc.item())
    if kd:
        assert abs(out[2] - lk.item()) < 1e-5 * abs(lk.item())
    assert rel_err(dz, zr.grad) < 1e-5
    # also equals torch.nn.functional on the same rows (what the reference file calls)
    ref_ce = F.cross_entropy(z[idx].double(), y[idx])
    assert abs(out[1] - ref_ce.item()) < 1e-5 * abs(ref_ce.item())
