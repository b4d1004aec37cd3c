"""CPU check that the data of tests/test_gat_layer_exact_gpu.py can tell a wrong fused GAT-layer kernel from a right one:
each subtly wrong formulation below, restated in fp32 on the CPU, must differ from the right one by more than that file's
check allows on that file's data."""
import pytest
import torch

from test_gat_layer_exact_gpu import TAIL_CASES, TAIL_IDS, U, _f32, near_zero, tail_data, tail_logits, tail_reference


@pytest.mark.parametrize("n,H,C,Dp,T,alpha,kd", [c for c in TAIL_CASES if c[1] > 1],
                         ids=[i for c, i in zip(TAIL_CASES, TAIL_IDS) if c[1] > 1])
def test_head_mean_by_reciprocal_differs_bitwise(n, H, C, Dp, T, alpha, kd):
    """s·(1/H) in place of s / H changes some logit's bits (the logits are compared bit for bit)."""
    agg, res, bc, bl, _, _ = tail_data(n, H, C, Dp, kd)
    s = agg[:, 0, :C].clone()
    for h in range(1, H):
        s = s + agg[:, h, :C]
    wrong = (s * (1.0 / float(H)) + bc[:C]) + (res[:, :C] + bl[:C])
    assert not torch.equal(wrong, tail_logits(agg, res, bc, bl, H, C))


def test_expf_minus_one_violates_the_elu_bound():
    """On the near-zero Z of the ELU check, fp32 expf(z) - 1 is outside the 1-ulp bound almost everywhere; fp32 expm1 is
    inside it everywhere."""
    z = near_zero((100_000,), torch.Generator().manual_seed(0)).float()
    e64 = torch.expm1(z.double())
    bound = 2 * U * e64.abs()
    assert bool(((torch.expm1(z).double() - e64).abs() <= bound).all())
    viol = (((torch.exp(z) - 1.0).double() - e64).abs() > bound).double().mean()
    assert float(viol) > 0.9, float(viol)


@pytest.mark.parametrize("n,H,C,Dp,T,alpha,kd", [c for c in TAIL_CASES if c[6] and c[5] > 0 and c[4] != 1.0],
                         ids=[i for c, i in zip(TAIL_CASES, TAIL_IDS) if c[6] and c[5] > 0 and c[4] != 1.0])
def test_kd_weight_without_T_squared_leaves_the_loss_bound(n, H, C, Dp, T, alpha, kd):
    """alpha in place of alpha·T² moves the loss by |alpha (T² - 1)|·loss_kd, far outside the loss bound at T = 2 and 0.5."""
    agg, res, bc, bl, y, t = tail_data(n, H, C, Dp, kd)
    ref = tail_reference(tail_logits(agg, res, bc, bl, H, C), y, t, alpha, T, kd)
    a32, T32 = _f32(alpha), _f32(T)
    shift = abs(ref["dis"] * a32 * (T32 * T32 - 1.0))
    assert shift > 10 * ref["B_loss"], (shift, ref["B_loss"])
