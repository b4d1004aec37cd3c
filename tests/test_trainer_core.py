"""The host plumbing every fused trainer shares (efficient-gnns_b200/trainer.py), on the CPU: the flat parameter store's
layout and its views, save / restore, and the autograd bridge of ``train_step(aux=)``."""
import pytest
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200.trainer import FlatParams, aux_grad, one_objective

SHAPES = [(3, 5), (5,), (7,), (2, 2, 3), (1,)]


def test_views_sit_in_declaration_order_back_to_back():
    st = FlatParams(SHAPES, "cpu")
    off = 0
    for (p, g), shape in zip(st.views, SHAPES):
        n = torch.Size(shape).numel()
        assert p.shape == g.shape == shape and p.is_contiguous() and g.is_contiguous()
        assert st.offset(p) == st.offset(g) == off
        assert p.untyped_storage().data_ptr() == st.params.untyped_storage().data_ptr()
        assert g.untyped_storage().data_ptr() == st._grads_buf.untyped_storage().data_ptr()
        off += n
    assert st.params.numel() == st.grads.numel() == st.exp_avg.numel() == st.exp_avg_sq.numel() == off
    assert st.step_count.dtype == torch.int32 and st.step_count.numel() == 1


@pytest.mark.parametrize("shapes", [SHAPES, [(4,)], [(1,)], [(2,), (3,)], [(5, 3), (2,)]])
def test_grads_exclude_the_loss_tail_which_is_16_byte_aligned(shapes):
    st = FlatParams(shapes, "cpu")
    n = st.params.numel()
    assert st.grads.storage_offset() == 0 and st.grads.numel() == n
    assert st.n_par_pad % 4 == 0 and n <= st.n_par_pad < n + 4
    assert st.loss_out.numel() == 3 and st.loss_out.storage_offset() == st.n_par_pad
    assert st._grads_buf.numel() == st.n_par_pad + 4
    st.grads.fill_(1.0)
    assert not st.loss_out.any()
    st.loss_out.fill_(2.0)
    assert (st.grads == 1.0).all()


def test_like_is_the_same_view_in_another_flat_buffer():
    st = FlatParams(SHAPES, "cpu")
    other = torch.arange(st.params.numel(), dtype=torch.float32)
    for p, g in st.views:
        o = st.offset(p)
        v = st.like(other, p)
        assert v.shape == p.shape
        assert torch.equal(v.reshape(-1), other[o:o + p.numel()])
        assert torch.equal(st.like(other, g), v)
        v.zero_()
    assert not other.any()


def test_attach_publishes_the_buffers_under_the_trainer_names():
    class T:
        pass
    t = T()
    st = FlatParams(SHAPES, "cpu").attach(t)
    for k in ("params", "grads", "_grads_buf", "loss_out", "exp_avg", "exp_avg_sq", "step_count"):
        assert getattr(t, k) is getattr(st, k)
    assert t.n_par_pad == st.n_par_pad


def test_preserved_round_trips_params_adam_state_and_counter():
    st = FlatParams(SHAPES, "cpu")
    g = torch.Generator().manual_seed(0)
    for t in (st.params, st.exp_avg, st.exp_avg_sq):
        t.copy_(torch.randn(t.shape, generator=g))
    st.step_count.fill_(7)
    before = [t.clone() for t in (st.params, st.exp_avg, st.exp_avg_sq, st.step_count)]
    with st.preserved():
        for t in (st.params, st.exp_avg, st.exp_avg_sq):
            t.add_(1.0)
        st.step_count.add_(3)
    for t, b in zip((st.params, st.exp_avg, st.exp_avg_sq, st.step_count), before):
        assert torch.equal(t, b)


def test_aux_grad_equals_autograd_and_returns_a_detached_loss():
    g = torch.Generator().manual_seed(1)
    f = torch.randn(6, 4, generator=g)
    w = torch.randn(4, generator=g)
    aux = lambda x: ((x * w).tanh().sum(1) ** 2).mean()            # noqa: E731
    beta = 0.7
    d, loss = aux_grad(f, aux, beta)
    fr = f.clone().requires_grad_(True)
    want, = torch.autograd.grad(aux(fr) * beta, fr)
    assert torch.equal(d, want) and d.is_contiguous()
    assert not loss.requires_grad and torch.equal(loss, aux(f))
    assert not f.requires_grad and f.grad is None


def test_aux_grad_is_zero_when_aux_ignores_its_input():
    f = torch.randn(5, 3)
    d, loss = aux_grad(f, lambda x: torch.tensor(2.0, requires_grad=True), 0.5)
    assert d.shape == f.shape and not d.any()
    assert not loss.requires_grad and loss.item() == 2.0


def test_at_most_one_objective():
    a, b, c = object(), object(), object()
    assert one_objective() is None
    assert one_objective(gcrd=a) is a and one_objective(lsp=b) is b and one_objective(gsp=c) is c
    with pytest.raises(ValueError):
        one_objective(gcrd=a, lsp=b)
    for kw in (dict(gcrd=a, gsp=c), dict(lsp=b, gsp=c)):
        with pytest.raises(ValueError):
            one_objective(**kw)
