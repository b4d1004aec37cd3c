"""fp64 restatement of one reference PPI ``train()`` step with ``--training gpw`` (ppi_pyg/gnn.py:230-239; criterion.py:54-89):
StudentNet (oracle/ppi.py) on the whole graph, GSP between its out_feat and the teacher's out_feat over a sample of rows
(oracle/criterion.py's pairwise similarities, no projection heads) and one Adam step over the model.  The sampled rows are
an input (the reference draws them with np.random.choice, the engine with Philox)."""
from __future__ import annotations

from typing import Dict

import torch

from . import criterion as oc
from .ppi import adjacency, forward, layers_of, loss


def gsp_step(x, y, edge_index, model: Dict[str, torch.Tensor], t_feat, kernel: str, sample=None, beta: float = 100.0,
             lr: float = 0.005, teacher_logits=None, alpha: float = 0.5, T: float = 1.0, adam_eps: float = 1e-8,
             dtype=torch.float64):
    """One reference PPI ``train()`` step with ``--training gpw`` restated in ``dtype``: StudentNet (``model``) on the whole
    graph, loss = BCE (or kd_criterion) + beta * mean((sim_s - sim_t)^2) over ``sample`` (positions, None = every row) and
    one Adam step from zero moments.  Returns dict(loss=[loss, loss_cls, loss_aux], grads, after) keyed by the model's
    state-dict names (lin_r, PyG's alias of lin_l, left out)."""
    n = x.shape[0]
    layers = layers_of("student", y.shape[1])
    m = {k: v.to(dtype, copy=True).requires_grad_(True) for k, v in model.items() if "lin_r" not in k}
    st = dict(m)
    st.update({k.replace("lin_l", "lin_r"): v for k, v in m.items() if "lin_l" in k})
    row, col = adjacency(edge_index, n)
    logits, feat = forward(x.to(dtype), row, col, st, layers)
    tl = None if teacher_logits is None else teacher_logits.to(dtype)
    loss_main, loss_cls, _ = loss(logits, y.to(dtype), tl, alpha, T)
    tf = t_feat.to(dtype)
    if sample is not None:
        inds = torch.as_tensor(sample, dtype=torch.long)
        feat, tf = feat[inds], tf[inds]
    loss_aux = (oc._pairwise(feat, kernel) - oc._pairwise(tf, kernel)).pow(2).mean()
    total = loss_main + beta * loss_aux
    keys = list(m)
    gr = torch.autograd.grad(total, [m[k] for k in keys])
    grads = dict(zip(keys, gr))
    after = {k: m[k].detach() - lr * g / (g.abs() + adam_eps) for k, g in grads.items()}   # Adam step 1: m_hat = g, v_hat = g^2
    return dict(loss=torch.stack([total, loss_cls, loss_aux]).detach(), grads=grads, after=after)
