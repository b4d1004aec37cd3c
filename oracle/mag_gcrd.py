"""One step of the reference's MAG ``train()`` with ``--training nce`` (mag_pyg/gnn_kd_and_aux.py:258-277, 424-441;
criterion.py:129-149), restated in float64 on the CPU or any device:

    out         = model(x_dict, b.edge_index, b.edge_attr, b.node_type, b.local_node_idx)[b.train_mask]   train mode
    teacher_out = teacher_model(...)[b.train_mask]                        eval, no_grad
    P_s         = student_proj(model.out_feat[b.train_mask])              Linear, BatchNorm1d (training), ReLU
    P_t         = teacher_proj(teacher_model.out_feat[b.train_mask])
    loss_aux    = nce_criterion(out, labels, P_s, P_t, beta, nce_T, max_samples)[2]      InfoNCE over S sampled rows
    loss        = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux
    one Adam over the model and both heads

The R-GCN forward is oracle/mag_lsp.py's (dropout keep masks injected), the heads and the InfoNCE oracle/gcrd.py's and
oracle/criterion.py's.  The sampled rows are an input (the reference draws them with np.random.choice, the engine with
Philox).  With no train row every term is a mean over nothing: the losses are NaN, the heads see no row (their running
statistics stay; num_batches_tracked still advances) and nothing carries a gradient.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import criterion as ocrit
from .gcrd import _head
from .mag_lsp import rgcn_forward


def nce_step_loss(student: Dict[str, torch.Tensor], teacher: Dict[str, torch.Tensor], sproj: Dict[str, torch.Tensor],
                  tproj: Dict[str, torch.Tensor], x_dict, batch, masks, sample: Optional[torch.Tensor], beta: float,
                  nce_T: float, student_layers: int = 2, teacher_layers: int = 3, alpha: float = 0.9, kd_T: float = 4.0,
                  bn_eps: float = 1e-5):
    """(loss, loss_cls, loss_aux, stats) of one step.  ``student`` and the heads' ``0.weight``, ``0.bias``, ``1.weight``,
    ``1.bias`` hold leaf tensors, so loss.backward() gives the gradients; ``sample``: positions into the train rows (None =
    every row); stats: {"sproj": (batch mean, biased var), "tproj": ...} for ``running_stats``, None with no train row."""
    logits, feat = rgcn_forward(student, x_dict, batch, student_layers, masks)
    with torch.no_grad():
        t_logits, t_feat = rgcn_forward(teacher, x_dict, batch, teacher_layers, None)
    tm = batch.train_mask.view(-1)
    out, labels = logits[tm], batch.y[tm].view(-1)
    loss, loss_cls, _ = ocrit.kd_criterion(out, labels, t_logits[tm], alpha, kd_T)
    if not bool(tm.any()):
        nan = torch.full((), float("nan"), dtype=logits.dtype, device=logits.device)
        return loss + beta * nan, loss_cls, nan, None
    ps, mu_s, var_s = _head(feat[tm], sproj, bn_eps)
    pt, mu_t, var_t = _head(t_feat[tm], tproj, bn_eps)
    S = ps.shape[0] if sample is None else len(sample)
    inds = None if sample is None else torch.as_tensor(sample, dtype=torch.long, device=ps.device)
    _, _, loss_aux = ocrit.nce_criterion(out, labels, ps, pt, beta, nce_T, S, sampled_inds=inds)
    return loss + beta * loss_aux, loss_cls, loss_aux, {"sproj": (mu_s, var_s), "tproj": (mu_t, var_t)}


def running_stats(sd: Dict[str, torch.Tensor], stats, n: int, momentum: float = 0.1) -> None:
    """BatchNorm1d's update of sd's running statistics in place from one batch of n rows (unbiased variance); stats
    (mean, biased var) of ``nce_step_loss``, or None for a batch without rows (nothing changes)."""
    if stats is None:
        return
    mu, var = (s.detach() for s in stats)
    with torch.no_grad():
        sd["1.running_mean"].mul_(1 - momentum).add_(momentum * mu)
        sd["1.running_var"].mul_(1 - momentum).add_(momentum * var * n / (n - 1))
