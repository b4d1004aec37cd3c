"""One step of the reference's MAG ``train()`` with ``--training gpw`` (mag_pyg/gnn_kd_and_aux.py:229-242; criterion.py:57-92),
restated in float64 on the CPU or any device:

    out         = model(x_dict, b.edge_index, b.edge_attr, b.node_type, b.local_node_idx)[b.train_mask]   train mode
    teacher_out = teacher_model(...)[b.train_mask]                        eval, no_grad
    t_feat      = teacher_model.out_feat[b.train_mask]                    ReLU of the teacher's last hidden layer
    out_feat    = model.out_feat[b.train_mask]                            the student's, after ReLU and dropout
    loss_aux    = mean((sim(out_feat[inds]) - sim(t_feat[inds]))^2)      over S x S pairs, no projection heads
    loss        = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux

The R-GCN forward is oracle/mag_lsp.py's (dropout keep masks injected), the pairwise similarities oracle/criterion.py's.
The sampled rows are an input (the reference draws them with np.random.choice, the engine with Philox).  With no train row
the mse runs over no pair and is NaN, as F.mse_loss gives it; the loss is then NaN and carries no GSP gradient.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import criterion as ocrit
from .mag_lsp import rgcn_forward


def gsp_loss(feat: torch.Tensor, t_feat: torch.Tensor, kernel: str, sample: Optional[torch.Tensor] = None) -> torch.Tensor:
    """mean((sim_s - sim_t)^2) over the S x S pairs of the rows ``sample`` (positions; None = every row)."""
    if sample is not None:
        inds = torch.as_tensor(sample, dtype=torch.long, device=feat.device)
        feat, t_feat = feat[inds], t_feat[inds]
    if feat.shape[0] == 0:
        return torch.full((), float("nan"), dtype=feat.dtype, device=feat.device)
    return (ocrit._pairwise(feat, kernel) - ocrit._pairwise(t_feat, kernel)).pow(2).mean()


def gpw_step_loss(student: Dict[str, torch.Tensor], teacher: Dict[str, torch.Tensor], x_dict, batch, masks, kernel: str,
                  sample: Optional[torch.Tensor], beta: float, student_layers: int = 2, teacher_layers: int = 3,
                  alpha: float = 0.9, kd_T: float = 4.0):
    """(loss, loss_cls, loss_aux) of one step; ``student`` holds leaf tensors, so loss.backward() gives the gradients.
    ``sample``: positions into the train rows (None = every row)."""
    logits, feat = rgcn_forward(student, x_dict, batch, student_layers, masks)
    with torch.no_grad():
        t_logits, t_feat = rgcn_forward(teacher, x_dict, batch, teacher_layers, None)
    tm = batch.train_mask.view(-1)
    out, labels = logits[tm], batch.y[tm].view(-1)
    loss_aux = gsp_loss(feat[tm], t_feat[tm], kernel, sample)
    loss, loss_cls, _ = ocrit.kd_criterion(out, labels, t_logits[tm], alpha, kd_T)
    return loss + beta * loss_aux, loss_cls, loss_aux
