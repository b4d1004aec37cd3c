"""One step of the reference's MAG ``train()`` with ``--training lpw`` (mag_pyg/gnn_kd_and_aux.py:174-268), restated in
float64 on the CPU or any device:

    out         = model(x_dict, b.edge_index, b.edge_attr, b.node_type, b.local_node_idx)[b.train_mask]   train mode
    teacher_out = teacher_model(...)[b.train_mask]                        eval, no_grad
    t_feat      = teacher_model.out_feat[b.train_mask]                    ReLU of the teacher's last hidden layer
    out_feat    = model.out_feat[b.train_mask]                            the student's, after ReLU and dropout
    edge_index  = subgraph(b.train_mask.nonzero().squeeze(1), b.edge_index, relabel_nodes=True)[0]
    loss_aux    = lpw_criterion(out, labels, out_feat, t_feat, edge_index, kernel, beta)[2]          kld
    loss        = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux

The R-GCN forward is the reference's formulation (per relation the mean of the transformed messages, plus one root
transform per node type; mag_pyg/gnn.py:26-137) with the dropout masks injected: the reference hard-codes
F.dropout(p=0.5), so a caller passes the keep masks of each hidden layer.  With no train-induced edge the KL's mean runs
over no term and is NaN, as torch's kl_div(reduction='mean') gives it; the loss is then NaN and carries no LSP gradient.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import numpy as np
import torch

from . import criterion as ocrit
from .graph import subgraph
from .ops import segment_softmax


def rgcn_forward(params: Dict[str, torch.Tensor], x_dict: Dict[int, torch.Tensor], batch, num_layers: int,
                 masks: Optional[Sequence[torch.Tensor]] = None, p: float = 0.5):
    """RGCN.forward in the dtype of ``params``: (logits [N, C], out_feat [N, H] of the last hidden layer).  masks: one keep
    mask [N, H] per hidden layer (training), or None (eval: no dropout)."""
    nt, li = batch.node_type.view(-1), batch.local_node_idx.view(-1)
    dt = next(iter(params.values())).dtype
    dev = nt.device
    n = nt.numel()
    types = sorted({int(k.split(".")[3]) for k in params if k.startswith("convs.0.root_lins.")})
    R = sum(1 for k in params if k.startswith("convs.0.rel_lins."))
    h = torch.zeros(n, params["convs.0.root_lins.0.weight"].shape[1], dtype=dt, device=dev)
    for t in types:
        m = nt == t
        tab = x_dict[t].to(dt) if t in x_dict else params[f"emb_dict.{t}"]
        h = h.index_put((m.nonzero().view(-1),), tab[li[m]])
    src, dst = batch.edge_index
    et = batch.edge_attr.view(-1)
    feat = None
    for i in range(num_layers):
        out = torch.zeros(n, params[f"convs.{i}.root_lins.0.weight"].shape[0], dtype=dt, device=dev)
        for r in range(R):
            m = et == r
            msg = h[src[m]] @ params[f"convs.{i}.rel_lins.{r}.weight"].t()
            agg = torch.zeros_like(out).index_add(0, dst[m], msg)
            cnt = torch.zeros(n, dtype=dt, device=dev).index_add(0, dst[m], torch.ones(int(m.sum()), dtype=dt, device=dev))
            out = out + agg / cnt.clamp(min=1)[:, None]
        for t in types:
            m = (nt == t).nonzero().view(-1)
            out = out.index_add(0, m, h[m] @ params[f"convs.{i}.root_lins.{t}.weight"].t()
                                + params[f"convs.{i}.root_lins.{t}.bias"])
        if i != num_layers - 1:
            out = torch.relu(out)
            if masks is not None:
                out = out * masks[i].to(dt) / (1 - p)
            feat = out
        h = out
    return h, feat


def _edge_similarity(feat, src, dst, kernel: str):
    """oracle.criterion._edge_similarity with the cosine norms taken by a square root whose derivative at 0 is 0, as torch's
    norm backward takes it: a student row can be all zero after ReLU and dropout, and its (zero) gradient must stay finite."""
    a, b = feat.index_select(0, src), feat.index_select(0, dst)
    if kernel in ("cosine", "poly"):
        na = ocrit._safe_sqrt(a.pow(2).sum(-1)).clamp_min(1e-8)
        nb = ocrit._safe_sqrt(b.pow(2).sum(-1)).clamp_min(1e-8)
        c = (a * b).sum(-1) / (na * nb)
        return c if kernel == "cosine" else c * c
    return ocrit._edge_similarity(feat, src, dst, kernel)


def lpw_kld(feat, teacher_feat, edge_index, kernel: str):
    """lpw_criterion's loss_aux, kld form (criterion.py:95-126): KL(softmax_dst(sim_t) || softmax_dst(sim_s)), mean over the
    E edges; NaN when E = 0."""
    src, dst = edge_index[0], edge_index[1]
    if src.numel() == 0:
        return torch.full((), float("nan"), dtype=feat.dtype, device=feat.device)
    ps = segment_softmax(_edge_similarity(feat, src, dst, kernel), dst)
    pt = segment_softmax(_edge_similarity(teacher_feat, src, dst, kernel), dst)
    return ocrit._kl_elementwise_mean(ps.log(), pt)


def train_induced_edges(train_mask: torch.Tensor, edge_index: torch.Tensor) -> torch.Tensor:
    """subgraph(train_mask.nonzero().squeeze(1), edge_index, relabel_nodes=True)[0]."""
    sub = train_mask.view(-1).nonzero().view(-1).cpu().numpy()
    ei = subgraph(sub, edge_index.cpu().numpy(), True)[0]
    return torch.from_numpy(np.ascontiguousarray(ei)).to(edge_index.device)


def lpw_step_loss(student: Dict[str, torch.Tensor], teacher: Dict[str, torch.Tensor], x_dict, batch, masks, kernel: str,
                  beta: float, student_layers: int = 2, teacher_layers: int = 3, alpha: float = 0.9, kd_T: float = 4.0):
    """(loss, loss_cls, loss_aux) of one step; ``student`` holds leaf tensors, so loss.backward() gives the gradients."""
    logits, feat = rgcn_forward(student, x_dict, batch, student_layers, masks)
    with torch.no_grad():
        t_logits, t_feat = rgcn_forward(teacher, x_dict, batch, teacher_layers, None)
    tm = batch.train_mask.view(-1)
    out, labels = logits[tm], batch.y[tm].view(-1)
    ei = train_induced_edges(tm, batch.edge_index)
    loss_aux = lpw_kld(feat[tm], t_feat[tm], ei, kernel)
    loss, loss_cls, _ = ocrit.kd_criterion(out, labels, t_logits[tm], alpha, kd_T)
    return loss + beta * loss_aux, loss_cls, loss_aux


def adam(params: Dict[str, torch.Tensor], m: Dict[str, torch.Tensor], v: Dict[str, torch.Tensor], step: int, lr: float,
         b1: float = 0.9, b2: float = 0.999, eps: float = 1e-8) -> None:
    """torch.optim.Adam's update (no weight decay, no amsgrad) of every parameter with a gradient, step counted from 1."""
    with torch.no_grad():
        for k, p in params.items():
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            m[k].mul_(b1).add_(g, alpha=1 - b1)
            v[k].mul_(b2).addcmul_(g, g, value=1 - b2)
            denom = (v[k] / (1 - b2 ** step)).sqrt() + eps
            p.sub_(lr / (1 - b1 ** step) * m[k] / denom)
