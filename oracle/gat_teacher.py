"""The arxiv GAT teacher's recipe (arxiv_dgl/gat.py) restated in plain torch on top of oracle/gat.py (CPU; the dtype follows
the inputs).  The random draws are injected: the label mask of a step (``torch.rand(n_train) < mask_rate``, gat.py:122 /
:129) and, per training forward, the (input, hidden, edge) keep masks of oracle.gat.gat_forward.

    custom_loss      gat.py:98-101     mean(log(eps + CE_i) - log eps), eps = 1 - ln 2
    add_labels       gat.py:104-107    [feat | one-hot of the rows idx]
    train            gat.py:116-148    label mask, forward, n_label_iters label-reuse forwards, loss on the last, BatchNorm
                                       running statistics updated by every training forward
    rmsprop_step     torch.optim.RMSprop (no momentum, not centred) at the rate of adjust_learning_rate (gat.py:110-113)
    evaluate         gat.py:151-183
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from . import gat as ogat

EPSILON = 1 - math.log(2)


def custom_loss(x, labels):
    y = F.cross_entropy(x, labels, reduction="none")
    return torch.mean(torch.log(EPSILON + y) - math.log(EPSILON))


def add_labels(feat, labels, idx, n_classes: int):
    onehot = torch.zeros(feat.shape[0], n_classes, dtype=feat.dtype)
    onehot[idx, labels[idx]] = 1
    return torch.cat([feat, onehot], dim=-1)


def lr_at(lr: float, epoch: int, warmup: int = 50) -> float:
    """adjust_learning_rate: the rate of epoch ``epoch`` (1-based)."""
    return lr * min(epoch, warmup) / warmup


def accuracy(pred, labels):
    return (pred.argmax(dim=-1) == labels).to(pred.dtype).mean()


def forward(x, row, col, state, n_layers, n_heads, sym, training, p=0.0, p_in=0.0, draws=None, bn_eps=1e-5,
            bn_momentum=0.1):
    """oracle.gat.gat_forward, and in training mode the update of the BatchNorm running statistics in ``state`` (in place,
    torch.nn.BatchNorm1d: unbiased batch variance).  The batch statistics come from the same layers (oracle.gat.gat_conv)."""
    inp, hid, edge = draws if draws is not None else (None, None, None)
    logits, feat = ogat.gat_forward(x, row, col, state, n_layers, n_heads, sym, training, p, p_in, inp, hid, edge, bn_eps)
    if training:
        with torch.no_grad():
            n = x.shape[0]
            h = x if inp is None else x * inp.to(x.dtype) / (1.0 - p_in)
            for i in range(n_layers - 1):
                h = ogat.gat_conv(h, row, col, n, state[f"convs.{i}.fc.weight"], state[f"convs.{i}.attn_l"],
                                  state.get(f"convs.{i}.attn_r"), state[f"convs.{i}.res_fc.weight"], n_heads, sym,
                                  None if edge is None else edge[i]).flatten(1)
                m, v = h.mean(0), h.var(0, unbiased=False)
                rm, rv = state[f"norms.{i}.running_mean"], state[f"norms.{i}.running_var"]
                rm.mul_(1 - bn_momentum).add_(bn_momentum * m)
                rv.mul_(1 - bn_momentum).add_(bn_momentum * v * n / (n - 1))
                h = torch.relu((h - m) / torch.sqrt(v + bn_eps) * state[f"norms.{i}.weight"] + state[f"norms.{i}.bias"])
                if hid is not None:
                    h = h * hid[i].to(h.dtype) / (1.0 - p)
    return logits, feat


def train(x, labels, row, col, train_idx, val_idx, test_idx, state: Dict[str, torch.Tensor], n_layers: int, n_heads: int,
          n_classes: int, use_labels: bool, n_label_iters: int, mask, draws: Optional[Sequence] = None, p: float = 0.0,
          p_in: float = 0.0, sym: bool = True):
    """gat.py:116-148 without the optimizer step.  state: parameters (requires_grad) and running statistics (updated).
    mask: bool[n_train] of the step; draws[f]: the keep masks of training forward f (None: no dropout).
    Returns (acc, loss, pred of the last forward, train_pred_idx); the parameters hold their gradients."""
    draws = draws if draws is not None else [None] * (n_label_iters + 1)
    feat = x
    if use_labels:
        train_pred_idx = train_idx[~mask]
        feat = add_labels(feat, labels, train_idx[mask], n_classes)
    else:
        train_pred_idx = train_idx[mask]
    pred, _ = forward(feat, row, col, state, n_layers, n_heads, sym, True, p, p_in, draws[0])
    if n_label_iters > 0:
        unlabel_idx = torch.cat([train_pred_idx, val_idx, test_idx])
        for it in range(n_label_iters):
            pred = pred.detach()
            feat = feat.clone()
            feat[unlabel_idx, -n_classes:] = F.softmax(pred[unlabel_idx], dim=-1)
            pred, _ = forward(feat, row, col, state, n_layers, n_heads, sym, True, p, p_in, draws[it + 1])
    loss = custom_loss(pred[train_pred_idx], labels[train_pred_idx])
    loss.backward()
    return accuracy(pred[train_idx].detach(), labels[train_idx]), loss.detach(), pred.detach(), train_pred_idx


@torch.no_grad()
def rmsprop_step(params: List[torch.Tensor], grads: List[torch.Tensor], square_avg: List[torch.Tensor], lr: float,
                 alpha: float = 0.99, eps: float = 1e-8, weight_decay: float = 0.0):
    """torch.optim.RMSprop's update, in the dtype of the tensors (in place)."""
    for p_, g, sq in zip(params, grads, square_avg):
        g = g + weight_decay * p_ if weight_decay else g
        sq.mul_(alpha).add_((1 - alpha) * g * g)
        p_.sub_(lr * g / (sq.sqrt() + eps))


@torch.no_grad()
def evaluate(x, labels, row, col, train_idx, val_idx, test_idx, state, n_layers: int, n_heads: int, n_classes: int,
             use_labels: bool, n_label_iters: int, sym: bool = True):
    """gat.py:151-183.  Returns ([train, val, test] accuracies, [train, val, test] losses, pred, feat)."""
    feat = add_labels(x, labels, train_idx, n_classes) if use_labels else x
    pred, h = forward(feat, row, col, state, n_layers, n_heads, sym, False)
    if n_label_iters > 0:
        unlabel_idx = torch.cat([val_idx, test_idx])
        for _ in range(n_label_iters):
            feat = feat.clone()
            feat[unlabel_idx, -n_classes:] = F.softmax(pred[unlabel_idx], dim=-1)
            pred, h = forward(feat, row, col, state, n_layers, n_heads, sym, False)
    idx = (train_idx, val_idx, test_idx)
    return ([accuracy(pred[i], labels[i]) for i in idx], [custom_loss(pred[i], labels[i]) for i in idx], pred, h)
