"""The PPI models of the reference (ppi_pyg/gnn.py:24-83, StudentNet and TeacherNet) restated functionally in plain torch
(CPU; the dtype follows the inputs, so the fp64 twin is the same code on double tensors).

PyG 1.7 ``GATConv`` (SURVEY Appendix A.6): a shared ``lin_l`` without bias, el = <x W, att_l>, er = <x W, att_r>, existing
self-loops removed and one per node added (duplicate edges kept), leaky_relu(0.2), softmax per destination with eps 1e-16,
concat or mean over heads, + bias.  Each layer adds a ``Linear`` skip on the same input; hidden layers are followed by ELU and
the last hidden activation is ``out_feat``.  Losses: ppi_pyg/gnn.py:203-212 and criterion.py:8-19.
"""
from __future__ import annotations

from typing import Dict, List, Tuple

import numpy as np
import torch
import torch.nn.functional as F

from . import graph as og, nn as onn

# (heads, width, concat) per layer of the two reference classes
STUDENT = [(2, 68, True)] * 4 + [(2, None, False)]
TEACHER = [(4, 256, True)] * 2 + [(6, None, False)]


def layers_of(kind: str, out_channels: int) -> List[Tuple[int, int, bool]]:
    spec = {"student": STUDENT, "teacher": TEACHER}[kind]
    return [(h, out_channels if d is None else d, c) for h, d, c in spec]


def adjacency(edge_index: torch.Tensor, n: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """(row = destination, col = source) as GATConv builds it: remove_self_loops + add_self_loops, duplicates kept."""
    ei = edge_index.cpu().numpy()
    r, c, _ = og.fill_diag(ei[1].astype(np.int64), ei[0].astype(np.int64), np.ones(ei.shape[1], dtype=np.float32), n)
    return torch.from_numpy(r), torch.from_numpy(c)


def gat_conv(x, row, col, lin_w, att_l, att_r, bias, heads: int, concat: bool, negative_slope: float = 0.2):
    n = x.shape[0]
    H = heads
    D = lin_w.shape[0] // H
    xl = F.linear(x, lin_w).view(n, H, D)
    el, er = (xl * att_l).sum(-1), (xl * att_r).sum(-1)
    out = onn.gat_aggregate(xl.reshape(n, H * D), el, er, row, col, n, H, negative_slope, softmax_eps=1e-16).view(n, H, D)
    out = out.reshape(n, H * D) if concat else out.mean(dim=1)
    return out + bias


def forward(x, row, col, state: Dict[str, torch.Tensor], layers) -> Tuple[torch.Tensor, torch.Tensor]:
    """StudentNet / TeacherNet.forward: returns (logits, out_feat)."""
    h, feat = x, None
    for i, (H, _, concat) in enumerate(layers, start=1):
        z = gat_conv(h, row, col, state[f"conv{i}.lin_l.weight"], state[f"conv{i}.att_l"], state[f"conv{i}.att_r"],
                     state[f"conv{i}.bias"], H, concat) + F.linear(h, state[f"lin{i}.weight"], state[f"lin{i}.bias"])
        if i < len(layers):
            h = feat = F.elu(z)
        else:
            h = z
    return h, feat


def loss(logits, y, teacher_logits=None, alpha: float = 0.5, T: float = 1.0):
    """(loss, loss_cls, loss_kd): BCE-with-logits over every entry, or criterion.py's kd_criterion."""
    loss_cls = F.binary_cross_entropy_with_logits(logits, y)
    if teacher_logits is None:
        return loss_cls, loss_cls, loss_cls * 0
    loss_kd = F.binary_cross_entropy_with_logits(logits, torch.sigmoid(teacher_logits))
    return loss_kd * (alpha * T * T) + loss_cls * (1 - alpha), loss_cls, loss_kd


def state_shapes(layers, in_channels: int) -> Dict[str, Tuple[int, ...]]:
    """Keys and shapes of the reference module's state_dict (conv*.lin_r.weight is PyG's alias of lin_l)."""
    shapes = {}
    fin = in_channels
    for i, (H, D, concat) in enumerate(layers, start=1):
        out = H * D if concat else D
        shapes[f"conv{i}.att_l"] = (1, H, D)
        shapes[f"conv{i}.att_r"] = (1, H, D)
        shapes[f"conv{i}.bias"] = (out,)
        shapes[f"conv{i}.lin_l.weight"] = (H * D, fin)
        shapes[f"conv{i}.lin_r.weight"] = (H * D, fin)
        shapes[f"lin{i}.weight"] = (out, fin)
        shapes[f"lin{i}.bias"] = (out,)
        fin = out
    return shapes


def seeded_state(layers, in_channels: int, seed: int) -> Dict[str, torch.Tensor]:
    """A reproducible state with every parameter non-trivial (biases included): N(0, 1/fan_in) weights, N(0, 0.3^2) attention
    vectors, N(0, 0.1^2) biases, drawn key by key from one CPU generator."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shp in state_shapes(layers, in_channels).items():
        if k.endswith("lin_r.weight"):
            sd[k] = sd[k.replace("lin_r", "lin_l")]
        elif k.endswith("weight"):
            sd[k] = torch.randn(shp, generator=g) / shp[1] ** 0.5
        elif ".att_" in k:
            sd[k] = torch.randn(shp, generator=g) * 0.3
        else:
            sd[k] = torch.randn(shp, generator=g) * 0.1
    return sd


def fingerprint(t: torch.Tensor, seed: int = 0, n_sample: int = 512) -> Dict[str, torch.Tensor]:
    """A compact, deterministic summary of a large tensor: fp64 column and row sums of its 2-D view and a seeded sample of its
    entries.  Small tensors are kept whole (``full``)."""
    t = t.detach()
    if t.numel() <= 8192:
        return {"full": t.clone()}
    m = t.reshape(t.shape[0], -1).double()
    idx = torch.randperm(t.numel(), generator=torch.Generator().manual_seed(seed))[:n_sample]
    return {"col": m.sum(0), "row": m.sum(1), "sample": t.reshape(-1)[idx].clone()}
