"""The reference's DGL ``GAT`` model restated functionally in plain torch (CPU; the dtype follows the inputs, so the fp64
twin is the same code on double tensors).

``GAT.forward`` arxiv_dgl/models.py:293-313: input_drop (:295) -> per layer GATConv (:298, restated from :154-236) ->
hidden layers flatten, BatchNorm1d, ReLU, dropout (:302-308, ``feat`` = the last hidden activation) -> mean over the last
layer's single head (:310) -> bias_last (:311).  The random draws are injected: ``in_keep`` [N, in] and ``hid_keep[l]``
[N, H*D] are dropout keep masks (kept entries are scaled by 1/(1-p), torch.nn.Dropout), ``edge_keep[l]`` [nnz] removes edges
from the softmax of layer l (:207-212: dropped edges get a = 0; which edges are dropped is the caller's draw).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn.functional as F


def gat_conv(h, row, col, n: int, fc_w, attn_l, attn_r, res_w, heads: int, symmetric_norm: bool, edge_keep=None,
             negative_slope: float = 0.2):
    """GATConv.forward (models.py:154-236) with residual; row = destination, col = source.  Returns [n, H, D]."""
    H = heads
    D = fc_w.shape[0] // H
    ft = F.linear(h, fc_w).view(-1, H, D)                                       # :171
    ft_dst = ft                                                                 # :177 bound before the rescale of :184
    if symmetric_norm:
        ft = ft * torch.bincount(col, minlength=n).clamp(min=1).to(h.dtype).pow(-0.5).view(-1, 1, 1)   # :179-184
    el = (ft * attn_l).sum(-1)                                                  # :196
    e = el.index_select(0, col)
    if attn_r is not None:
        e = e + (ft_dst * attn_r).sum(-1).index_select(0, row)                 # :200-202
    e = F.leaky_relu(e, negative_slope)                                         # :205
    keep = torch.ones(row.numel(), dtype=torch.bool) if edge_keep is None else edge_keep.bool()
    r_k, c_k, e_k = row[keep], col[keep], e[keep]
    idx = r_k.view(-1, 1).expand_as(e_k)
    m = torch.full((n, H), float("-inf"), dtype=e.dtype).scatter_reduce_(0, idx, e_k.detach(), "amax", include_self=True)
    ex = (e_k - m.index_select(0, r_k)).exp()
    s = torch.zeros(n, H, dtype=e.dtype).scatter_add_(0, idx, ex)
    a = ex / s.index_select(0, r_k)                                             # edge_softmax over the kept edges, :207-214
    msg = ft.index_select(0, c_k) * a.unsqueeze(-1)
    rst = torch.zeros(n, H, D, dtype=h.dtype).index_add_(0, r_k, msg)           # :217
    if symmetric_norm:
        rst = rst * torch.bincount(row, minlength=n).clamp(min=1).to(h.dtype).pow(0.5).view(-1, 1, 1)  # :220-225
    return rst + F.linear(h, res_w).view(n, H, D)                               # :228-230


def gat_forward(x, row, col, state: Dict[str, torch.Tensor], n_layers: int, n_heads: int, use_symmetric_norm: bool,
                training: bool = True, p: float = 0.0, p_in: float = 0.0, in_keep: Optional[torch.Tensor] = None,
                hid_keep: Optional[List[torch.Tensor]] = None, edge_keep: Optional[List[torch.Tensor]] = None,
                bn_eps: float = 1e-5):
    """GAT.forward.  state: the reference module's state_dict (any dtype matching x).  Returns (logits, feat)."""
    n = x.shape[0]
    h = x
    if training and in_keep is not None:
        h = h * in_keep.to(h.dtype) / (1.0 - p_in)                              # :295
    feat = None
    for i in range(n_layers):
        heads = n_heads if i < n_layers - 1 else 1
        h = gat_conv(h, row, col, n, state[f"convs.{i}.fc.weight"], state[f"convs.{i}.attn_l"], state.get(f"convs.{i}.attn_r"),
                     state[f"convs.{i}.res_fc.weight"], heads, use_symmetric_norm,
                     edge_keep[i] if training and edge_keep is not None else None)
        if i < n_layers - 1:
            h = h.flatten(1)                                                    # :303
            g, b = state[f"norms.{i}.weight"], state[f"norms.{i}.bias"]
            if training:
                h = (h - h.mean(0)) / torch.sqrt(h.var(0, unbiased=False) + bn_eps) * g + b
            else:
                h = (h - state[f"norms.{i}.running_mean"]) / torch.sqrt(state[f"norms.{i}.running_var"] + bn_eps) * g + b
            h = torch.relu(h)                                                   # :305
            if training and hid_keep is not None:
                h = h * hid_keep[i].to(h.dtype) / (1.0 - p)                     # :306
            feat = h                                                            # :308
    return h.mean(1) + state["bias_last.bias"], feat                            # :310-311
