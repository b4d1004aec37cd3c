"""The SIGN model (arxiv_dgl/sign.py:105-157) restated functionally on the reference's state_dict keys, CPU PyTorch.

FeedForwardNet (:105-133): Linear -> PReLU -> dropout -> ... -> Linear, one PReLU slope per FFN shared by its hidden
layers, a single Linear for n_layers == 1.  SIGN.forward (:150-157): input dropout on every hop, one FFN per hop,
out_feat = dropout(prelu(cat_h hidden_h)) with the model's own slope, then the project FFN.  Dropout masks are injected
(bool keep-masks) so that the CUDA engine and the oracle share them; masks=None is eval mode.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn.functional as F


def prelu(x, a):
    """nn.PReLU with one slope: x if x > 0 else a * x."""
    return torch.where(x > 0, x, a * x)


def dropout(x, keep: Optional[torch.Tensor], p: float):
    return x if keep is None else x * keep.to(x.dtype) / (1.0 - p)


def feed_forward(x, sd: Dict[str, torch.Tensor], prefix: str, n_layers: int, keeps: Optional[List[torch.Tensor]], p: float):
    """FeedForwardNet.forward (sign.py:128-133); keeps[i]: the mask of the dropout after hidden layer i."""
    for i in range(n_layers):
        x = F.linear(x, sd[f"{prefix}.layers.{i}.weight"], sd[f"{prefix}.layers.{i}.bias"])
        if i < n_layers - 1:
            x = dropout(prelu(x, sd[f"{prefix}.prelu.weight"]), None if keeps is None else keeps[i], p)
    return x


def sign_forward(feats: List[torch.Tensor], sd: Dict[str, torch.Tensor], n_layers: int, masks: Optional[dict] = None,
                 p: float = 0.5, p_in: float = 0.1):
    """SIGN.forward (sign.py:150-157).  masks: dict(input=[hop keep-masks], hidden=[[per hop FFN layer]],
    cat=keep-mask of out_feat, project=[per project FFN layer]) or None (eval).  Returns (logits, out_feat)."""
    hidden = []
    for h, x in enumerate(feats):
        x = dropout(x, None if masks is None else masks["input"][h], p_in)
        hidden.append(feed_forward(x, sd, f"inception_ffs.{h}", n_layers, None if masks is None else masks["hidden"][h], p))
    out_feat = dropout(prelu(torch.cat(hidden, dim=-1), sd["prelu.weight"]), None if masks is None else masks["cat"], p)
    return feed_forward(out_feat, sd, "project", n_layers, None if masks is None else masks["project"], p), out_feat
