"""fp64 restatement of one reference ``train()`` step with ``--training gpw`` (arxiv_pyg/gnn.py:132-137: CE + beta * gpw;
gnn_kd_and_aux.py:138-148: KD + beta * gpw) with the projection heads of gnn_kd_and_aux.py:275-297 (those of G-CRD,
oracle/gcrd.py) and one Adam over the model and both heads.  The sampled rows are an input (the reference draws them with
np.random.choice, the engine with Philox)."""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import criterion as oc, nn as onn
from .gcrd import _head


def gsp_step(kind: str, x, rowptr, col, val, model: Dict[str, torch.Tensor], sproj: Dict[str, torch.Tensor],
             tproj: Dict[str, torch.Tensor], y, train_idx, t_feat, t_logits: Optional[torch.Tensor], sample, kernel: str,
             beta: float, alpha: float = 0.9, kd_T: float = 4.0, masks=None, p: float = 0.0, lr: float = 0.01,
             bn_eps: float = 1e-5, momentum: float = 0.1, adam_eps: float = 1e-8):
    """Arguments as oracle.gcrd.gcrd_step, with the GSP kernel ('cosine', 'poly', 'l2', 'rbf') in place of nce_T.  Returns
    dict(loss, loss_cls, loss_aux, grads={model, sproj, tproj}, after={model, sproj, tproj}); ``after`` is the state after
    the FIRST Adam step from zero moments."""
    d = lambda sd: {k: v.detach().double().clone().requires_grad_(v.is_floating_point() and "running" not in k)
                    for k, v in sd.items() if "num_batches" not in k}
    m, s, t = d(model), d(sproj), d(tproj)
    L = sum(1 for k in m if k.startswith("convs.") and k.endswith((".weight", ".lin_l.weight")) and "lin_r" not in k)
    ga = [m[f"bns.{i}.weight"] for i in range(L - 1)]
    be = [m[f"bns.{i}.bias"] for i in range(L - 1)]
    if kind == "gcn":
        logits, hid = onn.gcn_forward(x.double(), rowptr, col, val.double(), [m[f"convs.{i}.weight"] for i in range(L)],
                                      [m[f"convs.{i}.bias"] for i in range(L)], ga, be, masks, p=p)
    else:
        params = [dict(w_l=m[f"convs.{i}.lin_l.weight"], b_l=m[f"convs.{i}.lin_l.bias"], w_r=m[f"convs.{i}.lin_r.weight"])
                  for i in range(L)]
        logits, hid = onn.sage_forward(x.double(), rowptr, col, params, ga, be, masks, p=p)
    z, lab = logits[train_idx], y[train_idx]
    if t_logits is None:
        loss_main = loss_cls = oc.cross_entropy(z, lab)
    else:
        loss_main, loss_cls, _ = oc.kd_criterion(z, lab, t_logits[train_idx].double(), alpha, kd_T)
    ps, mu_s, var_s = _head(hid[train_idx], s, bn_eps)
    pt, mu_t, var_t = _head(t_feat[train_idx].double(), t, bn_eps)
    _, _, loss_aux = oc.gpw_criterion(z, lab, ps, pt, kernel, beta, len(sample), sampled_inds=torch.as_tensor(sample))
    loss = loss_main + beta * loss_aux
    groups = {"model": m, "sproj": s, "tproj": t}
    leaves = [(g, k, v) for g, sd in groups.items() for k, v in sd.items() if v.requires_grad]
    gr = torch.autograd.grad(loss, [v for _, _, v in leaves])
    grads = {g: {} for g in groups}
    after = {g: {k: v.detach().clone() for k, v in sd.items()} for g, sd in groups.items()}
    for (g, k, v), dv in zip(leaves, gr):
        grads[g][k] = dv
        after[g][k] = v.detach() - lr * dv / (dv.abs() + adam_eps)                 # Adam step 1: m_hat = g, v_hat = g^2
    # the heads' BatchNorm running statistics (unbiased variance)
    n_rows = train_idx.numel()
    for g, mu, var in (("sproj", mu_s, var_s), ("tproj", mu_t, var_t)):
        a = after[g]
        a["1.running_mean"] = (1 - momentum) * a["1.running_mean"] + momentum * mu.detach()
        a["1.running_var"] = (1 - momentum) * a["1.running_var"] + momentum * var.detach() * n_rows / (n_rows - 1)
    return dict(loss=float(loss.detach()), loss_cls=float(loss_cls.detach()), loss_aux=float(loss_aux.detach()), grads=grads,
                after=after)
