"""fp64 restatement of one reference PPI ``train()`` step with ``--training nce`` (ppi_pyg/gnn.py:250-259, 355-372;
criterion.py:126-146): StudentNet (oracle/ppi.py) on the whole graph, the projection heads of oracle/gcrd.py over its n rows,
InfoNCE over a sample of them and one Adam over the model and both heads.  The sampled rows are an input (the reference
draws them with np.random.choice, the engine with Philox)."""
from __future__ import annotations

from typing import Dict, Tuple

import torch

from . import criterion as oc, gcrd as og_
from .ppi import adjacency, forward, layers_of, loss


def seeded_heads(hidden: int, teacher_width: int, proj_dim: int, seed: int) -> Tuple[Dict[str, torch.Tensor], Dict[str, torch.Tensor]]:
    """(student head, teacher head) state dicts of nn.Sequential(Linear, BatchNorm1d, ReLU) as gcrd.ProjectionHeads'
    ``reset_parameters(seed)`` draws them: nn.Linear's U(+-1/sqrt(fan_in)) for the student's weight and bias, then the
    teacher's, from one CPU generator; BatchNorm1d weight 1, bias 0, running mean 0, running var 1, no batch tracked."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for fan_in in (hidden, teacher_width):
        bound = 1.0 / fan_in ** 0.5
        w = (torch.rand(proj_dim, fan_in, generator=g) * 2 - 1) * bound
        b = (torch.rand(proj_dim, generator=g) * 2 - 1) * bound
        out.append({"0.weight": w, "0.bias": b, "1.weight": torch.ones(proj_dim), "1.bias": torch.zeros(proj_dim),
                    "1.running_mean": torch.zeros(proj_dim), "1.running_var": torch.ones(proj_dim),
                    "1.num_batches_tracked": torch.tensor(0)})
    return out[0], out[1]


def gcrd_step(x, y, edge_index, model: Dict[str, torch.Tensor], sproj: Dict[str, torch.Tensor], tproj: Dict[str, torch.Tensor],
              t_feat, sample=None, beta: float = 0.1, nce_T: float = 0.075, lr: float = 0.005, teacher_logits=None,
              alpha: float = 0.5, T: float = 1.0, bn_eps: float = 1e-5, momentum: float = 0.1, adam_eps: float = 1e-8,
              dtype=torch.float64):
    """One reference PPI ``train()`` step with ``--training nce`` (ppi_pyg/gnn.py:250-259; criterion.py:126-146) restated in
    ``dtype``: StudentNet (``model``, layers from its keys' count) on the whole graph, both projection heads in training
    mode over its n rows, InfoNCE over ``sample`` (positions, None = every row) and one Adam step from zero moments over
    the model and both heads.  Returns dict(loss=[loss, loss_cls, loss_aux], grads={model, sproj, tproj},
    after={model, sproj, tproj}); ``after`` includes the heads' running statistics (unbiased variance)."""
    n = x.shape[0]
    layers = layers_of("student", y.shape[1])
    d = lambda sd: {k: v.to(dtype, copy=True).requires_grad_(True) for k, v in sd.items()  # noqa: E731
                    if "lin_r" not in k and "running" not in k and "num_batches" not in k}
    m, s, t = d(model), d(sproj), d(tproj)
    st = dict(m)
    st.update({k.replace("lin_l", "lin_r"): v for k, v in m.items() if "lin_l" in k})
    row, col = adjacency(edge_index, n)
    logits, feat = forward(x.to(dtype), row, col, st, layers)
    tl = None if teacher_logits is None else teacher_logits.to(dtype)
    loss_main, loss_cls, _ = loss(logits, y.to(dtype), tl, alpha, T)
    ps, mu_s, var_s = og_._head(feat, s, bn_eps)
    pt, mu_t, var_t = og_._head(t_feat.to(dtype), t, bn_eps)
    if sample is not None:
        inds = torch.as_tensor(sample, dtype=torch.long)
        ps, pt = ps[inds], pt[inds]
    z = oc._l2_normalize(ps) @ oc._l2_normalize(pt).t() / nce_T
    loss_aux = -oc._log_softmax(z).diagonal().mean()
    total = loss_main + beta * loss_aux
    groups = {"model": m, "sproj": s, "tproj": t}
    leaves = [(g, k, v) for g, sd in groups.items() for k, v in sd.items()]
    gr = torch.autograd.grad(total, [v for _, _, v in leaves])
    grads = {g: {} for g in groups}
    after = {g: {k: v.detach().clone() for k, v in sd.items()} for g, sd in groups.items()}
    for (g, k, v), dv in zip(leaves, gr):
        grads[g][k] = dv
        after[g][k] = v.detach() - lr * dv / (dv.abs() + adam_eps)                  # Adam step 1: m_hat = g, v_hat = g^2
    for g, src, mu, var in (("sproj", sproj, mu_s, var_s), ("tproj", tproj, mu_t, var_t)):
        after[g]["1.running_mean"] = (1 - momentum) * src["1.running_mean"].to(dtype) + momentum * mu.detach()
        after[g]["1.running_var"] = (1 - momentum) * src["1.running_var"].to(dtype) + momentum * var.detach() * n / (n - 1)
    return dict(loss=torch.stack([total, loss_cls, loss_aux]).detach(), grads=grads, after=after)
