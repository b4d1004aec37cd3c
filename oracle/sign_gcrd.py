"""One step of the reference's SIGN ``train_kd_and_aux`` with ``--training nce`` (arxiv_dgl/sign.py:355-373, heads
:421-438), restated in float64 on the CPU:

    logits   = model(batch_feats)                                      train mode, dropout keep masks injected
    P_s      = student_proj(model.out_feat)                            Linear(hops * hidden, proj_dim), BatchNorm1d, ReLU
    P_t      = teacher_proj(teacher_out_feat[batch])                   Linear(750, proj_dim), BatchNorm1d, ReLU
    loss_aux = nce_criterion(logits, labels, P_s, P_t, beta, nce_T, max_samples)[2]      InfoNCE over S sampled rows
    loss     = kd_criterion(logits, labels, teacher_logits[batch], alpha, kd_T)[0] + beta * loss_aux
    one Adam over the model and both heads

The SIGN forward is oracle/sign.py's, the heads oracle/gcrd.py's, the InfoNCE and KD terms oracle/criterion.py's and Adam
oracle/mag_lsp.py's.  The sampled rows are an input (the reference draws them with np.random.choice, the engine with
Philox); every batch row is a row of the heads' BatchNorm.
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from . import criterion as oc, dropout as od
from .gcrd import _head
from .mag_gcrd import running_stats
from .mag_lsp import adam
from .sign import sign_forward

HEAD_KEYS = ("0.weight", "0.bias", "1.weight", "1.bias")


def engine_masks(H: int, F: int, hidden: int, ff: int, B: int, p: float, p_in: float, seed: int, step: int):
    """The keep masks SIGNStudentTrainer(seed=seed) draws at training step ``step`` for a batch of B rows, in
    oracle.sign.sign_forward's form (oracle.dropout's CPU restatement at oracle.dropout.sign_streams' offsets)."""
    s = od.sign_streams(H, ff, step)
    m = lambda rows, K, q, off: torch.from_numpy(od.mask(rows, K, q, seed, off))  # noqa: E731
    return dict(input=[m(B, F, p_in, s[f"hop{h}"]) for h in range(H)],
                hidden=[[m(B, hidden, p, s[f"hidden{h * (ff - 1) + i}"]) for i in range(ff - 1)] for h in range(H)],
                project=[m(B, hidden, p, s[f"hidden{H * (ff - 1) + i}"]) for i in range(ff - 1)],
                cat=m(B * H, hidden, p, s["cat"]).view(B, H * hidden))


def nce_step_loss(model: Dict[str, torch.Tensor], sproj: Dict[str, torch.Tensor], tproj: Dict[str, torch.Tensor], feats_b,
                  y_b, t_logits_b, t_feat_b, masks, sample: Optional[torch.Tensor], n_layers: int, beta: float, nce_T: float,
                  p: float = 0.5, p_in: float = 0.1, alpha: float = 0.9, kd_T: float = 4.0, bn_eps: float = 1e-5):
    """(loss, loss_cls, loss_aux, stats) of one step on a batch: feats_b the hop features of its rows, y_b / t_logits_b /
    t_feat_b its labels, teacher logits and teacher features; masks as oracle.sign.sign_forward takes them.  ``model`` and
    the heads' HEAD_KEYS hold leaf tensors, so loss.backward() gives the gradients; ``sample``: positions into the batch
    (None = every row); stats: {"sproj": (batch mean, biased var), "tproj": ...} for ``running_stats``."""
    logits, out_feat = sign_forward(feats_b, model, n_layers, masks, p, p_in)
    loss, loss_cls, _ = oc.kd_criterion(logits, y_b, t_logits_b, alpha, kd_T)
    ps, mu_s, var_s = _head(out_feat, sproj, bn_eps)
    pt, mu_t, var_t = _head(t_feat_b, tproj, bn_eps)
    S = ps.shape[0] if sample is None else len(sample)
    inds = None if sample is None else torch.as_tensor(sample, dtype=torch.long)
    _, _, loss_aux = oc.nce_criterion(logits, y_b, ps, pt, beta, nce_T, S, sampled_inds=inds)
    return loss + beta * loss_aux, loss_cls, loss_aux, {"sproj": (mu_s, var_s), "tproj": (mu_t, var_t)}


class Run:
    """Consecutive steps from one state: the model and both heads (state dicts under the reference's keys, copied to
    float64), one Adam over all three from zero moments, and the heads' running statistics."""

    def __init__(self, model: Dict[str, torch.Tensor], sproj: Dict[str, torch.Tensor], tproj: Dict[str, torch.Tensor],
                 lr: float):
        leaf = lambda sd: {k: v.detach().double().clone().requires_grad_(True) for k, v in sd.items()}  # noqa: E731
        self.groups = {"model": leaf(model), "sproj": leaf({k: sproj[k] for k in HEAD_KEYS}),
                       "tproj": leaf({k: tproj[k] for k in HEAD_KEYS})}
        self.running = {g: {k: v.double().clone() for k, v in sd.items() if "running" in k}
                        for g, sd in (("sproj", sproj), ("tproj", tproj))}
        self.params = {f"{g}/{k}": v for g, sd in self.groups.items() for k, v in sd.items()}
        self.m = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.v = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.lr, self.steps = float(lr), 0

    def step(self, feats_b, y_b, t_logits_b, t_feat_b, masks, sample, n_layers: int, beta: float, nce_T: float, **kw):
        """One step: returns (losses [3], grads {model, sproj, tproj}); the parameters, moments and running statistics
        advance."""
        for v in self.params.values():
            v.grad = None
        g = self.groups
        loss, cls, aux, stats = nce_step_loss(g["model"], g["sproj"], g["tproj"], [f.double() for f in feats_b], y_b,
                                              t_logits_b.double(), t_feat_b.double(), masks, sample, n_layers, beta, nce_T,
                                              **kw)
        loss.backward()
        grads = {n: {k: v.grad.detach().clone() for k, v in sd.items()} for n, sd in g.items()}
        self.steps += 1
        adam(self.params, self.m, self.v, self.steps, self.lr)
        for n in self.running:
            running_stats(self.running[n], stats[n], y_b.numel())
        return torch.stack([loss, cls, aux]).detach(), grads

    def state(self, group: str) -> Dict[str, torch.Tensor]:
        return {k: v.detach() for k, v in self.groups[group].items()}
