"""G-CRD inside the students' captured training step: the projection heads, the on-device row sample and the InfoNCE loss.

The reference's ``train()`` with ``--training nce`` (arxiv_pyg/gnn.py:153-159: CE + beta * nce; gnn_kd_and_aux.py:160-170:
KD + beta * nce) projects both feature sets through a head of its own (gnn.py:296-306) and contrasts a sample of rows
(criterion.py:129-149):

    P_s  = relu(BN_s(Linear_s(model.out_feat[train_idx])))          Linear_s: hidden -> proj_dim
    P_t  = relu(BN_t(Linear_t(teacher_out_feat[train_idx])))        Linear_t: 750 -> proj_dim (trained too)
    inds = S = min(max_samples, n_train) distinct rows of [0, n_train)
    loss_aux = CE(normalize(P_s[inds]) . normalize(P_t[inds])^T / nce_T, arange)
    one Adam over the model and both heads

``GCRD`` is built on heads.ProjectionHeads, which owns both heads, the sample and the head front and tail of the step.
``GCNStudentTrainer(..., gcrd=g)`` / ``SAGEStudentTrainer(..., gcrd=g)`` call it from inside their step, so ``capture()`` /
``replay()`` run the whole of it as one CUDA graph with no host read.  Its own part of the step:

    operands     the S sampled rows of both heads: BN apply, ReLU, L2 normalisation, 1/nce_T on the student
    InfoNCE      criterion.nce_chunks, the chunk loop nce_criterion runs too, on preallocated buffers
    backward     normalise backward, ReLU mask, beta, scattered into [n_train, P], pass 1 of the BatchNorm backward

The sample cannot equal numpy's ``np.random.choice`` draw; ``train_step(..., sample=)`` injects one (tests).
"""
from __future__ import annotations

import torch

from . import criterion, lib
from .heads import SAMPLE_STREAM, ProjectionHeads  # noqa: F401  (SAMPLE_STREAM: the sampler's Philox stream)

_EPS = 1e-12                                      # F.normalize


class GCRD(ProjectionHeads):
    NAME = "G-CRD"

    def __init__(self, teacher_feat: torch.Tensor, train_idx: torch.Tensor, hidden: int, proj_dim: int = 256,
                 max_samples: int = 8192, nce_T: float = 0.075, beta: float = 0.5, seed: int = 0, bn_eps: float = 1e-5,
                 bn_momentum: float = 0.1):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file, F_t = 750); train_idx: the
        training rows, the same tensor the trainer's step receives.  proj_dim a multiple of 32 in (48, 256]."""
        super().__init__(teacher_feat, train_idx, hidden, proj_dim, max_samples, beta, seed, bn_eps, bn_momentum)
        self.nce_T = float(nce_T)
        self.norm_s = torch.empty(self.S, dtype=torch.float32, device=self.device)
        self.norm_t = torch.empty(self.S, dtype=torch.float32, device=self.device)
        self.nce = criterion.NceBuffers(self.Sp, self.P, self.device)
        self.loss_aux = self.nce.loss

    def _objective(self, tr):
        L, st = lib.load(), lib.stream_ptr()
        S, P = self.S, self.P
        f = lambda t, name: lib.dptr(t, torch.float32, name)
        lib.check(L.b200gnn_gcrd_operands_f32(self.inds.data_ptr(), S, P, f(self.pre_s, "pre_s"), f(self.bn_s, "bn_s"),
                                              f(self.pre_t, "pre_t"), f(self.bn_t, "bn_t"), 1.0 / self.nce_T, _EPS,
                                              f(self.x_s, "x_s"), f(self.x_t, "x_t"), f(self.norm_s, "norm_s"),
                                              f(self.norm_t, "norm_t"), st), "gcrd_operands_f32")
        criterion.nce_chunks(self.x_s, self.x_t, S, self.nce)
        # backward: dz = beta * d loss / d BN output at the sampled rows, zero elsewhere; BatchNorm backward over all rows
        self.dz_s.zero_()
        self.dz_t.zero_()
        lib.check(L.b200gnn_gcrd_backward_f32(self.inds.data_ptr(), S, P, f(self.nce.g_s, "g_s"), f(self.nce.g_t, "g_t"),
                                              f(self.x_s, "x_s"), f(self.x_t, "x_t"), f(self.norm_s, "norm_s"),
                                              f(self.norm_t, "norm_t"), 1.0 / self.nce_T, _EPS, f(self.pre_s, "pre_s"),
                                              f(self.bn_s, "bn_s"), f(self.pre_t, "pre_t"), f(self.bn_t, "bn_t"), self.beta,
                                              f(self.dz_s, "dz_s"), f(self.dz_t, "dz_t"), f(self.bpart_s, "part_s"),
                                              f(self.bpart_t, "part_t"), f(self.loss_aux, "loss_aux"),
                                              f(tr.loss_out, "loss_out"), st), "gcrd_backward_f32")
