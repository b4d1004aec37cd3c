"""GSP inside the students' captured training step: the projection heads of G-CRD, the row sample and the pairwise-similarity
loss in L2-sized row chunks.

The reference's ``train()`` with ``--training gpw`` (arxiv_pyg/gnn.py:132-137: CE + beta * gpw; gnn_kd_and_aux.py:138-148:
KD + beta * gpw) projects both feature sets through the heads G-CRD uses and compares the pairwise similarities of a row
sample (criterion.py:57-92):

    P_s, P_t, inds          as heads.ProjectionHeads forms them
    cosine: x = normalize(P[inds]), sim = x x^T        poly: sim = (x x^T)^2
    l2:     sim_ij = ||P_i - P_j||                    rbf:  sim_ij = exp(-1/2 ||P_i - P_j||^2)       (P = P[inds])
    loss_aux = mean((sim_s - sim_t)^2) over S x S

``GSP`` is built on heads.ProjectionHeads.  ``GCNStudentTrainer(..., gsp=o)`` / ``SAGEStudentTrainer(..., gsp=o)`` call it
from inside their step, so ``capture()`` / ``replay()`` run it in the same CUDA graph.  Its own part of the step:

    operands     b200gnn_gsp_operands_f32: the S sampled rows of both heads, BN apply, ReLU, then L2 normalisation (cosine /
                 poly) or the squared row norm (l2 / rbf)
    loss         criterion.gsp_chunks, the chunk loop gpw_criterion runs too: two [R, Sp] Gram chunks at a time, never the
                 S x S matrices
    backward     b200gnn_gsp_backward_f32: 2 dG x (+ 4 rc x for l2 / rbf), normalise backward (cosine / poly), ReLU mask,
                 beta, scattered into [n_train, P], pass 1 of the BatchNorm backward

The row sample is G-CRD's (same sampler and Philox stream; a trainer runs one objective); ``train_step(..., sample=)``
injects one.
"""
from __future__ import annotations

import torch

from . import criterion, lib
from .heads import ProjectionHeads

_EPS = 1e-12                                      # F.normalize


class GSP(ProjectionHeads):
    NAME = "GSP"

    def __init__(self, teacher_feat: torch.Tensor, train_idx: torch.Tensor, hidden: int, proj_dim: int = 256,
                 max_samples: int = 8192, kernel: str = "rbf", beta: float = 0.5, seed: int = 0, bn_eps: float = 1e-5,
                 bn_momentum: float = 0.1):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file, F_t = 750); train_idx: the
        training rows, the same tensor the trainer's step receives.  proj_dim a multiple of 32 in (48, 256].  kernel:
        'cosine', 'poly', 'l2' or 'rbf'; the argparse defaults are rbf, beta 0.5, 8192 samples and proj_dim 256, the
        scripts' (run_kd_and_aux.sh) cosine, beta 10, 4096 and 128."""
        if kernel not in criterion._KERNELS:
            raise ValueError(f"kernel {kernel!r}: GSP kernels are {sorted(criterion._KERNELS)}")
        super().__init__(teacher_feat, train_idx, hidden, proj_dim, max_samples, beta, seed, bn_eps, bn_momentum)
        self.kernel, self.kernel_id = kernel, criterion._KERNELS[kernel]

    def _objective_buffers(self, r, alloc):
        r.gsp = criterion.GspBuffers(r.Sp, self.P, self.device)
        # the operands' norms (cosine / poly) or squared norms (l2 / rbf, which the pair pass reads)
        r.norm_s, r.norm_t = r.gsp.ns, r.gsp.nt
        r.loss_aux = r.gsp.loss

    def _objective(self, tr, r):
        L, st = lib.load(), lib.stream_ptr()
        S, P, k, b = r.S, self.P, self.kernel_id, r.gsp
        f = lambda t, name: lib.dptr(t, torch.float32, name)
        lib.check(L.b200gnn_gsp_operands_f32(r.inds.data_ptr(), S, P, k, f(r.pre_s, "pre_s"), f(self.bn_s, "bn_s"),
                                             f(r.pre_t, "pre_t"), f(self.bn_t, "bn_t"), _EPS, f(r.x_s, "x_s"),
                                             f(r.x_t, "x_t"), f(r.norm_s, "norm_s"), f(r.norm_t, "norm_t"), st),
                  "gsp_operands_f32")
        criterion.gsp_chunks(r.x_s, r.x_t, S, k, b)
        # backward: dz = beta * d loss / d BN output at the sampled rows, zero elsewhere; BatchNorm backward over all rows
        r.dz_s.zero_()
        r.dz_t.zero_()
        lib.check(L.b200gnn_gsp_backward_f32(r.inds.data_ptr(), S, P, k, f(b.g_s, "g_s"), f(b.g_t, "g_t"), f(r.x_s, "x_s"),
                                             f(r.x_t, "x_t"), f(r.norm_s, "norm_s"), f(r.norm_t, "norm_t"),
                                             f(b.rc_s, "rc_s"), f(b.rc_t, "rc_t"), _EPS, f(r.pre_s, "pre_s"),
                                             f(self.bn_s, "bn_s"), f(r.pre_t, "pre_t"), f(self.bn_t, "bn_t"), self.beta,
                                             f(r.dz_s, "dz_s"), f(r.dz_t, "dz_t"), f(self.bpart_s, "part_s"),
                                             f(self.bpart_t, "part_t"), f(r.loss_aux, "loss_aux"),
                                             f(tr.loss_out, "loss_out"), st), "gsp_backward_f32")
