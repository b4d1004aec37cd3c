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

``PerGraphGCRD`` is the same objective for engine_ppi's PPI student, whose step trains on one whole graph at a time: the
heads and the objective are GCRD's, the row set is the graph's n nodes.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import criterion, lib, ops
from .heads import SAMPLE_STREAM, HeadRows, ProjectionHeads, _ceil4, _Pool, check_widths  # noqa: F401

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

    def _objective_buffers(self, r, alloc):
        r.norm_s, r.norm_t = alloc(r.S), alloc(r.S)
        r.nce = criterion.NceBuffers(r.Sp, self.P, self.device, alloc=alloc)
        r.loss_aux = r.nce.loss

    def _objective(self, tr, r):
        L, st = lib.load(), lib.stream_ptr()
        S, P = r.S, self.P
        f = lambda t, name: lib.dptr(t, torch.float32, name)
        lib.check(L.b200gnn_gcrd_operands_f32(r.inds.data_ptr(), S, P, f(r.pre_s, "pre_s"), f(self.bn_s, "bn_s"),
                                              f(r.pre_t, "pre_t"), f(self.bn_t, "bn_t"), 1.0 / self.nce_T, _EPS,
                                              f(r.x_s, "x_s"), f(r.x_t, "x_t"), f(r.norm_s, "norm_s"),
                                              f(r.norm_t, "norm_t"), st), "gcrd_operands_f32")
        criterion.nce_chunks(r.x_s, r.x_t, S, r.nce)
        # backward: dz = beta * d loss / d BN output at the sampled rows, zero elsewhere; BatchNorm backward over all rows
        r.dz_s.zero_()
        r.dz_t.zero_()
        lib.check(L.b200gnn_gcrd_backward_f32(r.inds.data_ptr(), S, P, f(r.nce.g_s, "g_s"), f(r.nce.g_t, "g_t"),
                                              f(r.x_s, "x_s"), f(r.x_t, "x_t"), f(r.norm_s, "norm_s"),
                                              f(r.norm_t, "norm_t"), 1.0 / self.nce_T, _EPS, f(r.pre_s, "pre_s"),
                                              f(self.bn_s, "bn_s"), f(r.pre_t, "pre_t"), f(self.bn_t, "bn_t"), self.beta,
                                              f(r.dz_s, "dz_s"), f(r.dz_t, "dz_t"), f(self.bpart_s, "part_s"),
                                              f(self.bpart_t, "part_t"), f(r.loss_aux, "loss_aux"),
                                              f(tr.loss_out, "loss_out"), st), "gcrd_backward_f32")


class PerGraphGCRD(GCRD):
    """G-CRD inside engine_ppi's captured step: the reference's PPI ``train()`` with ``--training nce`` (ppi_pyg/gnn.py:250-259,
    355-372; criterion.py:126-146) projects ``model.out_feat`` and the teacher's out_feat of each training graph, every node
    a row, and contrasts S = min(max_samples, n) of them; its loss is BCE (or kd_criterion) + beta * nce.

    Per graph the teacher rows (padded to a 16-byte pitch), n, S and the sample are kept; every other buffer of the row set
    is a view of one flat buffer sized for the largest graph, at the graph's own geometry (the InfoNCE chunk of
    ``nce_chunk_rows(Sp)`` rows at row pitch Sp, as the eager nce_criterion would take it).  ``PPIGATTrainer.capture``
    records one CUDA graph per training graph with that graph's views.  On graph i the step runs:

        sample       only when S < n: the GCRD sampler at (trainer seed, SAMPLE_STREAM, device step counter)
        heads        out_feat (the trainer's A[L-2][:n], no gather) and the teacher rows through both heads
        objective    GCRD's: operands, InfoNCE chunks, backward
        tail         BatchNorm backward apply, weight gradients, and d out_feat = dz_s . W_s over all n rows, stored into the
                     buffer the last layer's input-gradient GEMM accumulates onto

    The parameters, Adam state, running statistics and state-dict I/O are ProjectionHeads'."""

    def __init__(self, teacher_feat: Sequence[torch.Tensor], hidden: int, proj_dim: int = 256, max_samples: int = 16384,
                 nce_T: float = 0.075, beta: float = 0.1, seed: int = 0, bn_eps: float = 1e-5, bn_momentum: float = 0.1,
                 device="cuda"):
        """teacher_feat: per training graph the teacher's [n_i, F_t] out_feat (``predict(..., return_feat=True)``; F_t =
        1024 for TeacherNet); hidden: the student's out_feat width (136 for StudentNet).  The defaults are the PPI scripts'
        (scripts/run.sh: beta 0.1, nce_T 0.075, max_samples 16384, proj_dim 256)."""
        if len(teacher_feat) == 0:
            raise ValueError("no training graphs")
        for k, t in enumerate(teacher_feat):
            if t.dim() != 2 or t.shape[0] < 1:
                raise ValueError(f"graph {k}: teacher features must be [n, F_t] with n >= 1")
        widths = {int(t.shape[1]) for t in teacher_feat}
        if len(widths) != 1:
            raise ValueError(f"the teacher features have different widths {sorted(widths)}")
        if int(max_samples) < 1:
            raise ValueError("max_samples must be at least 1")
        hidden = int(hidden)
        check_widths(hidden, proj_dim, widths.pop())
        self._init_heads(hidden, proj_dim, int(teacher_feat[0].shape[1]), beta, seed, bn_eps, bn_momentum, torch.device(device))
        self.nce_T = float(nce_T)
        dev, P = self.device, self.P
        sizes = [int(t.shape[0]) for t in teacher_feat]
        samples = [min(int(max_samples), n) for n in sizes]
        G_t = []
        for t in teacher_feat:
            g = torch.zeros(t.shape[0], self.Ft_pad, device=dev)
            g[:, :self.F_t].copy_(t.detach().to(dev, torch.float32))
            G_t.append(g)
        # the operands' padding rows must stay zero: every graph's S rows end at row S_max of one buffer, so the rows after
        # them are written by no graph
        S_max = max(samples)
        flat_s, flat_t = (torch.zeros((S_max + 3) * P, device=dev) for _ in range(2))

        def operands(S):
            o, Sp = (S_max - S) * P, _ceil4(S)
            return flat_s[o:o + Sp * P].view(Sp, P), flat_t[o:o + Sp * P].view(Sp, P)

        pool = _Pool(dev)
        for n, S, g in zip(sizes, samples, G_t):
            HeadRows(self, n, S, g, *operands(S), pool.recorder())
        self.graphs: List[HeadRows] = [HeadRows(self, n, S, g, *operands(S), pool.views())
                                       for n, S, g in zip(sizes, samples, G_t)]
        self.loss_aux = self.graphs[0].loss_aux          # one float that every graph's view shares
        n_draw = max((n for n, S in zip(sizes, samples) if S < n), default=0)
        self.sample_ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n_draw)), dtype=torch.uint8,
                                      device=dev) if n_draw else None)
        self._last = 0

    def check_graphs(self, sizes: Sequence[int], hidden: int):
        """ValueError unless the trainer's training graphs have these node counts and its out_feat this width (called by
        PPIGATTrainer before any device work)."""
        if len(sizes) != len(self.graphs):
            raise ValueError(f"G-CRD built for {len(self.graphs)} training graphs, the trainer has {len(sizes)}")
        if hidden != self.H:
            raise ValueError(f"G-CRD built for hidden width {self.H}, the student's out_feat is {hidden} wide")
        for k, (r, n) in enumerate(zip(self.graphs, sizes)):
            if r.n != n:
                raise ValueError(f"graph {k}: G-CRD built for {r.n} nodes, the trainer's graph has {n}")

    def sample(self) -> torch.Tensor:
        """The last step's sample: positions into the last graph's nodes (int64 [S])."""
        return self.graphs[self._last].inds.to(torch.int64)

    def forward_backward(self, i: int, tr, feat: torch.Tensor, d_feat: torch.Tensor, sample: Optional[torch.Tensor] = None):
        """Graph i's objective: reads out_feat ``feat`` [n_i, H], writes d (beta * loss_aux) / d out_feat into d_feat
        [n_i, H] (all rows), adds beta * loss_aux to tr.loss_out[0]; the value of loss_aux stays in self.loss_aux.  Enqueues
        launches only (capturable) unless ``sample`` (positions into the graph's nodes, [S_i]) replaces the draw."""
        r = self.graphs[i]
        self._last = i
        self._draw(tr, r, sample)
        self._front(r, feat)
        self._objective(tr, r)
        self._tail(r, feat)
        hi, lo = ops.split_tf32(self.W_s, transpose=True, hi=self.WsT_split[0], lo=self.WsT_split[1])
        ops.gemm_tf32x3(r.dz_s, hi, lo, out=d_feat)
