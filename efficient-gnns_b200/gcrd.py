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

``BatchGCRD`` is the same objective for rgcn's MAG student on GraphSAINT batches, where the teacher's features and the
number of train rows change with every batch: the row set is built per batch, on the sizes the step already holds.

``SIGNGCRD`` is the same objective for engine_sign's SIGN student: every batch row is a train row, one row set per batch
size, and the student head reads the 3072-wide dropout(prelu(cat)) through the PReLU prologue instead of a stored input.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import criterion, lib, ops
from .heads import (SAMPLE_STREAM, HeadRows, ProjectionHeads, _ceil4, _Pool, check_sample, check_widths,  # noqa: F401
                    draw_sample)

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


class BatchGCRD(GCRD):
    """G-CRD inside rgcn.RGCNTrainer's step: the reference's MAG ``train()`` with ``--training nce``
    (mag_pyg/gnn_kd_and_aux.py:258-271, 424-441) on every GraphSAINT batch b:

        out_feat = student_proj(model.out_feat[b.train_mask])                      Linear(hidden, proj_dim), BN, ReLU
        t_feat   = teacher_proj(teacher_model.out_feat[b.train_mask])              Linear(teacher hidden, proj_dim), BN, ReLU
        loss_aux = nce_criterion(out, labels, out_feat, t_feat, beta, nce_T, max_samples)[2]
        loss     = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux
        one Adam over the model and both heads

    Per batch, between the student's loss and its backward (``RGCNTrainer(..., gcrd=g).train_step(b, x, teacher=t)``):

        rows       a HeadRows for n = n_train rows and S = min(max_samples, n), its buffers from the caching allocator (the
                   step is uncaptured and sized on the host); the sampler's workspace only when S < n
        gather     G_t = the teacher's last hidden layer (eval: ReLU) and G_s = the student's (after ReLU and dropout) at the
                   train rows, row k the k-th train row in batch order (as BatchLSP gathers them)
        step       GCRD's draw (trainer seed, SAMPLE_STREAM, the student's device step counter), head front, objective, tail
        d out_feat dz_s . W_s stored straight into a zeroed internal-order [N, H] gradient at the train rows

    The trainer refuses a batch with one train row before any launch (the reference's BatchNorm1d raises ValueError).  A
    batch with none does what the reference does: loss[0] and loss[2] are NaN, no head kernel runs (bn_finalize would write
    NaN running statistics), the heads' gradients are zero and their Adam step is still taken (num_batches_tracked
    advances), and the model's step is the KD step.  Parameters, Adam state, running statistics and state-dict I/O are
    ProjectionHeads'."""

    def __init__(self, hidden: int, teacher_hidden: int, proj_dim: int = 128, max_samples: int = 24576, nce_T: float = 0.075,
                 beta: float = 0.1, seed: int = 0, bn_eps: float = 1e-5, bn_momentum: float = 0.1, device="cuda"):
        """hidden / teacher_hidden: the student's and the teacher's last hidden widths (32 and 512 in the reference's MAG
        models).  The defaults are the MAG script's (scripts/run_kd_and_aux.sh: beta 0.1, nce_T 0.075, max_samples 24576;
        proj_dim 128 from argparse)."""
        if int(max_samples) < 1:
            raise ValueError("max_samples must be at least 1")
        hidden, teacher_hidden = int(hidden), int(teacher_hidden)
        check_widths(hidden, proj_dim, teacher_hidden)
        self._init_heads(hidden, proj_dim, teacher_hidden, beta, seed, bn_eps, bn_momentum, torch.device(device))
        self.nce_T, self.max_samples = float(nce_T), int(max_samples)
        self.rows: Optional[HeadRows] = None                  # the last batch's row set
        self.loss_aux = torch.full((1,), float("nan"), device=self.device)

    def bind(self, trainer):
        """Called by the RGCNTrainer that owns this object: its last hidden layer must be the width built for."""
        if trainer.L < 2 or trainer.dims[-2] != self.H:
            raise ValueError(f"G-CRD head built for hidden width {self.H}, the student's last hidden layer is "
                             f"{trainer.dims[-2] if trainer.L >= 2 else 'absent'}")

    def check_teacher(self, teacher):
        """ValueError unless the teacher's last hidden layer has the width the teacher head was built for."""
        if teacher.L < 2 or teacher.dims[-2] != self.F_t:
            raise ValueError(f"G-CRD teacher head built for width {self.F_t}, the teacher's last hidden layer is "
                             f"{teacher.dims[-2] if teacher.L >= 2 else 'absent'}")

    def check_batch(self, n: int, sample=None):
        """ValueError for a batch of n train rows the step cannot take (one row: BatchNorm has no variance), or a sample
        that is not S = min(max_samples, n) distinct positions in [0, n)."""
        if n == 1:
            raise ValueError("a batch with one train row: the projection heads' BatchNorm needs more than one value per "
                             "channel in training")
        if sample is not None:
            check_sample(sample, n, min(self.max_samples, n))

    def sample(self) -> torch.Tensor:
        """The last batch's sample: positions into its train rows (int64 [S])."""
        return self.rows.inds.to(torch.int64) if self.rows is not None else torch.zeros(0, dtype=torch.int64)

    def forward_backward(self, tr, teacher, sample: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """After tr's loss on its forward and teacher's eval forward on the same plan: returns d (beta * loss_aux) / d out_feat
        [N, H] in internal row order (None when the batch has no train row) and adds beta * loss_aux to tr.loss_out[0]."""
        f, dev = tr._fwd, self.device
        train_int = f["train_int"]
        n = train_int.numel()
        if n == 0:
            self.rows = None
            self.grads.zero_()
            self.loss_aux = torch.full((1,), float("nan"), device=dev)
            tr.loss_out[:1].add_(self.loss_aux * self.beta)
            return None
        S, P = min(self.max_samples, n), self.P
        feat_t = teacher._fwd["xs"][-1]
        G_t = ops.gather_rows_act(feat_t, train_int, torch.empty(n, feat_t.shape[1], device=dev))
        r = HeadRows(self, n, S, G_t, torch.zeros(_ceil4(S), P, device=dev), torch.zeros(_ceil4(S), P, device=dev),
                     lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev))
        self.rows, self.loss_aux = r, r.loss_aux
        self.sample_ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n)), dtype=torch.uint8, device=dev)
                          if S < n else None)
        self._draw(tr, r, sample)
        G_s = ops.gather_rows_act(f["xs"][-1], train_int, torch.empty(n, self.H, device=dev))
        self._front(r, G_s)
        self._objective(tr, r)
        self._tail(r, G_s)
        d_feat = torch.zeros(f["P"].N, self.H, device=dev)
        hi, lo = ops.split_tf32(self.W_s, transpose=True, hi=self.WsT_split[0], lo=self.WsT_split[1])
        ops.gemm_tf32x3_rowidx(r.dz_s, hi, lo, d_feat, train_int)
        return d_feat


class SIGNGCRD(GCRD):
    """G-CRD inside engine_sign.SIGNStudentTrainer's captured step: the reference's ``train_kd_and_aux`` with
    ``--training nce`` (arxiv_dgl/sign.py:355-367, heads :421-438) on every batch of B training nodes:

        out_feat = student_proj(model.out_feat)          Linear(hops * hidden, proj_dim), BatchNorm1d, ReLU over all B rows
        t_feat   = teacher_proj(teacher_out_feat[batch])  Linear(750, proj_dim), BatchNorm1d, ReLU
        loss_aux = nce_criterion(logits, labels, out_feat, t_feat, beta, nce_T, max_samples)[2]
        loss     = kd_criterion(logits, labels, teacher_logits, alpha, kd_T)[0] + beta * loss_aux
        one Adam over the model and both heads

    model.out_feat = dropout(prelu(cat)) is [B, hops * hidden] ([50000, 3072] at the script's settings) and is never
    stored: the student head's Linear forms it in the A-operand prologue of ``gemm_tf32x3_prelu_stats`` from the
    concatenation, the model slope and the keep bits, with the BatchNorm statistics in the epilogue; its weight gradient
    is ``gemm_wgrad_tf32x3_prelu`` on the same three, transposed into gW_s.  Per step, between the trainer's loss and its
    backward:

        rows       the HeadRows of batch size B (S = min(max_samples, B)); row sets of the sizes ``prepare`` is given
                   together are views of one _Pool (one graph per batch size, never two at once)
        sample     only when S < B: the GCRD sampler at (trainer seed, SAMPLE_STREAM, the trainer's device step counter)
        teacher    G_t = the zero-padded teacher features at the batch's node indices (one gather launch)
        heads      the student front above, the teacher front, GCRD's objective, the BatchNorm backward, both weight
                   gradients
        d cat      dz_s . W_s stored straight into the trainer's dZcat over all B rows (every row is a train row); the
                   project FFN's first input-gradient GEMM then accumulates onto it

    Parameters, Adam state, running statistics and state-dict I/O are ProjectionHeads'."""

    def __init__(self, teacher_feat: torch.Tensor, hidden: int, proj_dim: int = 256, max_samples: int = 16384,
                 nce_T: float = 0.075, beta: float = 0.1, seed: int = 0, bn_eps: float = 1e-5, bn_momentum: float = 0.1):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file, F_t = 750); hidden: the
        student head's input width, hops * hidden of the SIGN model (3072 at the script's R = 5, num_hidden = 512).  The
        defaults are the SIGN script's (scripts/run_all_kd_and_aux.sh: beta 0.1, nce_T 0.075, max_samples 16384,
        proj_dim 256)."""
        if not isinstance(teacher_feat, torch.Tensor) or teacher_feat.dim() != 2 or teacher_feat.shape[0] < 1:
            raise ValueError("teacher features must be an [N, F_t] tensor")
        hidden = int(hidden)
        if int(max_samples) < 1:
            raise ValueError("max_samples must be at least 1")
        if not ops.gemm_stats_supported(proj_dim):
            raise ValueError("proj_dim must be a multiple of 32 in (48, 256]")
        if hidden % 32 or hidden <= 0:
            raise ValueError("the student head's width (hops * hidden) must be a positive multiple of 32")
        if not 0 < _ceil4(teacher_feat.shape[1]) <= 2048:
            raise ValueError("teacher feature width must be at most 2048 (the teacher head's weight-gradient GEMM)")
        self._init_heads(hidden, proj_dim, int(teacher_feat.shape[1]), beta, seed, bn_eps, bn_momentum, teacher_feat.device)
        self.nce_T, self.max_samples = float(nce_T), int(max_samples)
        self.N = int(teacher_feat.shape[0])
        # every row's teacher features at a 16-byte pitch; the padding columns must be zeros (W_t's zero columns do not
        # cancel a NaN)
        self.t_feat = torch.zeros(self.N, self.Ft_pad, device=self.device)
        self.t_feat[:, :self.F_t].copy_(teacher_feat.detach().to(torch.float32))
        H, P = self.H, self.P
        # the student head's weight gradient [H, P], column blocks of WGRAD_PRELU_BLOCK when H > 2048, then transposed
        self.gWs_T = torch.empty(H, P, device=self.device)
        self.wgrad_ws_s = torch.empty(ops.wgrad_workspace_floats(H if H <= 2048 else ops.WGRAD_PRELU_BLOCK, P),
                                      device=self.device)
        self.row_sets = {}                                  # batch size -> HeadRows
        self._pools = []                                  # keeps every pool's buffers alive (captured graphs read them)
        self._last: Optional[HeadRows] = None

    def prepare(self, batch_sizes: Sequence[int]):
        """Build the row sets of these batch sizes (those not built yet) on one _Pool: one buffer per request, sized for the
        largest; the operands' padding rows stay zero (every size's S rows end at row S_max of one zeroed buffer)."""
        new = sorted({int(b) for b in batch_sizes} - set(self.row_sets))
        if not new:
            return
        dev, P, Ftp = self.device, self.P, self.Ft_pad
        samples = [min(self.max_samples, B) for B in new]
        S_max = max(samples)
        flat_s, flat_t = (torch.zeros((S_max + 3) * P, device=dev) for _ in range(2))

        def operands(S):
            o, Sp = (S_max - S) * P, _ceil4(S)
            return flat_s[o:o + Sp * P].view(Sp, P), flat_t[o:o + Sp * P].view(Sp, P)

        def build(B, S, alloc):
            G_t = alloc(B, Ftp)
            return HeadRows(self, B, S, G_t, *operands(S), alloc)

        pool = _Pool(dev)
        for B, S in zip(new, samples):
            build(B, S, pool.recorder())
        n_draw = max((B for B, S in zip(new, samples) if S < B), default=0)
        ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n_draw)), dtype=torch.uint8, device=dev)
              if n_draw else None)
        for B, S in zip(new, samples):
            r = build(B, S, pool.views())
            r.sample_ws = ws
            self.row_sets[B] = r
        self._pools.append((pool, flat_s, flat_t, ws))

    def check_batch(self, B: int, sample=None):
        """ValueError for a batch the step cannot take (one row: BatchNorm has no variance, as the reference's BatchNorm1d
        raises), or a sample that is not S = min(max_samples, B) distinct positions in [0, B)."""
        if B == 1:
            raise ValueError("a batch of one row: the projection heads' BatchNorm needs more than one value per channel "
                             "in training")
        if sample is not None:
            check_sample(sample, B, min(self.max_samples, B))

    @property
    def loss_aux(self) -> torch.Tensor:
        return self._last.loss_aux if self._last is not None else torch.full((1,), float("nan"), device=self.device)

    def sample(self) -> torch.Tensor:
        """The last step's sample: positions into its batch (int64 [S])."""
        return self._last.inds.to(torch.int64)

    def _draw(self, tr, r: HeadRows, sample: Optional[torch.Tensor]):
        draw_sample(tr, r.n, r.S, r.perm, r.sample_ws, sample)

    def _front_student(self, r: HeadRows, src):
        Z, slope, bits, p = src
        hi, lo = ops.split_tf32(self.W_s, hi=self.Ws_split[0], lo=self.Ws_split[1])
        ops.gemm_tf32x3_prelu_stats(Z, slope, bits, p, hi, lo, self.b_s, r.pre_s, r.gp_s)
        ops.bn_finalize(r.gp_s, r.n, self.gamma_s, self.beta_s, self.bn_eps, self.bn_momentum, self.rm_s, self.rv_s,
                        out=self.bn_s)

    def _wgrad_student(self, r: HeadRows, src):
        Z, slope, bits, p = src
        ops.gemm_wgrad_tf32x3_prelu(Z, slope, bits, p, r.dz_s, out=self.gWs_T, workspace=self.wgrad_ws_s)
        lib.check(lib.load().b200gnn_transpose_f32(lib.dptr(self.gWs_T, torch.float32, "gWs_T"), self.H, self.P,
                                                   lib.dptr(self.gW_s, torch.float32, "gW_s"), lib.stream_ptr()),
                  "transpose_f32")

    def forward_backward(self, tr, idx: torch.Tensor, zcat: torch.Tensor, slope: torch.Tensor, bits: torch.Tensor, p: float,
                         d_zcat: torch.Tensor, sample: Optional[torch.Tensor] = None):
        """The objective of the batch ``idx`` (int64 [B] node indices; its row set must have been prepared): reads
        out_feat = dropout(prelu(zcat)) through (zcat [B, H], slope, bits [B, H/32], p), STORES d (beta * loss_aux) /
        d out_feat into d_zcat [B, H] and adds beta * loss_aux to tr.loss_out[0].  Enqueues launches only (capturable)
        unless ``sample`` (positions into the batch, [S]) replaces the draw."""
        B = idx.numel()
        r = self.row_sets[B]
        self._last = r
        self._draw(tr, r, sample)
        ops.gather_rows_act(self.t_feat, idx, r.G_t)
        src = (zcat, slope, bits, p)
        self._front(r, src)
        self._objective(tr, r)
        self._tail(r, src)
        hi, lo = ops.split_tf32(self.W_s, transpose=True, hi=self.WsT_split[0], lo=self.WsT_split[1])
        ops.gemm_tf32x3(r.dz_s, hi, lo, out=d_zcat)
