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

``PerGraphGSP`` is GSP for engine_ppi's PPI student, which has no heads: the loss compares the student's out_feat with the
frozen teacher's, so each graph's teacher similarities are constants built once.

``BatchGSP`` is GSP for rgcn.RGCNTrainer's MAG student on GraphSAINT batches, also without heads: per batch the teacher's
last hidden layer comes from its eval forward on the student's plan, and the student's narrow gradient dG . x runs on the
column-split contraction b200gnn_gsp_contract_narrow_f32 instead of the GEMM.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

from . import criterion, lib, ops
from .heads import ProjectionHeads, _ceil4, _Pool, check_sample, draw_sample

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


class _GraphGSP:
    """One training graph's share of PerGraphGSP: n, S = min(max_samples, n), Sp, its sample, its teacher similarities
    sim_t [n, n] (a view of the object's flat allocation) and its views of the per-step buffers, at the geometry the eager
    gpw_criterion gives S rows: operands [Sp, H], Gram chunks of gsp_chunk_rows(Sp) rows at pitch Sp."""

    def __init__(self, n: int, S: int, sim_t: torch.Tensor, x_s: torch.Tensor, H: int, device, alloc):
        self.n, self.S, self.Sp, self.sim_t, self.x_s = n, S, _ceil4(S), sim_t, x_s
        Sp = self.Sp
        self.perm = torch.arange(n, dtype=torch.int32, device=device)
        self.inds = self.perm[:S]
        self.G = alloc(criterion.gsp_chunk_rows(Sp), Sp)
        self.split, self.splitT = (alloc(Sp, H), alloc(Sp, H)), (alloc(H, Sp), alloc(H, Sp))
        self.g = alloc(Sp, H)                                   # dG . x
        self.norm, self.rc, self.part = alloc(Sp), alloc(Sp), alloc(Sp)
        self.loss_aux = alloc(1)


class PerGraphGSP:
    """GSP inside engine_ppi's captured step: the reference's PPI ``train()`` with ``--training gpw`` (ppi_pyg/gnn.py:230-239;
    criterion.py:54-89) applies ``gpw_criterion(out, labels, model.out_feat, teacher_model.out_feat, kernel, beta,
    max_samples)`` to each training graph, every node a row and no projection heads: BCE (or kd_criterion) + beta * mean((sim_s
    - sim_t)^2) over S = min(max_samples, n) rows.

    The teacher runs in eval mode with frozen parameters, so each graph's teacher similarity matrix is a constant: it is
    built once, at construction, with the eager path's kernels and shapes (normalise or squared norms, the 3xTF32 Gram at
    pitch Sp and K = F_t in row chunks, b200gnn_gsp_sim_chunk_f32), and kept as an [n, n] view of one flat allocation
    (``sim_bytes`` in all).  A GEMM row does not depend on the M tiling and these GEMMs have no split-K, so sim_t equals the
    teacher similarities the eager path forms, and the step never touches the 1024-wide teacher features again.  On graph
    i the step runs, as launches only (capturable):

        sample       only when S < n: G-CRD's sampler at (trainer seed, SAMPLE_STREAM, device step counter)
        operands     b200gnn_gsp_rows_operands_f32: the S rows of out_feat normalised (cosine / poly) or copied with their
                     squared norms (l2 / rbf), zero-padded to [Sp, H]
        loss         the student side of criterion.gsp_chunks: both splits of the operands, then per chunk the Gram GEMM,
                     b200gnn_gsp_pair_fixed_chunk_f32 against sim_t, and dG . x; b200gnn_gsp_finish_f32
        backward     b200gnn_gsp_rows_backward_f32: beta * d loss / d out_feat stored straight into the buffer the last
                     layer's input-gradient GEMM accumulates onto (zero-filled first when S < n), loss[0] += beta * loss

    Every float equals the eager ``train_step(i, aux=lambda f: criterion_ppi.gpw_criterion(..., f, teacher_feat[i], kernel,
    1, max_samples, sampled_inds=...)[2], beta)``.  The per-step buffers are sized for the largest graph and viewed at each
    graph's own geometry, as gcrd.PerGraphGCRD's."""

    NAME = "GSP"

    def __init__(self, teacher_feat: Sequence[torch.Tensor], hidden: int, kernel: str = "rbf", beta: float = 100.0,
                 max_samples: int = 8192, device="cuda"):
        """teacher_feat: per training graph the teacher's [n_i, F_t] out_feat (``predict(..., return_feat=True)``; F_t = 1024
        for TeacherNet); hidden: the student's out_feat width (136 for StudentNet), a multiple of 4 up to
        lib.GSP_ROWS_MAX_F.  kernel 'cosine', 'poly', 'l2' or 'rbf' and max_samples 8192 are the argparse defaults of
        ppi_pyg/gnn.py (8192 is above every PPI graph, so S = n).  The argparse beta default is 0, which switches the term
        off, and scripts/run.sh has no gpw line; the PPI README tunes beta in {100, 1000, 10000}, so the default here is
        100."""
        if kernel not in criterion._KERNELS:
            raise ValueError(f"kernel {kernel!r}: GSP kernels are {sorted(criterion._KERNELS)}")
        if int(max_samples) < 1:
            raise ValueError("max_samples must be at least 1")
        if len(teacher_feat) == 0:
            raise ValueError("no training graphs")
        for k, t in enumerate(teacher_feat):
            if t.dim() != 2 or t.shape[0] < 1 or t.shape[1] < 1:
                raise ValueError(f"graph {k}: teacher features must be [n, F_t] with n, F_t >= 1")
        widths = {int(t.shape[1]) for t in teacher_feat}
        if len(widths) != 1:
            raise ValueError(f"the teacher features have different widths {sorted(widths)}")
        hidden = int(hidden)
        if hidden % 4 or not 0 < hidden <= lib.GSP_ROWS_MAX_F:
            raise ValueError(f"hidden width {hidden}: the GSP row passes take a multiple of 4 up to {lib.GSP_ROWS_MAX_F}")
        self.device = dev = torch.device(device)
        self.H, self.F_t, self.beta = hidden, widths.pop(), float(beta)
        self.kernel, self.kernel_id = kernel, criterion._KERNELS[kernel]
        sizes = [int(t.shape[0]) for t in teacher_feat]
        samples = [min(int(max_samples), n) for n in sizes]

        # the teacher similarities: one flat allocation, an [n, n] view per graph
        offsets = [0]
        for n in sizes:
            offsets.append(offsets[-1] + n * n)
        self.sim_flat = torch.empty(offsets[-1], dtype=torch.float32, device=dev)
        self.sim_bytes = self.sim_flat.numel() * 4
        sims = [self.sim_flat[o:o + n * n].view(n, n) for o, n in zip(offsets, sizes)]
        for t, sim in zip(teacher_feat, sims):
            self._build_sim(t.detach().to(dev, torch.float32).contiguous(), sim)

        # the operands' padding rows must stay zero: every graph's S rows end at row S_max of one buffer, so the rows after
        # them are written by no graph
        H, S_max = self.H, max(samples)
        flat_x = torch.zeros((S_max + 3) * H, device=dev)

        def operands(S):
            o = (S_max - S) * H
            return flat_x[o:o + _ceil4(S) * H].view(_ceil4(S), H)

        pool = _Pool(dev)
        for n, S, sim in zip(sizes, samples, sims):
            _GraphGSP(n, S, sim, operands(S), H, dev, pool.recorder())
        self.graphs: List[_GraphGSP] = [_GraphGSP(n, S, sim, operands(S), H, dev, pool.views())
                                        for n, S, sim in zip(sizes, samples, sims)]
        self.loss_aux = self.graphs[0].loss_aux          # one float that every graph's view shares
        n_draw = max((n for n, S in zip(sizes, samples) if S < n), default=0)
        self.sample_ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n_draw)), dtype=torch.uint8,
                                      device=dev) if n_draw else None)
        self._last = 0

    def _build_sim(self, t: torch.Tensor, sim: torch.Tensor):
        """sim [n, n] = the teacher similarities of all n rows of t, as gpw_criterion's chunk loop forms them with S = n."""
        L, st = lib.load(), lib.stream_ptr()
        n, k = t.shape[0], self.kernel_id
        if k <= 1:
            x, _ = criterion._normalize(t)
            sq = None
        else:
            x, sq = t, torch.empty(n, dtype=torch.float32, device=t.device)
            lib.check(L.b200gnn_row_sqnorm_f32(lib.dptr(x, torch.float32, "x"), n, x.shape[1], lib.dptr(sq, torch.float32, "sq"),
                                               st), "row_sqnorm_f32")
        x = criterion._pad_k(criterion._pad_k(x, 1), 0)                 # [Sp, F_t padded], as the eager operand
        Sp = x.shape[0]
        hi, lo = ops.split_tf32(x)
        R = criterion.gsp_chunk_rows(Sp)
        G = torch.empty(R, Sp, dtype=torch.float32, device=t.device)
        for r0 in range(0, n, R):
            r = min(R, n - r0)
            ops.gemm_tf32x3(x[r0:r0 + r], hi, lo, out=G[:r])
            lib.check(L.b200gnn_gsp_sim_chunk_f32(lib.dptr(G, torch.float32, "G"), Sp, r, n, r0,
                                                  lib.dptr(sq, torch.float32, "sq"), k, lib.dptr(sim[r0], torch.float32, "sim"),
                                                  n, st), "gsp_sim_chunk_f32")

    def check_graphs(self, sizes: Sequence[int], hidden: int):
        """ValueError unless the trainer's training graphs have these node counts and its out_feat this width (called by
        PPIGATTrainer before any device work)."""
        if len(sizes) != len(self.graphs):
            raise ValueError(f"GSP built for {len(self.graphs)} training graphs, the trainer has {len(sizes)}")
        if hidden != self.H:
            raise ValueError(f"GSP built for hidden width {self.H}, the student's out_feat is {hidden} wide")
        for k, (r, n) in enumerate(zip(self.graphs, sizes)):
            if r.n != n:
                raise ValueError(f"graph {k}: GSP built for {r.n} nodes, the trainer's graph has {n}")

    def sample(self) -> torch.Tensor:
        """The last step's sample: positions into the last graph's nodes (int64 [S])."""
        return self.graphs[self._last].inds.to(torch.int64)

    def check_sample(self, i: int, sample: torch.Tensor):
        """ValueError unless ``sample`` is S_i distinct positions of graph i's nodes with S_i < n_i (PPIGATTrainer calls it
        before the step launches anything)."""
        r = self.graphs[i]
        if r.S == r.n:
            raise ValueError(f"GSP takes every row of graph {i} (max_samples >= {r.n}): there is no sample to inject")
        s = torch.as_tensor(sample).to("cpu", torch.int64).view(-1)
        if s.numel() != r.S or int(s.min()) < 0 or int(s.max()) >= r.n or s.unique().numel() != r.S:
            raise ValueError(f"sample must hold {r.S} distinct positions in [0, {r.n})")

    def forward_backward(self, i: int, tr, feat: torch.Tensor, d_feat: torch.Tensor, sample: Optional[torch.Tensor] = None):
        """Graph i's objective: reads out_feat ``feat`` [n_i, H], writes d (beta * loss_aux) / d out_feat into d_feat
        [n_i, H] (all rows; zero outside the sample), adds beta * loss_aux to tr.loss_out[0]; the value of loss_aux stays in
        self.loss_aux.  Enqueues launches only (capturable) unless ``sample`` (positions into the graph's nodes, [S_i],
        S_i < n_i) replaces the draw."""
        r = self.graphs[i]
        self._last = i
        n, S, Sp, H, k = r.n, r.S, r.Sp, self.H, self.kernel_id
        if sample is not None:
            self.check_sample(i, sample)
        draw_sample(tr, n, S, r.perm, self.sample_ws, sample)
        L, st = lib.load(), lib.stream_ptr()
        f = lambda t, name: lib.dptr(t, torch.float32, name)      # noqa: E731
        inds = r.inds.data_ptr() if S < n else None
        raw = k >= 2
        lib.check(L.b200gnn_gsp_rows_operands_f32(f(feat, "feat"), feat.stride(0), inds, S, H, k, _EPS, f(r.x_s, "x_s"), H,
                                                  f(r.norm, "norm"), st), "gsp_rows_operands_f32")
        hi, lo = ops.split_tf32(r.x_s, hi=r.split[0], lo=r.split[1])
        hiT, loT = ops.split_tf32(r.x_s, transpose=True, hi=r.splitT[0], lo=r.splitT[1])
        R = r.G.shape[0]
        for r0 in range(0, S, R):
            m = min(R, S - r0)
            ops.gemm_tf32x3(r.x_s[r0:r0 + m], hi, lo, out=r.G[:m])
            lib.check(L.b200gnn_gsp_pair_fixed_chunk_f32(f(r.G, "G"), Sp, m, S, r0, f(r.norm if raw else None, "ns"),
                                                         f(r.sim_t, "sim_t"), n, n, inds, k, f(r.rc if raw else None, "rc"),
                                                         f(r.part, "part"), st), "gsp_pair_fixed_chunk_f32")
            ops.gemm_tf32x3(r.G[:m], hiT, loT, out=r.g[r0:r0 + m])
        lib.check(L.b200gnn_gsp_finish_f32(f(r.part, "part"), S, f(r.loss_aux, "loss"), st), "gsp_finish_f32")
        if S < n:                  # rows outside the sample get no gradient; the buffer holds the previous step's
            d_feat.zero_()
        lib.check(L.b200gnn_gsp_rows_backward_f32(inds, S, H, k, f(r.g, "g"), f(r.x_s, "x_s"), H, f(r.norm, "norm"),
                                                  f(r.rc, "rc"), _EPS, self.beta, f(d_feat, "d_feat"), d_feat.stride(0),
                                                  f(r.loss_aux, "loss_aux"), f(tr.loss_out, "loss_out"), st),
                  "gsp_rows_backward_f32")


class BatchGSP:
    """GSP inside rgcn.RGCNTrainer's step: the reference's MAG ``train()`` with ``--training gpw``
    (mag_pyg/gnn_kd_and_aux.py:229-242; criterion.py:57-92) on every GraphSAINT batch b, with no projection heads:

        loss_aux = gpw_criterion(out, labels, model.out_feat[b.train_mask], teacher_model.out_feat[b.train_mask], kernel,
                                 beta, max_samples)[2]              mean((sim_s - sim_t)^2) over S = min(max_samples, n) rows
        loss     = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux

    Per batch, between the student's loss and its backward (``RGCNTrainer(..., gsp=o).train_step(b, x, teacher=t)``;
    uncaptured, the buffers sized on the host from the batch's n):

        rows         n = n_train, S = min(max_samples, n), Sp = S rounded up to 4
        draw         only when S < n: G-CRD's sampler (trainer seed, SAMPLE_STREAM, the student's device step counter) into
                     positions of the train rows, or the injected ``sample``; inds = train_int[perm[:S]] (int32 internal
                     rows), or train_int itself when S = n
        operands     b200gnn_gsp_rows_operands_f32 on the student's last hidden layer (after ReLU and dropout) and on the
                     teacher's (its eval forward on the student's plan: ReLU, no dropout), read at inds in place
        Gram chunks  per chunk of criterion.gsp_chunk_rows(Sp) rows, Gs_c = x_s[c] x_s^T and Gt_c = x_t[c] x_t^T on the
                     3xTF32 GEMM, as criterion.gsp_chunks forms them
        pair pass    b200gnn_gsp_pair_student_chunk_f32: d loss / d Gs_c in place, partial and (l2 / rbf) rc_s; the frozen
                     teacher's gradient is never formed
        contraction  b200gnn_gsp_contract_narrow_f32: g[c] = dGs_c . x_s in fp32 FMA over column slabs (the hidden width is
                     narrow: one GEMM tile per 128 rows would leave the device idle)
        finish       b200gnn_gsp_finish_f32
        backward     b200gnn_gsp_rows_backward_f32 into a zeroed internal-order [N, H] gradient at inds, which the trainer
                     adds at its last hidden layer; loss[0] += beta * loss_aux

    The operands, the Gram GEMMs, the pair pass and the finish are the eager route's (``train_step(teacher_logits=...,
    aux=lambda f: criterion.gpw_criterion(..., f[train_mask], t_feat[train_mask], kernel, 1, max_samples,
    sampled_inds=...)[2], beta=beta)``), so loss_aux and loss[0] equal it bit for bit; only the contraction's sums run in
    another order.  A batch with no train row does what the reference does: mse over nothing is NaN, so loss[0] and
    loss[2] are NaN, no GSP kernel runs and the model takes the KD step.  One train row is a 1 x 1 problem whose two
    similarities are equal: exactly for l2 and rbf (a row's distance to itself is 0), up to rounding for cosine and poly
    (|x / |x||^2 = 1; a zero row normalises to zero on both sides), so the loss and the gradient are zero or rounding.
    The reference's own loop refuses such a batch earlier, in cross_entropy (its labels.squeeze() leaves a 0-d target);
    the trainer's KD step takes it.  No parameters, no optimizer state."""

    NAME = "GSP"

    def __init__(self, hidden: int, teacher_hidden: int, kernel: str = "poly", beta: float = 1.0, max_samples: int = 24576,
                 device="cuda"):
        """hidden / teacher_hidden: the student's and the teacher's last hidden widths (32 and 512 in the reference's MAG
        models); hidden a multiple of 4 up to lib.GSP_CONTRACT_MAX_F, teacher_hidden a multiple of 4 up to
        lib.GSP_ROWS_MAX_F.  The defaults are the MAG script's (scripts/run_kd_and_aux.sh runs gpw with kernel poly and
        cosine, beta 1, max_samples 24576)."""
        if kernel not in criterion._KERNELS:
            raise ValueError(f"kernel {kernel!r}: GSP kernels are {sorted(criterion._KERNELS)}")
        if int(max_samples) < 1:
            raise ValueError("max_samples must be at least 1")
        hidden, teacher_hidden = int(hidden), int(teacher_hidden)
        if hidden % 4 or not 0 < hidden <= lib.GSP_CONTRACT_MAX_F:
            raise ValueError(f"hidden width {hidden}: the narrow GSP contraction takes a multiple of 4 up to "
                             f"{lib.GSP_CONTRACT_MAX_F}")
        if teacher_hidden % 4 or not 0 < teacher_hidden <= lib.GSP_ROWS_MAX_F:
            raise ValueError(f"teacher hidden width {teacher_hidden}: the GSP row passes take a multiple of 4 up to "
                             f"{lib.GSP_ROWS_MAX_F}")
        self.device = torch.device(device)
        self.H, self.F_t, self.beta, self.max_samples = hidden, teacher_hidden, float(beta), int(max_samples)
        self.kernel, self.kernel_id = kernel, criterion._KERNELS[kernel]
        self.loss_aux = torch.full((1,), float("nan"), device=self.device)
        self.inds: Optional[torch.Tensor] = None           # the last batch's sample: positions into its train rows

    def bind(self, trainer):
        """Called by the RGCNTrainer that owns this object: its last hidden layer must be the width built for."""
        if trainer.L < 2 or trainer.dims[-2] != self.H:
            raise ValueError(f"GSP built for hidden width {self.H}, the student's last hidden layer is "
                             f"{trainer.dims[-2] if trainer.L >= 2 else 'absent'}")

    def check_teacher(self, teacher):
        """ValueError unless the teacher's last hidden layer has the width built for."""
        if teacher.L < 2 or teacher.dims[-2] != self.F_t:
            raise ValueError(f"GSP built for teacher hidden width {self.F_t}, the teacher's last hidden layer is "
                             f"{teacher.dims[-2] if teacher.L >= 2 else 'absent'}")

    def check_batch(self, n: int, sample=None):
        """ValueError for a sample that is not S = min(max_samples, n) distinct positions in [0, n), or any sample when
        S = n (every train row is taken; there is nothing to draw)."""
        if sample is None:
            return
        S = min(self.max_samples, n)
        if S == n:
            raise ValueError(f"GSP takes every train row of this batch (max_samples {self.max_samples} >= {n}): there is "
                             "no sample to inject")
        check_sample(sample, n, S)

    def sample(self) -> torch.Tensor:
        """The last batch's sample: positions into its train rows (int64 [S])."""
        return self.inds.to(torch.int64) if self.inds is not None else torch.zeros(0, dtype=torch.int64)

    def forward_backward(self, tr, teacher, sample: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
        """After tr's loss on its forward and teacher's eval forward on the same plan: returns d (beta * loss_aux) / d out_feat
        [N, H] in internal row order (None when the batch has no train row) and adds beta * loss_aux to tr.loss_out[0]."""
        f, dev = tr._fwd, self.device
        train_int = f["train_int"]
        n = train_int.numel()
        if n == 0:
            self.inds = None
            self.loss_aux = torch.full((1,), float("nan"), device=dev)
            tr.loss_out[:1].add_(self.loss_aux * self.beta)
            return None
        S, H, Ft, k = min(self.max_samples, n), self.H, self.F_t, self.kernel_id
        Sp, raw = _ceil4(S), k >= 2
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)     # noqa: E731
        perm = torch.arange(n, dtype=torch.int32, device=dev)
        ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n)), dtype=torch.uint8, device=dev)
              if S < n and sample is None else None)
        draw_sample(tr, n, S, perm, ws, sample)
        self.inds = perm[:S]
        rows = (train_int[perm[:S].long()] if S < n else train_int).to(torch.int32)
        L, st = lib.load(), lib.stream_ptr()
        fp = lambda t, name: lib.dptr(t, torch.float32, name)      # noqa: E731
        # operands, zero-padded to Sp rows (the Gram GEMMs read all Sp rows of x as their B operand)
        x_s, x_t = torch.zeros(Sp, H, device=dev), torch.zeros(Sp, Ft, device=dev)
        norm_s, norm_t = e(Sp), e(Sp)
        for feat, x, nrm, F, name in ((f["xs"][-1], x_s, norm_s, H, "student"),
                                      (teacher._fwd["xs"][-1], x_t, norm_t, Ft, "teacher")):
            lib.check(L.b200gnn_gsp_rows_operands_f32(fp(feat, name), feat.stride(0), rows.data_ptr(), S, F, k, _EPS,
                                                      fp(x, "x"), F, fp(nrm, "norm"), st), "gsp_rows_operands_f32")
        hs, ls = ops.split_tf32(x_s)
        ht, lt = ops.split_tf32(x_t)
        R = criterion.gsp_chunk_rows(Sp)
        Gs, Gt = e(R, Sp), e(R, Sp)
        rc_s, part, g, loss = (e(Sp) if raw else None), e(Sp), e(Sp, H), e(1)
        cws = ops.gsp_contract_workspace(min(R, S), S, H, dev)
        for r0 in range(0, S, R):
            r = min(R, S - r0)
            ops.gemm_tf32x3(x_s[r0:r0 + r], hs, ls, out=Gs[:r])
            ops.gemm_tf32x3(x_t[r0:r0 + r], ht, lt, out=Gt[:r])
            lib.check(L.b200gnn_gsp_pair_student_chunk_f32(fp(Gs, "Gs"), fp(Gt, "Gt"), Sp, r, S, r0,
                                                           fp(norm_s if raw else None, "ns"), fp(norm_t if raw else None, "nt"),
                                                           k, fp(rc_s, "rc_s"), fp(part, "part"), st),
                      "gsp_pair_student_chunk_f32")
            ops.gsp_contract_narrow(Gs[:r], S, x_s, g[r0:r0 + r], cws)
        lib.check(L.b200gnn_gsp_finish_f32(fp(part, "part"), S, fp(loss, "loss"), st), "gsp_finish_f32")
        self.loss_aux = loss
        d_feat = torch.zeros(f["P"].N, H, device=dev)
        lib.check(L.b200gnn_gsp_rows_backward_f32(rows.data_ptr(), S, H, k, fp(g, "g"), fp(x_s, "x_s"), H, fp(norm_s, "norm"),
                                                  fp(rc_s, "rc"), _EPS, self.beta, fp(d_feat, "d_feat"), H, fp(loss, "loss_aux"),
                                                  fp(tr.loss_out, "loss_out"), st), "gsp_rows_backward_f32")
        return d_feat
