"""The projection heads of the students' captured distillation objectives (G-CRD in gcrd.py, GSP in gsp.py).

Both objectives of the reference (arxiv_pyg/gnn_kd_and_aux.py:275-297) project the student's and the teacher's features
through a head of their own, trained in the same Adam as the model:

    P_s  = relu(BN_s(Linear_s(model.out_feat[train_idx])))          Linear_s: hidden -> proj_dim
    P_t  = relu(BN_t(Linear_t(teacher_out_feat[train_idx])))        Linear_t: 750 -> proj_dim (trained too)
    inds = S = min(max_samples, n_train) distinct rows of [0, n_train)

``ProjectionHeads`` owns both heads (flat parameters, Adam state, BatchNorm running statistics, state-dict I/O); a
``HeadRows`` holds what one row set fixes (n, S, the teacher rows, the sample and every buffer whose shape follows n or S).
``ProjectionHeads`` builds one over train_idx; gcrd.PerGraphGCRD builds one per PPI training graph, on views of shared
buffers (``_Pool``).  Its ``forward_backward`` runs, as launches only (capturable):

    sample       Philox key per training row at (trainer seed, SAMPLE_STREAM, device step counter), radix argsort, first S
    gather       out_feat[train_idx] -> [n_train, H] (GCN: formed from Y, BN scale/shift and the keep bits)
    heads        3xTF32 GEMM with the BatchNorm statistics in its epilogue, bn_finalize (running statistics update)
    objective    the subclass's ``_objective``: operands of the S sampled rows, the loss, and a backward kernel that stores
                 dz = beta * d loss / d (BN output) at the sampled rows of the zero-filled [n_train, P] dz_s / dz_t, the
                 BatchNorm-backward partials bpart_s / bpart_t, and adds beta * loss_aux to the trainer's loss
    tail         bn_act_bwd_apply; weight gradients; the student head's input gradient stored straight into the training
                 rows of d out_feat

The draw, the heads, the objective and the tail (``_draw``, ``_front``, ``_objective``, ``_tail``) take the row set, so the
per-graph form runs the same launches with no gather and its own store of the input gradient.  The student head's halves
of the front and the tail (``_front_student``, ``_wgrad_student``) are separate, so gcrd.SIGNGCRD, whose head reads the
un-stored dropout(prelu(cat)), replaces them alone.
    Adam         over the heads' flat buffer, after the trainer's own Adam (same lr: one Adam over three groups)

The sample cannot equal numpy's ``np.random.choice`` draw; ``train_step(..., sample=)`` injects one (tests).
"""
from __future__ import annotations

import contextlib
import itertools
import math
from typing import Dict, Optional

import torch

from . import lib, ops
from .trainer import FlatParams

# Philox stream of the row sample.  The dropout masks use offsets layer + step * L, far below this.  G-CRD and GSP share
# it: a trainer runs one objective.
SAMPLE_STREAM = 1 << 62


def _ceil4(n: int) -> int:
    return (n + 3) // 4 * 4


class _Pool:
    """Per-step buffers of row sets that never live at once (one training graph per step): the k-th buffer each row set
    asks for is a view at the front of one flat buffer, sized for the largest such request.  ``recorder()`` hands out shapes
    only (meta tensors) and records the sizes; ``views()`` then hands out the views, so each row set is built twice."""

    def __init__(self, device):
        self.device, self.sizes, self.flat = device, [], None

    def recorder(self):
        k = itertools.count()

        def alloc(*shape, dtype=torch.float32):
            j = next(k)
            if j == len(self.sizes):
                self.sizes.append((0, dtype))
            assert self.sizes[j][1] == dtype, "row sets must ask for their buffers in the same order"
            self.sizes[j] = (max(self.sizes[j][0], math.prod(shape)), dtype)
            return torch.empty(*shape, dtype=dtype, device="meta")
        return alloc

    def views(self):
        if self.flat is None:
            self.flat = [torch.empty(size, dtype=dtype, device=self.device) for size, dtype in self.sizes]
        k = itertools.count()
        return lambda *shape, dtype=torch.float32: self.flat[next(k)][:math.prod(shape)].view(*shape)


class HeadRows:
    """One row set of the heads' step: its n rows (the BatchNorm batch), the S = min(max_samples, n) sampled of them, the
    teacher's rows and every buffer whose shape follows n or S.  ``alloc(*shape)`` makes the buffers (torch.empty, or views
    of a _Pool); x_s / x_t are the objective's zero-padded [Sp, P] operands, whose padding rows must stay zero."""

    def __init__(self, heads: "ProjectionHeads", n: int, S: int, G_t: torch.Tensor, x_s: torch.Tensor, x_t: torch.Tensor,
                 alloc):
        P = heads.P
        self.n, self.S, self.Sp, self.G_t = n, S, _ceil4(S), G_t
        self.pre_s, self.pre_t = alloc(n, P), alloc(n, P)             # Linear outputs (BatchNorm inputs)
        slots = ops.gemm_stat_slots(n, P)
        self.gp_s, self.gp_t = alloc(slots, 2, P), alloc(slots, 2, P)
        # the sample: positions into the row set (int32); all rows in order when max_samples >= n
        self.perm = torch.arange(n, dtype=torch.int32, device=heads.device)
        self.inds = self.perm[:S]
        self.x_s, self.x_t = x_s, x_t
        self.dz_s, self.dz_t = alloc(n, P), alloc(n, P)
        self.rows_part = alloc(ops.rows_slots(n), 2, P)
        heads._objective_buffers(self, alloc)


def check_sample(sample, n: int, S: int) -> torch.Tensor:
    """An injected sample as int64 [S] on the host; ValueError unless it holds S distinct positions in [0, n)."""
    # the kernels index rows and store gradient rows by these positions: refuse what would go out of bounds or store one
    # row twice (the override runs eagerly, so a host check costs nothing the step depends on)
    s = torch.as_tensor(sample).to("cpu", torch.int64).view(-1)
    if s.numel() != S or (S and (int(s.min()) < 0 or int(s.max()) >= n)) or s.unique().numel() != S:
        raise ValueError(f"sample must hold {S} distinct positions in [0, {n})")
    return s


def draw_sample(tr, n: int, S: int, perm: torch.Tensor, workspace: Optional[torch.Tensor], sample: Optional[torch.Tensor]):
    """The step's sample of S of n rows into perm[:S] (int32 [n]): the injected ``sample``, or, when S < n, the on-device
    draw at (trainer seed, SAMPLE_STREAM, the trainer's device step counter) on ``workspace``
    (b200gnn_gcrd_sample_workspace_bytes(n) bytes).  Nothing when S = n and no sample is given."""
    if sample is not None:
        perm[:S].copy_(check_sample(sample, n, S).to(torch.int32))
    elif S < n:
        L = lib.load()
        lib.check(L.b200gnn_gcrd_sample_i32(n, tr.seed, SAMPLE_STREAM, lib.dptr(tr.step_count, torch.int32, "step"),
                                            perm.data_ptr(), workspace.data_ptr(), lib.stream_ptr()), "gcrd_sample_i32")


def check_widths(hidden: int, proj_dim: int, teacher_width: int):
    """ValueError for a head shape the step's kernels do not take."""
    if not ops.gemm_stats_supported(proj_dim):
        raise ValueError("proj_dim must be a multiple of 32 in (48, 256]")
    if hidden % 4 or not 0 < hidden <= 512:
        raise ValueError("hidden width must be a multiple of 4 up to 512 (the student head's weight-gradient GEMM)")
    if not 0 < _ceil4(teacher_width) <= 2048:
        raise ValueError("teacher feature width must be at most 2048 (the teacher head's weight-gradient GEMM)")


class ProjectionHeads:
    NAME = "projection"                      # the objective's name in error messages

    def __init__(self, teacher_feat: torch.Tensor, train_idx: torch.Tensor, hidden: int, proj_dim: int, max_samples: int,
                 beta: float, seed: int, bn_eps: float, bn_momentum: float):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file, F_t = 750); train_idx: the
        training rows, the same tensor the trainer's step receives.  proj_dim a multiple of 32 in (48, 256]."""
        check_widths(hidden, proj_dim, teacher_feat.shape[1])
        self._init_heads(hidden, proj_dim, teacher_feat.shape[1], beta, seed, bn_eps, bn_momentum, teacher_feat.device)
        dev, P = self.device, self.P
        self.train_idx = train_idx.to(dev, torch.int64).contiguous()
        n = self.train_idx.numel()
        S = min(int(max_samples), n)
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=dev)
        # the teacher rows of the loss are constants: gathered once, zero-padded to a 16-byte row pitch
        G_t = z(n, self.Ft_pad)
        G_t[:, :self.F_t].copy_(teacher_feat.detach().to(torch.float32)[self.train_idx])
        self.rows = HeadRows(self, n, S, G_t, z(_ceil4(S), P), z(_ceil4(S), P),
                             lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev))
        self.__dict__.update(vars(self.rows))                   # n, S, G_t, pre_s, ..., the objective's buffers
        self.G_s = torch.empty(n, self.H, dtype=torch.float32, device=dev)   # out_feat[train_idx]
        self.sample_ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n)), dtype=torch.uint8, device=dev)
                          if S < n else None)
        self.d_feat: Optional[torch.Tensor] = None

    def _init_heads(self, hidden: int, proj_dim: int, teacher_width: int, beta: float, seed: int, bn_eps: float,
                    bn_momentum: float, dev):
        """Everything that does not depend on the rows: both heads, their Adam state, running statistics and the buffers
        whose shape is set by the widths alone."""
        self.device = dev
        self.H, self.P, self.F_t = hidden, proj_dim, teacher_width
        self.Ft_pad = _ceil4(self.F_t)
        self.beta = float(beta)
        self.bn_eps, self.bn_momentum = float(bn_eps), float(bn_momentum)
        P, H, Ftp = self.P, self.H, self.Ft_pad
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=dev)

        # flat parameters: student W [P, H], b, gamma, beta; teacher W [P, Ft_pad], b, gamma, beta.  step_count counts the
        # heads' Adam steps (= BN batches)
        self.store = FlatParams([(P, H), (P,), (P,), (P,), (P, Ftp), (P,), (P,), (P,)], dev).attach(self)
        self._nbt_base = {"s": 0, "t": 0}         # num_batches_tracked = step_count + base, per head
        views = self.store.views
        (self.W_s, self.gW_s), (self.b_s, self.gb_s), (self.gamma_s, self.ggamma_s), (self.beta_s, self.gbeta_s) = views[:4]
        (self.W_t, self.gW_t), (self.b_t, self.gb_t), (self.gamma_t, self.ggamma_t), (self.beta_t, self.gbeta_t) = views[4:]
        self.rm_s, self.rv_s, self.rm_t, self.rv_t = z(P), z(P), z(P), z(P)
        self.reset_parameters(seed)

        self.bn_s, self.bn_t = e(4, P), e(4, P)                  # mean, invstd, scale, shift
        self.Ws_split, self.Wt_split = (e(P, H), e(P, H)), (e(P, Ftp), e(P, Ftp))
        self.WsT_split = (e(H, P), e(H, P))
        bslots = int(lib.load().b200gnn_gcrd_bwd_slots())
        self.bpart_s, self.bpart_t = e(bslots, 2, P), e(bslots, 2, P)
        self.coef = e(3, P)
        self.gWt_T = e(Ftp, P)
        self.ws_wide = not ops.wgrad_supported(P, H)
        self.wgrad_ws = e(max(ops.wgrad_workspace_floats(P, H), ops.wgrad_workspace_floats(Ftp, P)))

    def _objective_buffers(self, rows: HeadRows, alloc):
        """The objective's own buffers of one row set (attributes of ``rows``), made with ``alloc``."""

    # ------------------------------------------------------------------ parameters
    def reset_parameters(self, seed: int = 0):
        """nn.Linear's default initialisation (U(+-1/sqrt(fan_in)) for weight and bias), BatchNorm1d ones / zeros."""
        g = torch.Generator().manual_seed(seed)
        for W, b, fan_in in ((self.W_s, self.b_s, self.H), (self.W_t, self.b_t, self.F_t)):
            bound = 1.0 / math.sqrt(fan_in)
            W.zero_()
            W[:, :fan_in].copy_((torch.rand(self.P, fan_in, generator=g) * 2 - 1) * bound)
            b.copy_((torch.rand(self.P, generator=g) * 2 - 1) * bound)
        for t in (self.gamma_s, self.gamma_t, self.rv_s, self.rv_t):
            t.fill_(1.0)
        for t in (self.beta_s, self.beta_t, self.rm_s, self.rm_t, self.exp_avg, self.exp_avg_sq, self.step_count):
            t.zero_()
        self._nbt_base = {"s": 0, "t": 0}

    def _state(self, W, b, gamma, beta, rm, rv, fan_in, head) -> Dict[str, torch.Tensor]:
        return {"0.weight": W[:, :fan_in].clone(), "0.bias": b.clone(), "1.weight": gamma.clone(), "1.bias": beta.clone(),
                "1.running_mean": rm.clone(), "1.running_var": rv.clone(),
                "1.num_batches_tracked": (self.step_count[0].to(torch.int64) + self._nbt_base[head]).cpu()}

    def student_proj_state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys of the reference's nn.Sequential(Linear, BatchNorm1d, ReLU) student head."""
        return self._state(self.W_s, self.b_s, self.gamma_s, self.beta_s, self.rm_s, self.rv_s, self.H, "s")

    def teacher_proj_state_dict(self) -> Dict[str, torch.Tensor]:
        """The teacher head's, with its Linear at the teacher's own width (750 columns, not the padded pitch)."""
        return self._state(self.W_t, self.b_t, self.gamma_t, self.beta_t, self.rm_t, self.rv_t, self.F_t, "t")

    def _load(self, sd, W, b, gamma, beta, rm, rv, fan_in, head):
        W.zero_()
        W[:, :fan_in].copy_(sd["0.weight"]); b.copy_(sd["0.bias"])
        gamma.copy_(sd["1.weight"]); beta.copy_(sd["1.bias"])
        if "1.running_mean" in sd:
            rm.copy_(sd["1.running_mean"]); rv.copy_(sd["1.running_var"])
        if "1.num_batches_tracked" in sd:
            self._nbt_base[head] = int(sd["1.num_batches_tracked"]) - int(self.step_count.item())

    def load_student_proj_state_dict(self, sd: Dict[str, torch.Tensor]):
        self._load(sd, self.W_s, self.b_s, self.gamma_s, self.beta_s, self.rm_s, self.rv_s, self.H, "s")

    def load_teacher_proj_state_dict(self, sd: Dict[str, torch.Tensor]):
        self._load(sd, self.W_t, self.b_t, self.gamma_t, self.beta_t, self.rm_t, self.rv_t, self.F_t, "t")

    def sample(self) -> torch.Tensor:
        """The last step's sample: positions into train_idx (int64 [S]), as ``np.random.choice(n_train, S)`` would give."""
        return self.inds.to(torch.int64)

    @contextlib.contextmanager
    def preserved(self):
        """Parameters, Adam state, the step counter (and with it num_batches_tracked) and the running statistics are put back
        on exit as they were on entry."""
        running = (self.rm_s, self.rv_s, self.rm_t, self.rv_t)
        saved = [t.clone() for t in running]
        with self.store.preserved():
            yield
        for t, v in zip(running, saved):
            t.copy_(v)

    # ------------------------------------------------------------------ the step
    def bind(self, trainer):
        """Called by the trainer that owns this object: the [N, H] gradient of out_feat the step writes."""
        if trainer.dims[-2] != self.H:
            raise ValueError(f"{self.NAME} head built for hidden width {self.H}, "
                             f"the student's last hidden layer is {trainer.dims[-2]}")
        self.d_feat = torch.zeros(trainer.N, self.H, device=self.device)
        self.trainer = trainer

    def forward_backward(self, tr, sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Everything between the trainer's loss and its backward: returns d (beta * loss_aux) / d out_feat [N, H] and adds
        beta * loss_aux to tr.loss_out[0].  Enqueues launches only (capturable)."""
        r = self.rows
        self._draw(tr, r, sample)
        # model.out_feat[train_idx]
        if getattr(tr, "_fwd_fused", False):
            l = tr.L - 2
            ops.gather_rows_act(tr.Y[l], self.train_idx, self.G_s, bits=tr.keep_bits[l], scale=tr.bn[l][2],
                                shift=tr.bn[l][3], p=tr.p)
        else:
            ops.gather_rows_act(tr.out_feat(), self.train_idx, self.G_s)
        self._front(r, self.G_s)
        self._objective(tr, r)
        self._tail(r, self.G_s)
        # d out_feat: the student head's input gradient in the training rows, zero elsewhere (the GCN backward reuses this
        # buffer as its dz, so it is cleared every step)
        self.d_feat.zero_()
        hi, lo = ops.split_tf32(self.W_s, transpose=True, hi=self.WsT_split[0], lo=self.WsT_split[1])
        ops.gemm_tf32x3_rowidx(r.dz_s, hi, lo, self.d_feat, self.train_idx)
        return self.d_feat

    def _draw(self, tr, r: HeadRows, sample: Optional[torch.Tensor]):
        """The step's sample into r.perm: the injected one, or the on-device draw when S < n (none when S = n)."""
        draw_sample(tr, r.n, r.S, r.perm, self.sample_ws, sample)

    def _front(self, r: HeadRows, G_s):
        """Both heads' Linear over the row set with the BatchNorm statistics in the GEMM epilogue, then finalize (running
        statistics).  G_s: the student head's input, as ``_front_student`` reads it."""
        self._front_student(r, G_s)
        self._front_teacher(r)

    def _front_student(self, r: HeadRows, G_s):
        """The student half of ``_front``; G_s the head's input [n, H].  A subclass whose student head reads its input in
        another form overrides this and ``_wgrad_student``."""
        hi, lo = ops.split_tf32(self.W_s, hi=self.Ws_split[0], lo=self.Ws_split[1])
        ops.gemm_tf32x3_stats(G_s, hi, lo, self.b_s, r.pre_s, r.gp_s)
        ops.bn_finalize(r.gp_s, r.n, self.gamma_s, self.beta_s, self.bn_eps, self.bn_momentum, self.rm_s, self.rv_s,
                        out=self.bn_s)

    def _front_teacher(self, r: HeadRows):
        hi, lo = ops.split_tf32(self.W_t, hi=self.Wt_split[0], lo=self.Wt_split[1])
        ops.gemm_tf32x3_stats(r.G_t, hi, lo, self.b_t, r.pre_t, r.gp_t)
        ops.bn_finalize(r.gp_t, r.n, self.gamma_t, self.beta_t, self.bn_eps, self.bn_momentum, self.rm_t, self.rv_t,
                        out=self.bn_t)

    def _tail(self, r: HeadRows, G_s):
        """The BatchNorm backward apply over the row set and both heads' weight gradients; the student head's input
        gradient r.dz_s . W_s is the caller's."""
        for dz, pre, bn, gamma, part, gg, gbe, gb in (
                (r.dz_s, r.pre_s, self.bn_s, self.gamma_s, self.bpart_s, self.ggamma_s, self.gbeta_s, self.gb_s),
                (r.dz_t, r.pre_t, self.bn_t, self.gamma_t, self.bpart_t, self.ggamma_t, self.gbeta_t, self.gb_t)):
            ops.bn_act_bwd_apply(dz, None, pre, bn[0], bn[1], gamma, part, r.n, 0.0, dz, gg, gbe, gb, r.rows_part, self.coef)
        self._wgrad_student(r, G_s)
        self._wgrad_teacher(r)

    def _wgrad_student(self, r: HeadRows, G_s):
        """gW_s = r.dz_s^T . G_s: the student half of ``_tail``."""
        ops.gemm_wgrad_tf32x3(r.dz_s, G_s, out=self.gW_s, workspace=self.wgrad_ws, wide=self.ws_wide)

    def _wgrad_teacher(self, r: HeadRows):
        ops.gemm_wgrad_tf32x3(r.G_t, r.dz_t, out=self.gWt_T, workspace=self.wgrad_ws, wide=True)
        lib.check(lib.load().b200gnn_transpose_f32(lib.dptr(self.gWt_T, torch.float32, "gWt_T"), self.Ft_pad, self.P,
                                                   lib.dptr(self.gW_t, torch.float32, "gW_t"), lib.stream_ptr()),
                  "transpose_f32")

    def _objective(self, tr, r: HeadRows):
        """The objective between the head front and the tail on row set r (see the module docstring); enqueues launches
        only."""
        raise NotImplementedError

    def optimizer_step(self, lr: float):
        self.store.adam(lr)

    def launches_per_step(self, x, y, train_idx, teacher_logits=None) -> int:
        """b200gnn kernel launches of one whole training step of the bound trainer, the objective included.  Counted by running
        one real step on these inputs: it advances the trainer's and the heads' parameters, Adam state, running statistics and
        step counters like any other step.  (The trainer's own launches_per_step counts the same step on its captured inputs.)"""
        before = lib.launch_count()
        self.trainer._step_impl(x, y, train_idx, teacher_logits)
        return lib.launch_count() - before
