"""The projection heads of the students' captured distillation objectives (G-CRD in gcrd.py, GSP in gsp.py).

Both objectives of the reference (arxiv_pyg/gnn_kd_and_aux.py:275-297) project the student's and the teacher's features
through a head of their own, trained in the same Adam as the model:

    P_s  = relu(BN_s(Linear_s(model.out_feat[train_idx])))          Linear_s: hidden -> proj_dim
    P_t  = relu(BN_t(Linear_t(teacher_out_feat[train_idx])))        Linear_t: 750 -> proj_dim (trained too)
    inds = S = min(max_samples, n_train) distinct rows of [0, n_train)

``ProjectionHeads`` owns both heads (flat parameters, Adam state, BatchNorm running statistics, state-dict I/O), the row
sample and every buffer around the objective.  Its ``forward_backward`` runs, as launches only (capturable):

    sample       Philox key per training row at (trainer seed, SAMPLE_STREAM, device step counter), radix argsort, first S
    gather       out_feat[train_idx] -> [n_train, H] (GCN: formed from Y, BN scale/shift and the keep bits)
    heads        3xTF32 GEMM with the BatchNorm statistics in its epilogue, bn_finalize (running statistics update)
    objective    the subclass's ``_objective``: operands of the S sampled rows, the loss, and a backward kernel that stores
                 dz = beta * d loss / d (BN output) at the sampled rows of the zero-filled [n_train, P] dz_s / dz_t, the
                 BatchNorm-backward partials bpart_s / bpart_t, and adds beta * loss_aux to the trainer's loss
    tail         bn_act_bwd_apply; weight gradients; the student head's input gradient stored straight into the training
                 rows of d out_feat
    Adam         over the heads' flat buffer, after the trainer's own Adam (same lr: one Adam over three groups)

The sample cannot equal numpy's ``np.random.choice`` draw; ``train_step(..., sample=)`` injects one (tests).
"""
from __future__ import annotations

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


class ProjectionHeads:
    NAME = "projection"                      # the objective's name in error messages

    def __init__(self, teacher_feat: torch.Tensor, train_idx: torch.Tensor, hidden: int, proj_dim: int, max_samples: int,
                 beta: float, seed: int, bn_eps: float, bn_momentum: float):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file, F_t = 750); train_idx: the
        training rows, the same tensor the trainer's step receives.  proj_dim a multiple of 32 in (48, 256]."""
        if not ops.gemm_stats_supported(proj_dim):
            raise ValueError("proj_dim must be a multiple of 32 in (48, 256]")
        if hidden % 4 or not 0 < hidden <= 512:
            raise ValueError("hidden width must be a multiple of 4 up to 512 (the student head's weight-gradient GEMM)")
        if not 0 < _ceil4(teacher_feat.shape[1]) <= 2048:
            raise ValueError("teacher feature width must be at most 2048 (the teacher head's weight-gradient GEMM)")
        dev = teacher_feat.device
        self.device = dev
        self.train_idx = train_idx.to(dev, torch.int64).contiguous()
        self.n = n = self.train_idx.numel()
        self.H, self.P, self.F_t = hidden, proj_dim, teacher_feat.shape[1]
        self.Ft_pad = _ceil4(self.F_t)
        self.S = min(int(max_samples), n)
        self.Sp = _ceil4(self.S)
        self.beta = float(beta)
        self.bn_eps, self.bn_momentum = float(bn_eps), float(bn_momentum)
        P, H, Ftp = self.P, self.H, self.Ft_pad
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        z = lambda *shape: torch.zeros(*shape, dtype=torch.float32, device=dev)

        # the teacher rows of the loss are constants: gathered once, zero-padded to a 16-byte row pitch
        self.G_t = z(n, Ftp)
        self.G_t[:, :self.F_t].copy_(teacher_feat.detach().to(torch.float32)[self.train_idx])

        # flat parameters: student W [P, H], b, gamma, beta; teacher W [P, Ft_pad], b, gamma, beta.  step_count counts the
        # heads' Adam steps (= BN batches)
        self.store = FlatParams([(P, H), (P,), (P,), (P,), (P, Ftp), (P,), (P,), (P,)], dev).attach(self)
        self._nbt_base = {"s": 0, "t": 0}         # num_batches_tracked = step_count + base, per head
        views = self.store.views
        (self.W_s, self.gW_s), (self.b_s, self.gb_s), (self.gamma_s, self.ggamma_s), (self.beta_s, self.gbeta_s) = views[:4]
        (self.W_t, self.gW_t), (self.b_t, self.gb_t), (self.gamma_t, self.ggamma_t), (self.beta_t, self.gbeta_t) = views[4:]
        self.rm_s, self.rv_s, self.rm_t, self.rv_t = z(P), z(P), z(P), z(P)
        self.reset_parameters(seed)

        # forward buffers
        self.G_s = e(n, H)                                       # out_feat[train_idx]
        self.pre_s, self.pre_t = e(n, P), e(n, P)                # Linear outputs (BatchNorm inputs)
        slots = ops.gemm_stat_slots(n, P)
        self.gp_s, self.gp_t = e(slots, 2, P), e(slots, 2, P)
        self.bn_s, self.bn_t = e(4, P), e(4, P)                  # mean, invstd, scale, shift
        self.Ws_split, self.Wt_split = (e(P, H), e(P, H)), (e(P, Ftp), e(P, Ftp))
        self.WsT_split = (e(H, P), e(H, P))
        # the sample: positions into train_idx (int32); all rows in order when max_samples >= n_train
        self.perm = torch.arange(n, dtype=torch.int32, device=dev)
        self.inds = self.perm[:self.S]
        self.sample_ws = (torch.empty(int(lib.load().b200gnn_gcrd_sample_workspace_bytes(n)), dtype=torch.uint8, device=dev)
                          if self.S < n else None)
        self.x_s, self.x_t = z(self.Sp, P), z(self.Sp, P)        # the objective's operands; padding rows stay zero
        # backward buffers
        self.dz_s, self.dz_t = e(n, P), e(n, P)
        bslots = int(lib.load().b200gnn_gcrd_bwd_slots())
        self.bpart_s, self.bpart_t = e(bslots, 2, P), e(bslots, 2, P)
        self.rows_part, self.coef = e(ops.rows_slots(n), 2, P), e(3, P)
        self.gWt_T = e(Ftp, P)
        self.ws_wide = not ops.wgrad_supported(P, H)
        self.wgrad_ws = e(max(ops.wgrad_workspace_floats(P, H), ops.wgrad_workspace_floats(Ftp, P)))
        self.d_feat: Optional[torch.Tensor] = None

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
        L, st = lib.load(), lib.stream_ptr()
        n, P, S = self.n, self.P, self.S
        if sample is not None:
            # the kernels index pre_s / pre_t and store dz rows by these positions: refuse what would go out of bounds or
            # store one row twice (the override runs eagerly, so a host check costs nothing the step depends on)
            s = torch.as_tensor(sample).to("cpu", torch.int64).view(-1)
            if s.numel() != S or (S and (int(s.min()) < 0 or int(s.max()) >= n)) or s.unique().numel() != S:
                raise ValueError(f"sample must hold {S} distinct positions in [0, {n})")
            self.perm[:S].copy_(s.to(torch.int32))
        elif S < n:
            lib.check(L.b200gnn_gcrd_sample_i32(n, tr.seed, SAMPLE_STREAM, lib.dptr(tr.step_count, torch.int32, "step"),
                                                self.perm.data_ptr(), self.sample_ws.data_ptr(), st), "gcrd_sample_i32")
        # model.out_feat[train_idx]
        if getattr(tr, "_fwd_fused", False):
            l = tr.L - 2
            ops.gather_rows_act(tr.Y[l], self.train_idx, self.G_s, bits=tr.keep_bits[l], scale=tr.bn[l][2],
                                shift=tr.bn[l][3], p=tr.p)
        else:
            ops.gather_rows_act(tr.out_feat(), self.train_idx, self.G_s)
        # heads: Linear with the BatchNorm statistics in the GEMM epilogue, then finalize (running statistics)
        for G, W, b, gamma, beta, rm, rv, pre, gp, bn, split in (
                (self.G_s, self.W_s, self.b_s, self.gamma_s, self.beta_s, self.rm_s, self.rv_s, self.pre_s, self.gp_s, self.bn_s,
                 self.Ws_split),
                (self.G_t, self.W_t, self.b_t, self.gamma_t, self.beta_t, self.rm_t, self.rv_t, self.pre_t, self.gp_t, self.bn_t,
                 self.Wt_split)):
            hi, lo = ops.split_tf32(W, hi=split[0], lo=split[1])
            ops.gemm_tf32x3_stats(G, hi, lo, b, pre, gp)
            ops.bn_finalize(gp, n, gamma, beta, self.bn_eps, self.bn_momentum, rm, rv, out=bn)
        self._objective(tr)
        for dz, pre, bn, gamma, part, gg, gbe, gb in (
                (self.dz_s, self.pre_s, self.bn_s, self.gamma_s, self.bpart_s, self.ggamma_s, self.gbeta_s, self.gb_s),
                (self.dz_t, self.pre_t, self.bn_t, self.gamma_t, self.bpart_t, self.ggamma_t, self.gbeta_t, self.gb_t)):
            ops.bn_act_bwd_apply(dz, None, pre, bn[0], bn[1], gamma, part, n, 0.0, dz, gg, gbe, gb, self.rows_part, self.coef)
        ops.gemm_wgrad_tf32x3(self.dz_s, self.G_s, out=self.gW_s, workspace=self.wgrad_ws, wide=self.ws_wide)
        ops.gemm_wgrad_tf32x3(self.G_t, self.dz_t, out=self.gWt_T, workspace=self.wgrad_ws, wide=True)
        lib.check(L.b200gnn_transpose_f32(lib.dptr(self.gWt_T, torch.float32, "gWt_T"), self.Ft_pad, P,
                                          lib.dptr(self.gW_t, torch.float32, "gW_t"), st), "transpose_f32")
        # d out_feat: the student head's input gradient in the training rows, zero elsewhere (the GCN backward reuses this
        # buffer as its dz, so it is cleared every step)
        self.d_feat.zero_()
        hi, lo = ops.split_tf32(self.W_s, transpose=True, hi=self.WsT_split[0], lo=self.WsT_split[1])
        ops.gemm_tf32x3_rowidx(self.dz_s, hi, lo, self.d_feat, self.train_idx)
        return self.d_feat

    def _objective(self, tr):
        """The objective between the head front and the tail (see the module docstring); enqueues launches only."""
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
