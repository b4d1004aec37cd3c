"""Fused mini-batch training step for the SIGN student (arxiv_dgl/sign.py:105-157, loops :221-401).

One step of ``train_kd_and_aux`` on a batch of training nodes, with the hop features precomputed by
``nn.neighbor_average_features``:

    x_h   = input_dropout(feats[h][batch])                 one gather launch for every hop, + label / teacher rows
    Z_h,i = x Wᵀ + b through each hop's FeedForwardNet     3xTF32 GEMMs; x = dropout(prelu_h(Z_h,i-1)) is formed in the
                                                           A-operand prologue, never stored
    cat   = [Z_0,last | ... | Z_H-1,last]                  the hop FFNs' last GEMMs write their column blocks (ldc)
    logits = project(dropout(prelu(cat)))                  same prologue on the 3072-wide concatenation
    loss, dlogits = fused CE / logit-KD row kernel
    backward: dW from the weight-gradient GEMM with the same prologue; dZ (and the PReLU slope gradient) from the
    input-gradient GEMM whose epilogue applies the PReLU/dropout backward; bias gradients by fixed-order column sums.
    Adam over one flat parameter buffer (slopes included).

No autograd tape: buffers are preallocated for the batch size and a step is graph-capturable (one graph per batch size).
Dropout decisions are a pure function of (seed, step, layer, element) through the project's Philox generator.

With ``gcrd=`` (a gcrd.SIGNGCRD) the step is ``train_kd_and_aux`` with ``--training nce`` (sign.py:355-367): between the
loss and the backward the projection heads read dropout(prelu(cat)) through the same prologue, the InfoNCE runs on a sample
of the batch, and the student head's input gradient is stored into dZcat, onto which the project FFN's first input-gradient
GEMM accumulates; the heads' Adam follows the model's.  The step stays one CUDA graph per batch size.
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict, List, Optional

import torch

from . import lib, ops
from .trainer import FlatParams, aux_grad, capture_graph


class _Acts:
    """Forward activations of ``rows`` batch rows (and, for training, their gradients)."""

    def __init__(self, t: "SIGNStudentTrainer", rows: int, train: bool):
        dev, H, F, hid, C, ff = t.device, t.H, t.F, t.hidden, t.C, t.ff
        self.rows, self.H, self.F = rows, H, F
        self.xg = torch.empty(H * rows * F, device=dev)                       # gathered, input-dropped hop features
        self.Zh = [[torch.empty(rows, hid, device=dev) for _ in range(ff - 1)] for _ in range(H)]
        self.Zcat = torch.empty(rows, H * hid, device=dev)
        self.Zp = [torch.empty(rows, hid, device=dev) for _ in range(ff - 1)]
        self.logits = torch.empty(rows, C, device=dev)
        self.labels = torch.empty(rows, dtype=torch.int64, device=dev)
        self.teacher = torch.empty(rows, C, device=dev)
        self.n_hbits = (H + 1) * (ff - 1)                                    # hidden dropout layers of the step
        self.hbits = torch.empty(max(self.n_hbits, 1) * rows * (hid // 32), dtype=torch.int32, device=dev)
        self.catbits = torch.empty(rows * H * hid // 32, dtype=torch.int32, device=dev)
        if train:
            self.dlogits = torch.empty(rows, C, device=dev)
            self.dZh = [[torch.empty(rows, hid, device=dev) for _ in range(ff - 1)] for _ in range(H)]
            self.dZcat = torch.empty(rows, H * hid, device=dev)
            self.dZp = [torch.empty(rows, hid, device=dev) for _ in range(ff - 1)]
            self.out_feat = torch.empty(rows, H * hid, device=dev)
        else:                                                                 # eval: every element kept
            self.hbits.fill_(-1)
            self.catbits.fill_(-1)

    def xall(self, B: int) -> torch.Tensor:
        return self.xg[:self.H * B * self.F].view(self.H, B, self.F)

    def hb(self, B: int, j: int, hid: int) -> torch.Tensor:
        """keep bits [B, hid/32] of hidden dropout layer j (hop h layer i: j = h (ff-1) + i; project layer i: H (ff-1) + i)."""
        w = hid // 32
        return self.hbits[:max(self.n_hbits, 1) * B * w].view(-1, B, w)[j]

    def hb_all(self, B: int, hid: int) -> torch.Tensor:
        w = hid // 32
        return self.hbits[:self.n_hbits * B * w].view(self.n_hbits, B, w)

    def cb(self, B: int, width: int) -> torch.Tensor:
        return self.catbits[:B * width // 32].view(B, width // 32)


class SIGNStudentTrainer:
    """State + fused step of the SIGN model (``SIGN(in, hidden, n_classes, len(feats), ff_layer, dropout, input_drop)``)."""

    def __init__(self, feats: List[torch.Tensor], n_classes: int, hidden: int = 512, ff_layer: int = 2, dropout: float = 0.5,
                 input_drop: float = 0.1, lr: float = 1e-3, weight_decay: float = 0, alpha: float = 0.9, kd_T: float = 4.0,
                 batch_size: int = 50000, seed: int = 0, gcrd=None):
        """gcrd: a gcrd.SIGNGCRD built for these N nodes and the head width len(feats) * hidden; the step then adds
        beta * G-CRD (see the module docstring) and returns [kd + beta * nce, loss_cls, nce]."""
        if weight_decay != 0:
            raise ValueError("SIGNStudentTrainer: weight_decay != 0 is not supported (sign.py's default is 0)")
        if not feats or any(not isinstance(f, torch.Tensor) or not f.is_cuda for f in feats):
            raise lib.B200GnnError("SIGNStudentTrainer: feats must be CUDA tensors (there is no CPU path)")
        n, F = feats[0].shape
        for f in feats:
            if f.dtype != torch.float32 or f.shape != (n, F) or not f.is_contiguous():
                raise lib.B200GnnError("SIGNStudentTrainer: feats must be contiguous float32 [N, F] matrices of one shape")
        if F % 4 or F > 2048:
            raise lib.B200GnnError(f"SIGNStudentTrainer: input width {F} must be a multiple of 4, at most 2048")
        if hidden % 32 or not 0 < hidden <= 512:
            raise lib.B200GnnError(f"SIGNStudentTrainer: hidden={hidden} must be a multiple of 32, at most 512")
        if n_classes % 4 or not 0 < n_classes <= 512:
            raise lib.B200GnnError(f"SIGNStudentTrainer: n_classes={n_classes} must be a multiple of 4, at most 512")
        if ff_layer < 1 or len(feats) > 16 or batch_size < 1 or not 0 <= dropout < 1 or not 0 <= input_drop < 1:
            raise ValueError("SIGNStudentTrainer: ff_layer >= 1, at most 16 hops, batch_size >= 1, dropout rates in [0, 1)")
        if gcrd is not None:               # refused before any device work
            if gcrd.H != len(feats) * hidden:
                raise ValueError(f"gcrd=: the student head is built for width {gcrd.H}, model.out_feat is "
                                 f"{len(feats)} hops x {hidden} = {len(feats) * hidden} wide")
            if gcrd.N != n:
                raise ValueError(f"gcrd=: the teacher features have {gcrd.N} rows, the hop features {n}")
        self.gcrd = gcrd
        self.device = feats[0].device
        self.feats = list(feats)
        self.N, self.F, self.H, self.hidden, self.C, self.ff = n, F, len(feats), hidden, n_classes, ff_layer
        self.p, self.p_in = float(dropout), float(input_drop)
        self.lr, self.alpha, self.kd_T = float(lr), float(alpha), float(kd_T)
        self.batch_size, self.seed = int(batch_size), int(seed)
        # Philox offsets of one step: H input masks, (H + 1)(ff - 1) hidden layers, the concatenation
        self.D = self.H + (self.H + 1) * (ff_layer - 1) + 1
        H, hid, C, ff = self.H, hidden, n_classes, ff_layer
        dev = self.device

        # ---- flat parameters: weights stored [in, out] (the wgrad GEMM's layout; nn.Linear's [out, in] in state_dict)
        dims_h = [F] + [hid] * ff
        dims_p = [H * hid] + [hid] * (ff - 1) + [C]
        shapes = []
        for h in range(H):
            for i in range(ff):
                shapes.append((f"h{h}.W{i}", (dims_h[i], dims_h[i + 1])))
                if i < ff - 1:
                    shapes.append((f"h{h}.b{i}", (hid,)))
        shapes.append(("hb_last", (H, hid)))               # last-layer biases of all hops: one column sum of dZcat
        for i in range(ff):
            shapes.append((f"p.W{i}", (dims_p[i], dims_p[i + 1])))
            shapes.append((f"p.b{i}", (dims_p[i + 1],)))
        # the slopes last: every matrix above starts 16-byte aligned (the GEMMs' TMA operands)
        if ff > 1:
            shapes.append(("h_slope", (H,)))
            shapes.append(("p_slope", (1,)))
        shapes.append(("slope", (1,)))
        self.store = FlatParams([s for _, s in shapes], dev).attach(self)
        self.P: Dict[str, torch.Tensor] = {}
        self.G: Dict[str, torch.Tensor] = {}
        for (name, _), (p, g) in zip(shapes, self.store.views):
            self.P[name], self.G[name] = p, g
        # tf32 (hi, lo) splits: the input-gradient GEMMs read every weight in its stored layout (one launch over the flat
        # buffer); the forward GEMMs read Wᵀ, split per layer
        self._split_hi = torch.empty_like(self.params)
        self._split_lo = torch.empty_like(self.params)
        self._fsplit = {name: (torch.empty(s[1], s[0], device=dev), torch.empty(s[1], s[0], device=dev))
                        for name, s in shapes if ".W" in name}
        wg = [(F, hid), (hid, hid), (hid, C), (H * hid if H * hid <= 2048 else ops.WGRAD_PRELU_BLOCK, hid if ff > 1 else C)]
        self.wgrad_ws = torch.empty(max(ops.wgrad_workspace_floats(a, b) for a, b in wg), device=dev)
        self.reset_parameters(seed)

        self._tr = _Acts(self, self.batch_size, train=True)
        self._ev: Optional[_Acts] = None
        self.slope_part = torch.empty(ops.gemm_stat_slots(self.batch_size, H * hid), dtype=torch.float64, device=dev)
        self.cs_part = torch.empty(int(lib.load().b200gnn_col_sum_ld_slots(self.batch_size)) * H * hid, device=dev)
        self.kd_part = torch.empty(2 * int(lib.load().b200gnn_kd_partials(self.batch_size)), device=dev)
        self._side = torch.cuda.Stream(device=dev)
        self._ev_fork, self._ev_bits = torch.cuda.Event(), torch.cuda.Event()
        self._B = 0                        # rows of the last training forward
        self._slope_fwd = torch.empty(1, device=dev)   # the model slope that forward used (Adam moves P["slope"] after it)
        self._feat_stale = False
        self._graphs: Dict[int, torch.cuda.CUDAGraph] = {}
        self._idx_static = torch.zeros(self.batch_size, dtype=torch.int64, device=dev)
        self._graph_inputs = None
        self.epoch = 0

    # ------------------------------------------------------------------ parameters
    def _linears(self):
        """(stored-weight key, bias key or None, reference key prefix) of every Linear."""
        out = []
        for h in range(self.H):
            for i in range(self.ff):
                out.append((f"h{h}.W{i}", f"h{h}.b{i}" if i < self.ff - 1 else None, f"inception_ffs.{h}.layers.{i}"))
        for i in range(self.ff):
            out.append((f"p.W{i}", f"p.b{i}", f"project.layers.{i}"))
        return out

    def _bias(self, key: Optional[str], h: int) -> torch.Tensor:
        return self.P[key] if key is not None else self.P["hb_last"][h]

    def reset_parameters(self, seed: int = 0):
        """FeedForwardNet.reset_parameters (sign.py:122-126): xavier_uniform_(gain=calculate_gain('relu')), zero bias;
        nn.PReLU's slope 0.25.  Seeded on the CPU."""
        g = torch.Generator().manual_seed(seed)
        for wk, bk, _ in self._linears():
            fan_in, fan_out = self.P[wk].shape
            bound = math.sqrt(2.0) * math.sqrt(6.0 / (fan_in + fan_out))
            self.P[wk].copy_(((torch.rand(fan_out, fan_in, generator=g) * 2 - 1) * bound).t())
        self.P["hb_last"].zero_()
        for k in self.P:
            if ".b" in k:
                self.P[k].zero_()
            elif "slope" in k:
                self.P[k].fill_(0.25)
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_count.zero_()

    def _to_ref(self, src: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        sd = {}
        for wk, bk, ref in self._linears():
            sd[f"{ref}.weight"] = src[wk].t().contiguous()
            h = int(wk[1:wk.index(".")]) if wk.startswith("h") else 0
            sd[f"{ref}.bias"] = (src[bk] if bk is not None else src["hb_last"][h]).clone()
        if self.ff > 1:
            for h in range(self.H):
                sd[f"inception_ffs.{h}.prelu.weight"] = src["h_slope"][h:h + 1].clone()
            sd["project.prelu.weight"] = src["p_slope"].clone()
        sd["prelu.weight"] = src["slope"].clone()
        return sd

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys and layouts of the reference's SIGN module (nn.Linear weights [out, in], PReLU weights [1])."""
        return self._to_ref(self.P)

    def grad_dict(self) -> Dict[str, torch.Tensor]:
        """The last step's parameter gradients under the state_dict keys and layouts."""
        return self._to_ref(self.G)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for wk, bk, ref in self._linears():
            self.P[wk].copy_(sd[f"{ref}.weight"].t())
            h = int(wk[1:wk.index(".")]) if wk.startswith("h") else 0
            self._bias(bk, h).copy_(sd[f"{ref}.bias"])
        if self.ff > 1:
            for h in range(self.H):
                self.P["h_slope"][h:h + 1].copy_(sd[f"inception_ffs.{h}.prelu.weight"])
            self.P["p_slope"].copy_(sd["project.prelu.weight"])
        self.P["slope"].copy_(sd["prelu.weight"])

    # ------------------------------------------------------------------ forward / backward
    def _slope(self, h: Optional[int]) -> torch.Tensor:
        """PReLU slope of hop h's FFN (h = None: the project FFN)."""
        return self.P["p_slope"] if h is None else self.P["h_slope"][h:h + 1]

    def _gslope(self, h: Optional[int]) -> torch.Tensor:
        return self.G["p_slope"] if h is None else self.G["h_slope"][h:h + 1]

    def _fw(self, key: str):
        hi, lo = self._fsplit[key]
        return ops.split_tf32(self.P[key], transpose=True, hi=hi, lo=lo)

    def _bw(self, key: str):
        """(hi, lo) of the stored [in, out] weight: the B operand of the input-gradient GEMM."""
        return self.store.like(self._split_hi, self.P[key]), self.store.like(self._split_lo, self.P[key])

    def _forward(self, a: _Acts, idx: torch.Tensor, training: bool, y=None, teacher=None) -> torch.Tensor:
        B, H, hid, ff = idx.numel(), self.H, self.hidden, self.ff
        p = self.p if training else 0.0
        if training:
            # the keep bits need no input: drawn on the side stream next to the gather, joined before the first reader
            self._ev_fork.record(torch.cuda.current_stream())
            self._side.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side):
                if a.n_hbits:
                    ops.dropout_bits(a.hb_all(B, hid), p, self.seed, H, step_dev=self.step_count, step_mul=self.D, K=hid)
                ops.dropout_bits(a.catbits[:B * H * hid // 32].view(1, B * H, hid // 32), p, self.seed, H + a.n_hbits,
                                 step_dev=self.step_count, step_mul=self.D, K=hid)
            self._ev_bits.record(self._side)
        ops.sign_gather(self.feats, idx, self.p_in if training else 0.0, self.seed, 0, a.xall(B),
                        step_dev=self.step_count if training else None, step_mul=self.D if training else 0,
                        labels=y, labels_out=a.labels[:B] if y is not None else None,
                        teacher=teacher, teacher_out=a.teacher[:B] if teacher is not None else None)
        if training:
            self._slope_fwd.copy_(self.P["slope"])
            torch.cuda.current_stream().wait_event(self._ev_bits)
        Zcat = a.Zcat[:B]
        for h in range(H):
            for i in range(ff):
                wk = f"h{h}.W{i}"
                dst = Zcat[:, h * hid:(h + 1) * hid] if i == ff - 1 else a.Zh[h][i][:B]
                bias = self._bias(f"h{h}.b{i}" if i < ff - 1 else None, h)
                if i == 0:
                    ops.gemm_tf32x3_rows(a.xall(B)[h], *self._fw(wk), out=dst, bias=bias)
                else:
                    ops.gemm_tf32x3_prelu(a.Zh[h][i - 1][:B], self._slope(h), a.hb(B, h * (ff - 1) + i - 1, hid), p, *self._fw(wk),
                                          bias=bias, out=dst)
        for i in range(ff):
            dst = a.logits[:B] if i == ff - 1 else a.Zp[i][:B]
            if i == 0:
                ops.gemm_tf32x3_prelu(Zcat, self.P["slope"], a.cb(B, H * hid), p, *self._fw("p.W0"), bias=self.P["p.b0"], out=dst)
            else:
                ops.gemm_tf32x3_prelu(a.Zp[i - 1][:B], self._slope(None), a.hb(B, H * (ff - 1) + i - 1, hid), p,
                                      *self._fw(f"p.W{i}"), bias=self.P[f"p.b{i}"], out=dst)
        return a.logits[:B]

    def _backward(self, B: int, d_out_feat: Optional[torch.Tensor], d_cat_stored: bool = False):
        """d_out_feat: the auxiliary loss's gradient of out_feat, copied into dZcat; d_cat_stored: the G-CRD head has stored
        it there already.  Either is the starting value of the project FFN's first input-gradient GEMM's accumulate."""
        a, H, hid, ff, p = self._tr, self.H, self.hidden, self.ff, self.p
        ops.split_tf32(self.params.view(1, -1), hi=self._split_hi.view(1, -1), lo=self._split_lo.view(1, -1))
        Zcat, dZcat = a.Zcat[:B], a.dZcat[:B]
        if d_out_feat is not None:
            dZcat.copy_(d_out_feat)          # the auxiliary loss's gradient: the starting value of the epilogue's accumulate
        for i in range(ff - 1, -1, -1):       # project FFN
            G = a.dlogits[:B] if i == ff - 1 else a.dZp[i][:B]
            ops.col_sum_ld(G, out=self.G[f"p.b{i}"], partial=self.cs_part)
            if i == 0:
                X, slope, bits, gslope = Zcat, self.P["slope"], a.cb(B, H * hid), self.G["slope"]
                dst, acc, sacc = dZcat, d_out_feat is not None or d_cat_stored, False
            else:
                X, slope, bits, gslope = a.Zp[i - 1][:B], self._slope(None), a.hb(B, H * (ff - 1) + i - 1, hid), self._gslope(None)
                dst, acc, sacc = a.dZp[i - 1][:B], False, i != ff - 1
            ops.gemm_wgrad_tf32x3_prelu(X, slope, bits, p, G, out=self.G[f"p.W{i}"], workspace=self.wgrad_ws)
            ops.gemm_tf32x3_prelu_bwd(G, *self._bw(f"p.W{i}"), out=dst, z=X, bits=bits, slope=slope, p=p, slope_grad=gslope,
                                      partial=self.slope_part, accumulate=acc, slope_accumulate=sacc)
        ops.col_sum_ld(dZcat, out=self.G["hb_last"].view(-1), partial=self.cs_part)
        for h in range(H):                    # hop FFNs
            for i in range(ff - 1, -1, -1):
                G = dZcat[:, h * hid:(h + 1) * hid] if i == ff - 1 else a.dZh[h][i][:B]
                if i < ff - 1:
                    ops.col_sum_ld(G, out=self.G[f"h{h}.b{i}"], partial=self.cs_part)
                if i == 0:
                    ops.gemm_wgrad_tf32x3_rows(a.xall(B)[h], G, out=self.G[f"h{h}.W0"], workspace=self.wgrad_ws)
                    continue
                Z, bits = a.Zh[h][i - 1][:B], a.hb(B, h * (ff - 1) + i - 1, hid)
                ops.gemm_wgrad_tf32x3_prelu(Z, self._slope(h), bits, p, G, out=self.G[f"h{h}.W{i}"], workspace=self.wgrad_ws)
                ops.gemm_tf32x3_prelu_bwd(G, *self._bw(f"h{h}.W{i}"), out=a.dZh[h][i - 1][:B], z=Z, bits=bits, slope=self._slope(h),
                                          p=p, slope_grad=self._gslope(h), partial=self.slope_part, slope_accumulate=i != ff - 1)

    def _check_batch(self, idx: torch.Tensor, sample=None):
        if not isinstance(idx, torch.Tensor) or not idx.is_cuda or idx.dtype != torch.int64 or idx.dim() != 1:
            raise lib.B200GnnError("batch indices: expected a CUDA int64 vector")
        if not 0 < idx.numel() <= self.batch_size:
            raise ValueError(f"batch of {idx.numel()} rows: expected 1..{self.batch_size}")
        if self.gcrd is not None:
            self.gcrd.check_batch(idx.numel(), sample)

    def _check_aux(self, aux, sample=None):
        if aux is not None and self.gcrd is not None:
            raise ValueError("aux= and the trainer's gcrd= objective are two auxiliary losses; pass one")
        if sample is not None and self.gcrd is None:
            raise ValueError("sample= is the G-CRD row sample; this trainer has no gcrd= objective")

    def _step_impl(self, idx, y, teacher_logits, aux=None, beta: float = 1.0, sample=None):
        B = idx.numel()
        a = self._tr
        logits = self._forward(a, idx, True, y, teacher_logits)
        ops.kd_loss_fwd_bwd(logits, a.labels[:B], None, a.teacher[:B] if teacher_logits is not None else None, self.alpha,
                            self.kd_T, d_logits=a.dlogits[:B], loss_out=self.loss_out, partial=self.kd_part)
        self._B, self._feat_stale = B, True
        d_feat, g = None, self.gcrd
        if g is not None:
            g.forward_backward(self, idx, a.Zcat[:B], self.P["slope"], a.cb(B, self.H * self.hidden), self.p, a.dZcat[:B],
                               sample)
            self.loss_out[2].copy_(g.loss_aux[0])
        elif aux is not None:
            d_feat, self.loss_aux = aux_grad(self.out_feat(), aux, beta)
        self._backward(B, d_feat, d_cat_stored=g is not None)
        self.store.adam(self.lr)
        if g is not None:
            g.optimizer_step(self.lr)
        if aux is not None:
            self.loss_out[0].add_(self.loss_aux * beta)

    def train_step(self, batch_idx: torch.Tensor, y: torch.Tensor, teacher_logits: Optional[torch.Tensor] = None, aux=None,
                   beta: float = 1.0, sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One iteration of ``train_kd_and_aux`` (sign.py:293-373) on the nodes ``batch_idx`` (CUDA int64): cross-entropy
        without a teacher, kd_criterion with ``teacher_logits`` ([N, C], gathered in the step).  ``aux(out_feat)`` receives
        the batch's [B, hops*hidden] ``model.out_feat`` (requires_grad) and returns an auxiliary loss that enters as
        kd + beta*aux; heads inside it keep their gradients in the caller's autograd.  Returns the device tensor
        [loss, loss_cls, loss_kd] (beta*aux folded into loss); no host sync.  With the trainer's gcrd= objective it returns
        [loss + beta * nce, loss_cls, nce], and ``sample`` (positions into the batch, [S]) replaces its on-device draw."""
        self._check_aux(aux, sample)
        self._check_batch(batch_idx, sample)
        if self.gcrd is not None:
            self.gcrd.prepare([batch_idx.numel()])
        self._step_impl(batch_idx, y, teacher_logits, aux, beta, sample)
        return self.loss_out

    def out_feat(self) -> torch.Tensor:
        """The last training step's ``model.out_feat`` = dropout(prelu(cat)), [B, hops*hidden], materialised on first read."""
        a, B = self._tr, self._B
        if self._feat_stale:
            self._feat_stale = False
            ops.prelu_bits(a.Zcat[:B], a.cb(B, self.H * self.hidden), self._slope_fwd, self.p, out=a.out_feat[:B])
        return a.out_feat[:B]

    def logits(self) -> torch.Tensor:
        return self._tr.logits[:self._B]

    # ------------------------------------------------------------------ epochs, graphs, inference
    def epoch_order(self, train_idx: torch.Tensor, epoch: int) -> torch.Tensor:
        """The training nodes in the epoch's shuffled order: a permutation drawn on the device from (seed, epoch)."""
        g = torch.Generator(device=self.device)
        g.manual_seed((self.seed * 1_000_003 + epoch) & 0x7FFFFFFFFFFFFFFF)
        return train_idx[torch.randperm(train_idx.numel(), generator=g, device=self.device)]

    def train_epoch(self, train_idx: torch.Tensor, y: torch.Tensor, teacher_logits: Optional[torch.Tensor] = None, aux=None,
                    beta: float = 1.0, epoch: Optional[int] = None) -> torch.Tensor:
        """One pass of sign.py's train loop: the batches of DataLoader(train_idx, batch_size, shuffle=True,
        drop_last=False) (same sizes, every node once) in a device-drawn order.  Captured batch sizes replay their graph.
        Returns the per-step losses [n_steps, 3] (device, no sync)."""
        self._check_aux(aux)
        n, bs = train_idx.numel(), self.batch_size
        sizes = [min(bs, n - s) for s in range(0, n, bs)]
        if self.gcrd is not None:          # every batch is checked (the ragged last one too) before the first step runs
            for B in set(sizes):
                self.gcrd.check_batch(B)
            self.gcrd.prepare(sizes)
        epoch = self.epoch if epoch is None else int(epoch)
        self.epoch = epoch + 1
        order = self.epoch_order(train_idx, epoch)
        losses = []
        gi = self._graph_inputs
        graphs_ok = aux is None and gi is not None and gi[0] is y and gi[1] is teacher_logits
        for s in range(0, order.numel(), self.batch_size):
            b = order[s:s + self.batch_size]
            if graphs_ok and b.numel() in self._graphs:
                losses.append(self.replay(b).clone())
            else:
                losses.append(self.train_step(b, y, teacher_logits, aux, beta).clone())
        return torch.stack(losses)

    def capture(self, batch_sizes, y: torch.Tensor, teacher_logits: Optional[torch.Tensor] = None):
        """Capture one CUDA graph of the step per batch size (the batch indices are read from a static buffer).  The
        warm-up steps run on a copy of the optimiser state (and of the gcrd= heads' state), which is restored: capturing
        does not train."""
        sizes = sorted(set(int(b) for b in batch_sizes))
        g = self.gcrd
        if g is not None:
            for B in sizes:
                g.check_batch(B)
            g.prepare(sizes)
        heads = g.preserved() if g is not None else contextlib.nullcontext()
        with self.store.preserved(), heads:
            for B in sizes:
                idx = self._idx_static[:B]
                self._graphs[B] = capture_graph(lambda: self._step_impl(idx, y, teacher_logits), warmup=1)
        self._graph_inputs = (y, teacher_logits)
        self._feat_stale = False
        return self

    def replay(self, batch_idx: torch.Tensor) -> torch.Tensor:
        B = batch_idx.numel()
        self._idx_static[:B].copy_(batch_idx)
        self._graphs[B].replay()
        self._B, self._feat_stale = B, True
        if self.gcrd is not None:
            self.gcrd._last = self.gcrd.row_sets[B]
        return self.loss_out

    @torch.no_grad()
    def predict(self, batch_size: int = 100000) -> torch.Tensor:
        """Eval-mode logits of all N nodes (sign.py:385-401): no dropout, PReLU only, the training kernels."""
        rows = min(int(batch_size), self.N)
        if self._ev is None or self._ev.rows != rows:
            self._ev = _Acts(self, rows, train=False)
        out = torch.empty(self.N, self.C, device=self.device)
        for s in range(0, self.N, rows):
            idx = torch.arange(s, min(s + rows, self.N), device=self.device)
            out[s:s + idx.numel()].copy_(self._forward(self._ev, idx, False))
        return out

    def useful_flop(self, B: int) -> int:
        """Multiply-adds x 2 of one training step's dense contractions (forward, input and weight gradients)."""
        H, F, hid, C, ff = self.H, self.F, self.hidden, self.C, self.ff
        dims_h = [F] + [hid] * ff
        dims_p = [H * hid] + [hid] * (ff - 1) + [C]
        fwd = H * sum(dims_h[i] * dims_h[i + 1] for i in range(ff)) + sum(dims_p[i] * dims_p[i + 1] for i in range(ff))
        dgrad = fwd - H * dims_h[0] * dims_h[1]          # no input gradient of the features
        return 2 * B * (2 * fwd + dgrad)
