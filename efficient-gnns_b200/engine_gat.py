"""Fused full-batch training step for the reference's DGL ``GAT`` model — BASELINE.json configs[3].

The model is ``GAT`` of arxiv_dgl/models.py:239-313 built from its ``GATConv`` (:95-236): hidden layers of ``n_heads`` heads
of ``n_hidden``, a last layer of one head of ``n_classes``, residual everywhere, BatchNorm1d -> ReLU -> dropout after every
hidden layer, ``input_drop`` on the features, ``bias_last``.  One layer of the step:

    [ft | res] = h [W_fc | W_res]          one 3xTF32 GEMM; h is formed in its registers from the layer below's pre-BatchNorm
                                           output, scale / shift and keep bits (layer 0: x under the input-drop bits)
    el, er     = gat_scores(ft)            one read of ft; el carries out_deg^-1/2, er the raw projection
    a          = edge_softmax(el, er)      with the edge-drop keep mask
    Y          = in_deg^1/2 · Σ a·out_deg^-1/2[src]·ft[src] + res   gat_aggregate_epi: the per-source scale vector in the
                                           coefficient, residual and BatchNorm partial sums (last layer: bias_last) in the epilogue

so a hidden layer writes two [N, ·] tensors ([ft | res] and Y) and the [nnz, H] coefficients.  The backward is hand-written
from the same kernels (gat_bwd_rows, the aggregation on the transposed graph with the two scale vectors exchanged,
segment_sum_heads, gat_scores_bwd, the input-gradient GEMMs with the BatchNorm-backward reduction in the epilogue where their
width allows, weight gradients on a side stream); Adam runs over one flat parameter buffer and the supervised / KD step is
captured into one CUDA graph.

Head widths are stored with a padded stride Dp (a multiple of 4 with H·Dp a multiple of 32: the aggregation moves 128-bit
vectors inside a head, the keep bits and the GEMM epilogues work on 32-column chunks).  Padded weight columns / rows and
attention entries are zero, stay exactly zero through BatchNorm and Adam, and never appear in state_dict() or out_feat().
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from . import lib, ops
from .nn import _csr2csc_i32, _hub_args
from .sparse import SparseTensor
from .trainer import FlatParams, FullBatchStudent

WGRAD_BLOCK = 512          # widest output block of one weight-gradient launch


def padded_head(H: int, D: int, hidden: bool = True) -> int:
    """Stored head stride: the smallest multiple of 4 >= D, for a hidden layer with H * stride a multiple of 32."""
    Dp = (D + 3) // 4 * 4
    while hidden and (H * Dp) % 32:
        Dp += 4
    return Dp


class GATTrainer(FullBatchStudent):
    """State + fused step of the reference's GAT on one GPU (adj rows = destinations, bidirected with self-loops)."""

    def __init__(self, adj: SparseTensor, in_feats: int, n_classes: int, n_hidden: int, n_layers: int, n_heads: int,
                 dropout: float = 0.0, input_drop: float = 0.0, edge_drop: float = 0.0, use_attn_dst: bool = True,
                 use_symmetric_norm: bool = False, lr: float = 0.002, seed: int = 0, alpha: float = 0.9, T: float = 4.0,
                 attn_drop: float = 0.0, negative_slope: float = 0.2, bn_eps: float = 1e-5, bn_momentum: float = 0.1,
                 step_streams: Optional[int] = None):
        """step_streams: Philox offsets one training step spans (default 2 * n_layers, one forward's streams); a recipe that
        runs several training forwards per step passes more and draws forward f at stream base f * 2 * n_layers."""
        assert adj.is_cuda(), "the engine runs on a CUDA device"
        if attn_drop != 0.0:
            raise ValueError("attn_drop > 0 is not implemented (every reference configuration passes 0)")
        if n_layers < 2:
            raise ValueError("GATTrainer needs at least one hidden layer")
        if in_feats % 4:
            raise ValueError("in_feats must be a multiple of 4 (128-bit rows)")
        st = adj.storage
        if bool((st.rowcount() == 0).any()):
            raise ValueError("zero in-degree rows: add self-loops (the reference asserts, arxiv_dgl/models.py:156-158)")
        self.device = dev = adj.device
        self.N, self.L, self.H = adj.size(0), int(n_layers), int(n_heads)
        self.in_feats, self.n_classes, self.n_hidden = int(in_feats), int(n_classes), int(n_hidden)
        self.p, self.p_in, self.p_edge = float(dropout), float(input_drop), float(edge_drop)
        self.use_attn_dst, self.sym = bool(use_attn_dst), bool(use_symmetric_norm)
        self.lr, self.seed, self.alpha, self.kd_T = float(lr), int(seed), float(alpha), float(T)
        self.slope, self.bn_eps, self.bn_momentum = float(negative_slope), bn_eps, bn_momentum
        N, L = self.N, self.L
        self.step_mul = 2 * L if step_streams is None else int(step_streams)

        self.G = st.engine_csr_unweighted() if st.value() is None else st.engine_csr()
        self.Gt = st.engine_csc("value")
        self.perm = _csr2csc_i32(st)
        self.nnz = self.G.nnz
        # per layer: heads, true / stored head width, stored output width, stored input width
        self.Hl = [self.H] * (L - 1) + [1]
        self.Dl = [self.n_hidden] * (L - 1) + [self.n_classes]
        self.Dp = [padded_head(h, d, l < L - 1) for l, (h, d) in enumerate(zip(self.Hl, self.Dl))]
        self.K = [h * d for h, d in zip(self.Hl, self.Dp)]
        self.Kin = [self.in_feats] + self.K[:-1]
        if max(self.K) > 1536 or self.H > 16:
            raise ValueError("heads * padded head width must be <= 1536 and heads <= 16")
        self.blocks = [[(c, min(WGRAD_BLOCK, k - c)) for c in range(0, k, WGRAD_BLOCK)] for k in self.K]
        if self.sym:
            self.src_scale = torch.bincount(st.col(), minlength=adj.size(1)).float().clamp(min=1).pow(-0.5).contiguous()
            self.dst_scale = st.rowcount().float().clamp(min=1).pow(0.5).contiguous()
            # gat_bwd_rows chains d a through the constant the aggregation multiplied a by: out_deg^-1/2[src]·in_deg^1/2[dst]
            es = (self.src_scale[st.col()] * self.dst_scale[st.row()]).view(-1, 1)
            self.edge_scale = {h: es.expand(-1, h).contiguous() for h in set(self.Hl)}
        else:
            self.src_scale = self.dst_scale = None
            self.edge_scale = {h: None for h in set(self.Hl)}

        # ---- flat parameters: per layer the column blocks of W_fc and W_res ([in, block], so that a weight gradient is one
        # contiguous output), attn_l, attn_r, BatchNorm gamma / beta; bias_last at the end
        shapes = []
        for l in range(L):
            shapes += [(self.Kin[l], nb) for _ in range(2) for _, nb in self.blocks[l]]
            shapes += [(self.K[l],)] * ((2 if self.use_attn_dst else 1) + (2 if l < L - 1 else 0))
        shapes.append((self.K[-1],))
        self.store = FlatParams(shapes, dev).attach(self)
        views = iter(self.store.views)
        self.Wfc, self.Wres, self.gWfc, self.gWres = [], [], [], []
        self.attn_l, self.attn_r, self.g_attn_l, self.g_attn_r = [], [], [], []
        self.gamma, self.beta, self.ggamma, self.gbeta = [], [], [], []
        for l in range(L):
            for W, gW in ((self.Wfc, self.gWfc), (self.Wres, self.gWres)):
                pairs = [next(views) for _ in self.blocks[l]]
                W.append([p for p, _ in pairs]); gW.append([g for _, g in pairs])
            a, ga = next(views)
            self.attn_l.append(a); self.g_attn_l.append(ga)
            a, ga = next(views) if self.use_attn_dst else (None, None)
            self.attn_r.append(a); self.g_attn_r.append(ga)
            if l < L - 1:
                (g, gg), (b, gb) = next(views), next(views)
                self.gamma.append(g); self.ggamma.append(gg); self.beta.append(b); self.gbeta.append(gb)
        self.bias_last, self.g_bias_last = next(views)
        # tf32 hi / lo splits, refreshed every step: [W_fc | W_res]^T stacked [2K, in] feeds the forward GEMM, the blocks as
        # stored ([in, block]) feed the input-gradient GEMMs
        self.Wt_split = [tuple(torch.empty(2 * self.K[l], self.Kin[l], device=dev) for _ in range(2)) for l in range(L)]
        self.W_split = [[[tuple(torch.empty(self.Kin[l], nb, device=dev) for _ in range(2)) for _, nb in self.blocks[l]]
                         for _ in range(2)] if l > 0 else None for l in range(L)]
        self.wgrad_ws = torch.empty(max(ops.wgrad_workspace_floats(self.Kin[l], nb) for l in range(L) for _, nb in self.blocks[l]),
                                    device=dev)
        Kh = self.K[0]
        self.running_mean = [torch.zeros(Kh, device=dev) for _ in range(L - 1)]
        self.running_var = [torch.ones(Kh, device=dev) for _ in range(L - 1)]
        self.reset_parameters(seed)

        # ---- activations / gradients (preallocated; CUDA-graph friendly)
        self.cat = [torch.zeros(N, 2 * k, device=dev) for k in self.K]           # [ft | res]
        self.Y = [torch.zeros(N, k, device=dev) for k in self.K]                 # pre-BatchNorm output (last: logits)
        self.dY = [torch.zeros(N, k, device=dev) for k in self.K]                # d Y = d res; also the input-gradient target
        self.dft = [torch.zeros(N, k, device=dev) for k in self.K]
        self.el = [torch.zeros(N, h, device=dev) for h in self.Hl]
        self.er = [torch.zeros(N, h, device=dev) if self.use_attn_dst else None for h in self.Hl]
        self.d_el = [torch.zeros(N, h, device=dev) for h in self.Hl]
        self.d_er = [torch.zeros(N, h, device=dev) if self.use_attn_dst else None for h in self.Hl]
        self.a = [torch.zeros(self.nnz, h, device=dev) for h in self.Hl]
        self.dpre = [torch.zeros(self.nnz, h, device=dev) for h in self.Hl]
        self.stat_part = [torch.empty(ops.gat_stat_slots(self.G), 2, Kh, device=dev) for _ in range(L - 1)]
        self.bn = [torch.empty(4, Kh, device=dev) for _ in range(L - 1)]          # mean, invstd, scale, shift
        self.bn_eval = [torch.empty(2, Kh, device=dev) for _ in range(L - 1)]
        self.score_part = torch.empty(ops.gat_scores_slots(N), 2, max(self.K), device=dev)
        self.rs = ops.rows_slots(N)
        self.row_part = torch.empty(self.rs, 2, max(self.K), device=dev)
        self.coef = torch.empty(3, Kh, device=dev)
        # the BatchNorm-backward reduction rides in the epilogue of the last input-gradient GEMM where the width allows;
        # wider layers materialise the activation once for the unfused backward pass
        self.fuse_bnbwd = ops.gemm_stats_supported(Kh)
        self.gemm_part = torch.empty(ops.gemm_stat_slots(N, Kh), 2, Kh, device=dev) if self.fuse_bnbwd else None
        self.A_mat = None if self.fuse_bnbwd else torch.empty(N, Kh, device=dev)
        words = Kh // 32
        self.keep_bits = torch.full((L - 1, N, words), -1, dtype=torch.int32, device=dev)
        self.ones_bits = torch.full((N, words), -1, dtype=torch.int32, device=dev)
        self.in_bits = torch.full((1, N, (self.in_feats + 31) // 32), -1, dtype=torch.int32, device=dev)
        self.one = torch.ones(1, device=dev)                                       # PReLU slope 1: "dropout only"
        self.edge_keep = [torch.ones((self.nnz + 3) // 4 * 4, dtype=torch.uint8, device=dev) for _ in range(L)]
        self.kd_part = torch.empty(2 * int(lib.load().b200gnn_kd_partials(N)), device=dev)
        self._side = torch.cuda.Stream(device=dev)
        self._ev_fork, self._ev_join, self._ev_bits = torch.cuda.Event(), torch.cuda.Event(), torch.cuda.Event()
        self._static: Dict[str, torch.Tensor] = {}
        self._training = False

    # ------------------------------------------------------------------ parameters
    def _cols(self, l: int) -> torch.Tensor:
        """Stored column of every true output column of layer l."""
        h = torch.arange(self.Hl[l], device=self.device).view(-1, 1)
        return (h * self.Dp[l] + torch.arange(self.Dl[l], device=self.device).view(1, -1)).reshape(-1)

    def _store(self, blocks: List[torch.Tensor], l: int, w: torch.Tensor):
        """w: reference weight [H*D, in_true] -> the [in_stored, block] column blocks, padding zero."""
        full = torch.zeros(self.Kin[l], self.K[l], device=self.device)
        rows = self._cols(l - 1) if l > 0 else torch.arange(self.in_feats, device=self.device)
        full[rows.view(-1, 1), self._cols(l).view(1, -1)] = w.to(self.device, torch.float32).t()
        for (c0, nb), blk in zip(self.blocks[l], blocks):
            blk.copy_(full[:, c0:c0 + nb])

    def _load_vec(self, dst: torch.Tensor, l: int, v: torch.Tensor, fill: float = 0.0):
        dst.fill_(fill)
        dst[self._cols(l)] = v.to(self.device, torch.float32).reshape(-1)

    def reset_parameters(self, seed: int = 0):
        """GATConv.reset_parameters (arxiv_dgl/models.py:138-149): xavier-normal, gain sqrt(2); BatchNorm ones / zeros;
        bias_last zero."""
        g = torch.Generator().manual_seed(seed)
        gain = math.sqrt(2.0)

        def xavier(shape, fan_in, fan_out):
            return torch.randn(shape, generator=g) * (gain * math.sqrt(2.0 / (fan_in + fan_out)))
        for l in range(self.L):
            H, D = self.Hl[l], self.Dl[l]
            fin = self.in_feats if l == 0 else self.Hl[l - 1] * self.Dl[l - 1]
            self._store(self.Wfc[l], l, xavier((H * D, fin), fin, H * D))
            self._load_vec(self.attn_l[l], l, xavier((H, D), H * D, D))          # tensor [1, H, D]: fan_in H*D, fan_out D
            if self.use_attn_dst:
                self._load_vec(self.attn_r[l], l, xavier((H, D), H * D, D))
            self._store(self.Wres[l], l, xavier((H * D, fin), fin, H * D))
        for l in range(self.L - 1):
            self.gamma[l].fill_(1.0); self.beta[l].zero_()
            self.running_mean[l].zero_(); self.running_var[l].fill_(1.0)
        self.bias_last.zero_()
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_count.zero_()

    def _export(self, Wfc, Wres, attn_l, attn_r, gamma, beta, bias_last) -> Dict[str, torch.Tensor]:
        """Stored tensors (parameters or their gradients) under the reference's names and shapes, padding removed."""
        sd = {}
        for l in range(self.L):
            rows = self._cols(l - 1) if l > 0 else torch.arange(self.in_feats, device=self.device)
            c = self._cols(l)
            sd[f"convs.{l}.fc.weight"] = torch.cat(Wfc[l], dim=1)[rows][:, c].t().contiguous()
            sd[f"convs.{l}.attn_l"] = attn_l[l][c].view(1, self.Hl[l], self.Dl[l]).clone()
            if self.use_attn_dst:
                sd[f"convs.{l}.attn_r"] = attn_r[l][c].view(1, self.Hl[l], self.Dl[l]).clone()
            sd[f"convs.{l}.res_fc.weight"] = torch.cat(Wres[l], dim=1)[rows][:, c].t().contiguous()
        for l in range(self.L - 1):
            c = self._cols(l)
            sd[f"norms.{l}.weight"] = gamma[l][c].clone(); sd[f"norms.{l}.bias"] = beta[l][c].clone()
        sd["bias_last.bias"] = bias_last[self._cols(self.L - 1)].clone()
        return sd

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys and shapes of the reference's GAT module."""
        sd = self._export(self.Wfc, self.Wres, self.attn_l, self.attn_r, self.gamma, self.beta, self.bias_last)
        for l in range(self.L - 1):
            c = self._cols(l)
            sd[f"norms.{l}.running_mean"] = self.running_mean[l][c].clone()
            sd[f"norms.{l}.running_var"] = self.running_var[l][c].clone()
        return sd

    def named_gradients(self) -> Dict[str, torch.Tensor]:
        """The last backward's parameter gradients under the reference's names."""
        return self._export(self.gWfc, self.gWres, self.g_attn_l, self.g_attn_r, self.ggamma, self.gbeta, self.g_bias_last)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for l in range(self.L):
            self._store(self.Wfc[l], l, sd[f"convs.{l}.fc.weight"])
            self._store(self.Wres[l], l, sd[f"convs.{l}.res_fc.weight"])
            self._load_vec(self.attn_l[l], l, sd[f"convs.{l}.attn_l"])
            if self.use_attn_dst:
                self._load_vec(self.attn_r[l], l, sd[f"convs.{l}.attn_r"])
        for l in range(self.L - 1):
            self._load_vec(self.gamma[l], l, sd[f"norms.{l}.weight"], 1.0)
            self._load_vec(self.beta[l], l, sd[f"norms.{l}.bias"])
            if f"norms.{l}.running_mean" in sd:
                self._load_vec(self.running_mean[l], l, sd[f"norms.{l}.running_mean"])
                self._load_vec(self.running_var[l], l, sd[f"norms.{l}.running_var"], 1.0)
        self._load_vec(self.bias_last, self.L - 1, sd["bias_last.bias"])

    # ------------------------------------------------------------------ forward
    def stream_offset(self, kind: str, layer: int, step: int, fwd: int = 0) -> int:
        """Philox offset of a random stream of training forward ``fwd`` of step ``step``: 'dropout' (hidden layer), 'input',
        'edge' (layer)."""
        base = {"dropout": layer, "input": self.L - 1, "edge": self.L + layer}[kind]
        return base + fwd * 2 * self.L + step * self.step_mul

    def _draw(self, base: int = 0):
        """All keep decisions of the step: they need no input, so they run on the side stream next to the first GEMM.
        base: the first Philox offset of this forward's streams within the step."""
        mul = self.step_mul
        if self.p > 0:
            ops.dropout_bits(self.keep_bits, self.p, self.seed, base, step_dev=self.step_count, step_mul=mul)
        if self.p_in > 0:
            ops.dropout_bits(self.in_bits, self.p_in, self.seed, base + self.L - 1, step_dev=self.step_count, step_mul=mul,
                             K=self.in_feats)
        if self.p_edge > 0:
            for l in range(self.L):
                ops.dropout_mask_step(self.edge_keep[l], self.p_edge, self.seed, base + self.L + l, self.step_count, mul)

    def _act(self, l: int):
        """(Y, scale, shift, keep bits, p) from which the fused kernels form hidden activation l of the last forward."""
        if self._training:
            return self.Y[l], self.bn[l][2], self.bn[l][3], self.keep_bits[l], self.p
        return self.Y[l], self.bn_eval[l][0], self.bn_eval[l][1], self.ones_bits, 0.0

    def forward(self, x: torch.Tensor, training: bool = True, stream_base: int = 0) -> torch.Tensor:
        """Logits [N, n_classes]; training=False uses the running statistics and draws nothing.  stream_base: see _draw."""
        self._training = training
        L_ = lib.load()
        draws = training and (self.p > 0 or self.p_in > 0 or self.p_edge > 0)
        if draws:
            self._ev_fork.record(torch.cuda.current_stream())
            self._side.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side):
                self._draw(stream_base)
                self._ev_bits.record(self._side)
        for l in range(self.L):
            H, K, last = self.Hl[l], self.K[l], l == self.L - 1
            hi, lo = self.Wt_split[l]
            for half, W in enumerate((self.Wfc[l], self.Wres[l])):
                for (c0, nb), blk in zip(self.blocks[l], W):
                    r0 = half * K + c0
                    ops.split_tf32(blk, transpose=True, hi=hi[r0:r0 + nb], lo=lo[r0:r0 + nb])
            if l == 0:
                if draws:
                    torch.cuda.current_stream().wait_event(self._ev_bits)
                if training and self.p_in > 0:
                    ops.gemm_tf32x3_prelu(x, self.one, self.in_bits[0], self.p_in, hi, lo, out=self.cat[0])
                else:
                    ops.gemm_tf32x3(x, hi, lo, out=self.cat[0])
            else:
                y, scale, shift, bits, p = self._act(l - 1)
                ops.gemm_tf32x3_act(y, scale, shift, bits, p, hi, lo, out=self.cat[l])
            ft, res = self.cat[l][:, :K], self.cat[l][:, K:]
            ops.gat_scores(ft, self.attn_l[l], self.attn_r[l], self.src_scale, H, el=self.el[l], er=self.er[l])
            keep = self.edge_keep[l] if training and self.p_edge > 0 else None
            lib.check(L_.b200gnn_gat_edge_softmax_f32(self.G.rowptr.data_ptr(), self.G.col.data_ptr(), self.el[l].data_ptr(),
                                                      None if self.er[l] is None else self.er[l].data_ptr(), self.N, H, self.slope,
                                                      0.0, self.a[l].data_ptr(), None if keep is None else keep.data_ptr(),
                                                      lib.stream_ptr()), "gat_edge_softmax_f32")
            ops.gat_aggregate_epi(self.G, None, self.a[l], ft, self.Y[l], H, src_scale=self.src_scale, row_scale=self.dst_scale,
                                  res=res, bias=self.bias_last if last else None,
                                  stat_partial=self.stat_part[l] if training and not last else None)
            if last:
                break
            if training:
                ops.bn_finalize(self.stat_part[l], self.N, self.gamma[l], self.beta[l], self.bn_eps, self.bn_momentum,
                                self.running_mean[l], self.running_var[l], out=self.bn[l])
            else:
                scale = self.gamma[l] * torch.rsqrt(self.running_var[l] + self.bn_eps)
                self.bn_eval[l][0].copy_(scale); self.bn_eval[l][1].copy_(self.beta[l] - self.running_mean[l] * scale)
        return self.Y[-1][:, :self.n_classes]

    def _hidden(self, l: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Hidden activation l of the last forward, materialised in the stored layout [N, K]."""
        y, scale, shift, bits, p = self._act(l)
        return ops.affine_relu_bits(y, bits, scale, shift, p, out=out)

    def out_feat(self) -> torch.Tensor:
        """The reference's ``model.feat`` (arxiv_dgl/models.py:308): the last hidden activation, [N, n_heads * n_hidden]."""
        a = self._hidden(self.L - 2)
        return a if self.Dp[0] == self.Dl[0] else a[:, self._cols(self.L - 2)].contiguous()

    # ------------------------------------------------------------------ backward
    def _wgrad(self, l: int, x: torch.Tensor):
        """[dW_fc ; dW_res] = h^T [d ft | d res], block by block, straight into the flat gradient buffer."""
        L_, s = lib.load(), lib.stream_ptr()
        N, Kin = self.N, self.Kin[l]
        for G_, gW in ((self.dft[l], self.gWfc[l]), (self.dY[l], self.gWres[l])):
            for (c0, nb), out in zip(self.blocks[l], gW):
                g = G_[:, c0:c0 + nb]
                if l > 0:
                    y, scale, shift, bits, p = self._act(l - 1)
                    rc = L_.b200gnn_gemm_wgrad_tf32x3_act_f32(y.data_ptr(), y.stride(0), g.data_ptr(), g.stride(0), out.data_ptr(), N,
                                                              Kin, nb, scale.data_ptr(), shift.data_ptr(), bits.data_ptr(), p,
                                                              self.wgrad_ws.data_ptr(), s)
                elif self.p_in > 0:
                    rc = L_.b200gnn_gemm_wgrad_tf32x3_prelu_f32(x.data_ptr(), x.stride(0), g.data_ptr(), g.stride(0), out.data_ptr(),
                                                                N, Kin, nb, self.one.data_ptr(), self.in_bits.data_ptr(),
                                                                self.in_bits.shape[2], self.p_in, self.wgrad_ws.data_ptr(), s)
                else:
                    rc = L_.b200gnn_gemm_wgrad_tf32x3_f32(x.data_ptr(), x.stride(0), g.data_ptr(), g.stride(0), out.data_ptr(), N,
                                                          Kin, nb, self.wgrad_ws.data_ptr(), s)
                lib.check(rc, "gemm_wgrad_tf32x3")

    def _dgrad(self, l: int, seeded: bool):
        """dY[l-1] (the gradient at hidden activation l-1) (+)= [d ft | d res] [W_fc | W_res]^T; the last GEMM stores
        dz and reduces the BatchNorm-backward column sums where its width allows."""
        L_, s = lib.load(), lib.stream_ptr()
        N, Kin = self.N, self.Kin[l]
        out = self.dY[l - 1]
        jobs = []
        for half, (G_, W) in enumerate(((self.dY[l], self.Wres[l]), (self.dft[l], self.Wfc[l]))):
            for b, ((c0, nb), blk) in enumerate(zip(self.blocks[l], W)):
                hi, lo = self.W_split[l][half][b]
                ops.split_tf32(blk, transpose=False, hi=hi, lo=lo)
                jobs.append((G_[:, c0:c0 + nb], hi, lo, nb))
        for i, (g, hi, lo, nb) in enumerate(jobs):
            acc = seeded or i > 0
            if i == len(jobs) - 1 and self.fuse_bnbwd:
                y, scale, shift, bits, p = self._act(l - 1)
                rc = L_.b200gnn_gemm_tf32x3_bnbwd_bits_f32(g.data_ptr(), g.stride(0), hi.data_ptr(), lo.data_ptr(), nb, out.data_ptr(),
                                                           Kin, N, Kin, nb, int(acc), bits.data_ptr(), y.data_ptr(),
                                                           self.bn[l - 1][0].data_ptr(), self.bn[l - 1][1].data_ptr(),
                                                           scale.data_ptr(), shift.data_ptr(), p, self.gemm_part.data_ptr(),
                                                           self.gemm_part.shape[0], s)
            elif acc:
                rc = L_.b200gnn_gemm_tf32x3_acc_f32(g.data_ptr(), g.stride(0), hi.data_ptr(), lo.data_ptr(), nb, out.data_ptr(), Kin,
                                                    N, Kin, nb, s)
            else:
                rc = L_.b200gnn_gemm_tf32x3_f32(g.data_ptr(), g.stride(0), hi.data_ptr(), lo.data_ptr(), nb, out.data_ptr(), Kin,
                                                N, Kin, nb, None, s)
            lib.check(rc, "gemm_tf32x3 (input gradient)")

    def backward(self, x: torch.Tensor, d_out_feat: Optional[torch.Tensor] = None):
        """Consumes self.dY[-1] (d loss / d logits, stored layout) and optionally d loss / d out_feat (out_feat()'s layout);
        fills self.grads."""
        L_ = lib.load()
        N = self.N
        ops.col_sum(self.dY[-1], out=self.g_bias_last, partial=self.row_part)
        for l in range(self.L - 1, -1, -1):
            H, D, K = self.Hl[l], self.Dp[l], self.K[l]
            ft, dR = self.cat[l][:, :K], self.dY[l]
            es = self.edge_scale[H]
            lib.check(L_.b200gnn_gat_bwd_rows_f32(
                self.G.rowptr.data_ptr(), self.G.col.data_ptr(), self.a[l].data_ptr(), ft.data_ptr(), ft.stride(0), dR.data_ptr(),
                dR.stride(0), self.el[l].data_ptr(), None if self.er[l] is None else self.er[l].data_ptr(), N, H, D, self.slope,
                self.dpre[l].data_ptr(), None if self.d_er[l] is None else self.d_er[l].data_ptr(), self.G.chunk_rowptr.data_ptr(),
                self.G.n_chunks, *_hub_args(self.G, H), None if es is None else es.data_ptr(), lib.stream_ptr()), "gat_bwd_rows_f32")
            # d ft: the same aggregation on the transposed graph, the two degree vectors exchanged
            ops.gat_aggregate_epi(self.Gt, self.perm, self.a[l], dR, self.dft[l], H, src_scale=self.dst_scale, row_scale=self.src_scale)
            lib.check(L_.b200gnn_segment_sum_heads_f32(self.Gt.rowptr.data_ptr(), self.perm.data_ptr(), self.dpre[l].data_ptr(), N, H,
                                                       self.d_el[l].data_ptr(), lib.stream_ptr()), "segment_sum_heads_f32")
            ops.gat_scores_bwd(ft, self.attn_l[l], self.attn_r[l], self.src_scale, self.d_el[l], self.d_er[l], H, self.dft[l],
                               self.g_attn_l[l], self.g_attn_r[l], partial=self.score_part)
            if l > 0:
                seeded = d_out_feat is not None and l == self.L - 1
                if seeded and self.Dp[0] != self.Dl[0]:             # into the stored columns, padding zero
                    self.dY[l - 1].zero_()
                    self.dY[l - 1][:, self._cols(self.L - 2)] = d_out_feat
                elif seeded:
                    self.dY[l - 1].copy_(d_out_feat)
                self._dgrad(l, seeded)
            self._ev_fork.record(torch.cuda.current_stream())     # weight gradients only feed Adam: side stream
            self._side.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side):
                self._wgrad(l, x)
            if l > 0:
                k = l - 1
                if self.fuse_bnbwd:
                    ops.bn_act_bwd_apply(self.dY[k], None, self.Y[k], self.bn[k][0], self.bn[k][1], self.gamma[k], self.gemm_part, N,
                                         self.p, self.dY[k], self.ggamma[k], self.gbeta[k], None, self.row_part, self.coef)
                else:
                    # the weight-gradient GEMM above reads Y[k], not A_mat: no hazard with the side stream
                    self._hidden(k, out=self.A_mat)
                    ops.bn_act_bwd(self.dY[k], self.A_mat, self.Y[k], self.bn[k][0], self.bn[k][1], self.gamma[k], self.p,
                                   d_y=self.dY[k], d_gamma=self.ggamma[k], d_beta=self.gbeta[k], partial=self.row_part,
                                   coef=self.coef, want_dbias=False)
        self._ev_join.record(self._side)
        torch.cuda.current_stream().wait_event(self._ev_join)

    # ------------------------------------------------------------------ step
    def _loss(self, x, y, train_idx, teacher_logits):
        """Training forward, then the fused CE / logit-KD over rows train_idx; d loss / d logits into the stored-layout dY[-1]
        (padding stays zero)."""
        logits = self.forward(x, training=True)
        self.dY[-1].zero_()
        t = teacher_logits
        lib.check(lib.load().b200gnn_kd_loss_fwd_bwd_f32(
            logits.data_ptr(), logits.stride(0), lib.dptr(train_idx, torch.int64, "train_idx"), train_idx.numel(),
            lib.dptr(y, torch.int64, "labels"), None if t is None else lib.dptr(t, torch.float32, "teacher_logits"),
            0 if t is None else t.stride(0), self.n_classes, self.alpha, self.kd_T, 0, self.dY[-1].data_ptr(), self.dY[-1].stride(0),
            self.loss_out.data_ptr(), self.kd_part.data_ptr(), lib.stream_ptr()), "kd_loss_fwd_bwd_f32")

    def replay(self, key: int = 0) -> torch.Tensor:
        super().replay(key)
        self._training = True
        return self.loss_out

    # ------------------------------------------------------------------ accounting
    def algorithmic_bytes(self) -> Dict[str, int]:
        """Compulsory HBM bytes per launch of the sparse kernels of one layer at the hidden width, from shapes:
        aggregation = read ft + write Y + read res + coefficients and indices; scores = one read of ft + el, er."""
        N, K, H, nnz = self.N, self.K[0], self.H, self.nnz
        return {"gat_aggregate_epi": 3 * N * K * 4 + nnz * (H * 4 + 4) + (N + 1) * 4,
                "gat_scores": N * K * 4 + N * H * 8,
                "gat_scores_bwd": 3 * N * K * 4 + N * H * 8,
                "gat_edge_softmax": nnz * (H * 4 + 4 + 1) + 2 * N * H * 4}

    def useful_flop(self) -> int:
        """Dense FLOP of one step's GEMMs (forward, input gradient, weight gradient), stored widths."""
        fl = 0
        for l in range(self.L):
            g = 2 * self.N * self.Kin[l] * 2 * self.K[l]
            fl += g * (3 if l > 0 else 2)
        return fl
