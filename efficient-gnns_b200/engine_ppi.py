"""Fused training step for the reference's PPI GAT models — ``StudentNet`` and ``TeacherNet`` of ppi_pyg/gnn.py:24-83.

Each layer is a PyG 1.7 ``GATConv`` plus a ``Linear`` skip on the same input; hidden layers are x = elu(conv(x) + lin(x)), the
last one averages its heads (concat=False).  PPI trains on 20 small graphs one at a time (gnn.py:308), so every per-step tensor
lives in L2 and the step is bound by launches: the engine builds every graph's plans once, records one CUDA graph per
training graph and runs few launches per layer.  One hidden layer of the step:

    [ft | res] = h [W_lin | W_skip]^T + [0 | b_lin]   one 3xTF32 GEMM (the Linear bias in its epilogue)
    el, er     = gat_scores(ft)                     one read of ft
    a          = edge_softmax(el, er)               eps 1e-16
    Z, A       = gat_aggregate_elu(a, ft, res, b_conv)   Z = Σ a·ft[src] + res + b_conv kept for the backward, A = elu(Z) the
                                                    next GEMM's operand and ``out_feat``

The last layer runs the plain aggregation and ``ppi_logits_loss`` (head mean, both biases, the BCE or logit-KD loss and the
seed gradients).  The backward is hand-written from the same kernels (elu_bwd into the d res half of the layer's [d ft | d res]
buffer, gat_bwd_rows, the aggregation on the transposed graph, segment_sum_heads, gat_scores_bwd, one input-gradient GEMM
with inner dimension 2K, weight gradients on a side stream in column blocks of at most 512, bias column sums); Adam runs over
one flat parameter buffer.

Head widths are stored with a stride Dp, a multiple of 4 (121 classes as 124); x is stored with 52 columns (a 200-byte row is
not a TMA operand).  Padded weight rows / columns, attention entries and biases are zero, their gradients and Adam moments
stay exactly zero, and state_dict() / out_feat() never show them.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import lib, ops
from .nn import _as_adj, _csr2csc_i32, _fill_diag_pattern, _hub_args
from .trainer import FlatParams, aux_grad, capture_graph

WGRAD_BLOCK = 512          # widest output block of one weight-gradient launch
STUDENT_LAYERS = [(2, 68, True)] * 4 + [(2, 121, False)]     # ppi_pyg/gnn.py:50-83
TEACHER_LAYERS = [(4, 256, True)] * 2 + [(6, 121, False)]    # ppi_pyg/gnn.py:24-47


def _pad4(d: int) -> int:
    return (d + 3) // 4 * 4


class _Graph:
    """One input graph as GATConv sees it (self-loops removed, one per node added, duplicates kept) with its engine plans."""

    def __init__(self, edge_index: torch.Tensor, n: int, device):
        adj = _fill_diag_pattern(_as_adj(edge_index.to(device=device, dtype=torch.long), n))
        st = adj.storage
        self.n = n
        self.G = st.engine_csr_unweighted()
        self.Gt = st.engine_csc("value")
        self.perm = _csr2csc_i32(st)
        self.nnz = self.G.nnz
        self.adj = adj


class _Bufs:
    """Activations and gradients of one step for up to n nodes and nnz edges; view(n, nnz) slices them for a smaller graph."""

    def __init__(self, t: "PPIGATTrainer", n: int, nnz: int, training: bool, _from=None):
        if _from is not None:
            return
        dev = t.device
        z = lambda *s: torch.zeros(*s, device=dev)          # noqa: E731
        L = t.L
        self.cat = [z(n, t.Ktot[l]) for l in range(L)]
        self.Z = [z(n, t.Kout[l]) for l in range(L - 1)]
        self.A = [z(n, t.Kout[l]) for l in range(L - 1)]
        self.el = [z(n, h) for h in t.Hl]
        self.er = [z(n, h) for h in t.Hl]
        self.a = [z(nnz, h) for h in t.Hl]
        self.agg = z(n, t.Kft[-1])
        self.logits = z(n, t.C)
        if training:
            self.gcat = [z(n, t.Ktot[l]) for l in range(L)]
            self.dA = [z(n, t.Kout[l]) for l in range(L - 1)]
            self.dagg = z(n, t.Kft[-1])
            self.d_el = [z(n, h) for h in t.Hl]
            self.d_er = [z(n, h) for h in t.Hl]
            self.dpre = [z(nnz, h) for h in t.Hl]
        self.training = training

    def view(self, n: int, nnz: int) -> "_Bufs":
        v = _Bufs(None, 0, 0, False, _from=self)
        for k, val in self.__dict__.items():
            if isinstance(val, list):
                setattr(v, k, [x[:nnz] if k in ("a", "dpre") else x[:n] for x in val])
            elif isinstance(val, torch.Tensor):
                setattr(v, k, val[:n])
            else:
                setattr(v, k, val)
        return v


class PPIGATTrainer:
    """State + fused step of a stack of PyG-GAT-with-linear-skip layers ``(heads, width, concat)`` on a fixed set of training
    graphs ``[(x [n, F], y [n, C] multi-hot, edge_index [2, E]), ...]``.  With ``teacher_logits`` (one [n, C] tensor per
    training graph) the step minimises kd_criterion (ppi_pyg/criterion.py:8-19), otherwise BCE-with-logits."""

    def __init__(self, graphs: Sequence[Tuple[torch.Tensor, torch.Tensor, torch.Tensor]], layers, in_channels: int = 50,
                 out_channels: int = 121, lr: float = 0.005, seed: int = 0, alpha: float = 0.5, T: float = 1.0,
                 teacher_logits: Optional[Sequence[torch.Tensor]] = None,
                 teacher_feat: Optional[Sequence[torch.Tensor]] = None, dropout: float = 0.0, attn_dropout: float = 0.0,
                 weight_decay: float = 0.0, negative_slope: float = 0.2, device="cuda", lsp=None, gcrd=None, gsp=None):
        """lsp: an lsp.PerGraphLSP built for these graphs, run inside every step (and every captured graph): the loss becomes
        BCE (or kd_criterion) + beta * LSP on the graph's edge list, as ppi_pyg/gnn.py's ``--training lpw``.  gcrd: a
        gcrd.PerGraphGCRD built for these graphs, run the same way: BCE (or kd_criterion) + beta * G-CRD through its
        projection heads, as ``--training nce``; its heads take one Adam step after the model's.  gsp: a gsp.PerGraphGSP
        built for these graphs, run the same way: BCE (or kd_criterion) + beta * GSP between out_feat and the teacher's
        out_feat, as ``--training gpw``."""
        if dropout != 0.0:
            raise ValueError("dropout > 0 is not implemented (ppi_pyg's GAT baseline class; StudentNet / TeacherNet have none)")
        if attn_dropout != 0.0:
            raise ValueError("attention dropout is not implemented (StudentNet / TeacherNet use GATConv's default 0)")
        if weight_decay != 0.0:
            raise ValueError("weight decay is not implemented (ppi_pyg/gnn.py's Adam has none)")
        layers = [(int(h), int(d), bool(c)) for h, d, c in layers]
        if len(layers) < 2 or not all(c for _, _, c in layers[:-1]) or layers[-1][2] or layers[-1][1] != out_channels:
            raise ValueError("layers: concat hidden layers and a last concat=False layer of out_channels")
        self.device = dev = torch.device(device)
        self.layers, self.L = layers, len(layers)
        self.F, self.C = int(in_channels), int(out_channels)
        self.lr, self.seed, self.alpha, self.kd_T, self.slope = float(lr), int(seed), float(alpha), float(T), float(negative_slope)
        L = self.L
        self.Hl = [h for h, _, _ in layers]
        self.Dl = [d for _, d, _ in layers]
        self.Dp = [_pad4(d) for d in self.Dl]
        self.Kft = [h * dp for h, dp in zip(self.Hl, self.Dp)]
        self.Kout = [h * dp if c else dp for (h, _, c), dp in zip(layers, self.Dp)]
        self.Ktot = [a + b for a, b in zip(self.Kft, self.Kout)]
        self.Fp = _pad4(self.F)
        self.Kin = [self.Fp] + self.Kout[:-1]
        if max(self.Ktot) > 2048 or max(self.Kin) > 2048 or max(self.Hl) > 16:
            raise ValueError("stored layer widths above 2048 or more than 16 heads are not built")
        self.blocks = [[(c, min(WGRAD_BLOCK, k - c)) for c in range(0, k, WGRAD_BLOCK)] for k in self.Ktot]
        if gcrd is not None:           # refused before any device work
            if lsp is not None:
                raise ValueError("gcrd= and lsp= are two auxiliary losses; pass one")
            if self.Dp[-2] != self.Dl[-2] or self.Kout[-2] > 512:
                raise ValueError(f"gcrd=: out_feat is stored {self.Kout[-2]} wide for a true width of "
                                 f"{self.Hl[-2] * self.Dl[-2]}; the student head reads unpadded rows at most 512 wide "
                                 "(its weight-gradient GEMM)")
            gcrd.check_graphs([int(x.shape[0]) for x, _, _ in graphs], self.Kout[-2])
        if gsp is not None:
            if lsp is not None or gcrd is not None:
                raise ValueError("gsp= and lsp= / gcrd= are two auxiliary losses; pass one")
            if self.Dp[-2] != self.Dl[-2]:
                raise ValueError(f"gsp=: out_feat is stored {self.Dp[-2]} wide per head for a true width of {self.Dl[-2]}; "
                                 "the GSP row passes read unpadded rows")
            gsp.check_graphs([int(x.shape[0]) for x, _, _ in graphs], self.Kout[-2])

        # ---- flat parameters, per layer: the column blocks of [W_lin | W_skip] as [in, block] (a weight gradient is one
        # contiguous output), att_l, att_r, a zero vector and b_lin (together the GEMM's bias [0 | b_lin]), b_conv
        shapes = []
        for l in range(L):
            shapes += [(self.Kin[l], nb) for _, nb in self.blocks[l]] + [(self.Kft[l],)] * 3 + [(self.Kout[l],)] * 2
        self.store = FlatParams(shapes, dev).attach(self)
        views = iter(self.store.views)
        self.W, self.gW, self.att_l, self.g_att_l, self.att_r, self.g_att_r = [], [], [], [], [], []
        self.gemm_bias, self.b_lin, self.g_b_lin, self.b_conv, self.g_b_conv = [], [], [], [], []
        for l in range(L):
            pairs = [next(views) for _ in self.blocks[l]]
            self.W.append([p for p, _ in pairs]); self.gW.append([g for _, g in pairs])
            for P, G_ in ((self.att_l, self.g_att_l), (self.att_r, self.g_att_r)):
                p, g = next(views)
                P.append(p); G_.append(g)
            zero, _ = next(views)
            p, g = next(views)
            self.b_lin.append(p); self.g_b_lin.append(g)
            o0 = self.store.offset(zero)
            self.gemm_bias.append(self.params[o0:o0 + self.Kft[l] + self.Kout[l]])
            p, g = next(views)
            self.b_conv.append(p); self.g_b_conv.append(g)
        # tf32 hi / lo splits, refreshed every step: [W_lin | W_skip]^T [Ktot, in] feeds the forward GEMM, [in, Ktot] the
        # input-gradient GEMM
        self.Wt_split = [tuple(torch.empty(self.Ktot[l], self.Kin[l], device=dev) for _ in range(2)) for l in range(L)]
        self.W_split = [tuple(torch.empty(self.Kin[l], self.Ktot[l], device=dev) for _ in range(2)) if l > 0 else None
                        for l in range(L)]
        self.wgrad_ws = torch.empty(max(ops.wgrad_workspace_floats(self.Kin[l], nb) for l in range(L) for _, nb in self.blocks[l]),
                                    device=dev)
        self.reset_parameters(seed)

        # ---- training graphs: plans, padded inputs, labels, teacher outputs (built once)
        self.graphs: List[_Graph] = []
        self.x, self.y = [], []
        for x, y, ei in graphs:
            n = int(x.shape[0])
            self.graphs.append(_Graph(ei, n, dev))
            self.x.append(self._pad_x(x))
            self.y.append(y.to(dev, torch.float32).contiguous())
        self.teacher_logits = None if teacher_logits is None else [t.to(dev, torch.float32).contiguous() for t in teacher_logits]
        self.teacher_feat = None if teacher_feat is None else [t.to(dev, torch.float32).contiguous() for t in teacher_feat]
        n_max = max(g.n for g in self.graphs)
        self.bufs = _Bufs(self, n_max, max(g.nnz for g in self.graphs), training=True)
        self.score_part = torch.empty(ops.gat_scores_slots(n_max), 2, max(self.Kft), device=dev)
        self.col_part = torch.empty(int(lib.load().b200gnn_col_sum_ld_slots(n_max)) * max(self.Kout), device=dev)
        self.tail_part = torch.empty(2 * int(lib.load().b200gnn_ppi_tail_slots(n_max)), dtype=torch.float64, device=dev)
        self._side = torch.cuda.Stream(device=dev)
        self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        self._graph: Dict[int, torch.cuda.CUDAGraph] = {}
        self._predict_cache: Dict[tuple, _Graph] = {}
        self._last: Optional[Tuple[_Graph, _Bufs]] = None
        self.epoch = 0
        self.lsp, self.gcrd, self.gsp = lsp, gcrd, gsp
        if lsp is not None:
            if self.Dp[-2] != self.Dl[-2]:
                raise ValueError(f"lsp=: out_feat is stored {self.Dp[-2]} wide per head for a true width of {self.Dl[-2]}; "
                                 "the LSP kernel reads unpadded rows")
            lsp.bind(self)

    # ------------------------------------------------------------------ parameters
    def _pad_x(self, x: torch.Tensor) -> torch.Tensor:
        xp = torch.zeros(x.shape[0], self.Fp, device=self.device)
        xp[:, :self.F] = x.to(self.device, torch.float32)
        return xp

    def _cols(self, l: int, width: str = "out") -> torch.Tensor:
        """Stored column of every true column of layer l's output ('out') or projection ('ft'); l = -1: the input x."""
        if l < 0:
            return torch.arange(self.F, device=self.device)
        H, D, Dp = self.Hl[l], self.Dl[l], self.Dp[l]
        heads = H if (width == "ft" or self.layers[l][2]) else 1
        h = torch.arange(heads, device=self.device).view(-1, 1)
        return (h * Dp + torch.arange(D, device=self.device).view(1, -1)).reshape(-1)

    def _store_w(self, l: int, w_lin: torch.Tensor, w_skip: torch.Tensor):
        """Reference weights [out, in] -> the [in_stored, block] column blocks of [W_lin | W_skip], padding zero."""
        full = torch.zeros(self.Kin[l], self.Ktot[l], device=self.device)
        rows = self._cols(l - 1).view(-1, 1)
        full[rows, self._cols(l, "ft").view(1, -1)] = w_lin.to(self.device, torch.float32).t()
        full[rows, self.Kft[l] + self._cols(l).view(1, -1)] = w_skip.to(self.device, torch.float32).t()
        for (c0, nb), blk in zip(self.blocks[l], self.W[l]):
            blk.copy_(full[:, c0:c0 + nb])

    def _load_vec(self, dst: torch.Tensor, cols: torch.Tensor, v: torch.Tensor):
        dst.zero_()
        dst[cols] = v.to(self.device, torch.float32).reshape(-1)

    def reset_parameters(self, seed: int = 0):
        """GATConv.reset_parameters (glorot lin_l / att_l / att_r, zero bias) and torch.nn.Linear's default init, drawn from a
        CPU generator seeded with ``seed``; Adam state cleared."""
        g = torch.Generator().manual_seed(seed)

        def glorot(shape, fan_a, fan_b):
            a = (6.0 / (fan_a + fan_b)) ** 0.5
            return torch.rand(shape, generator=g) * 2 * a - a

        fin = self.F
        for l, (H, D, concat) in enumerate(self.layers):
            out = H * D if concat else D
            w_lin = glorot((H * D, fin), H * D, fin)
            b = 1.0 / fin ** 0.5
            w_skip = torch.rand(out, fin, generator=g) * 2 * b - b
            self._store_w(l, w_lin, w_skip)
            self._load_vec(self.att_l[l], self._cols(l, "ft"), glorot((H, D), H, D))
            self._load_vec(self.att_r[l], self._cols(l, "ft"), glorot((H, D), H, D))
            self._load_vec(self.b_lin[l], self._cols(l), torch.rand(out, generator=g) * 2 * b - b)
            self.b_conv[l].zero_()
            fin = out
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_count.zero_()

    def _export(self, W, att_l, att_r, b_lin, b_conv) -> Dict[str, torch.Tensor]:
        sd = {}
        for l, (H, D, concat) in enumerate(self.layers):
            i = l + 1
            full = torch.cat(W[l], dim=1)[self._cols(l - 1)]
            sd[f"conv{i}.att_l"] = att_l[l][self._cols(l, "ft")].view(1, H, D).clone()
            sd[f"conv{i}.att_r"] = att_r[l][self._cols(l, "ft")].view(1, H, D).clone()
            sd[f"conv{i}.bias"] = b_conv[l][self._cols(l)].clone()
            sd[f"conv{i}.lin_l.weight"] = full[:, self._cols(l, "ft")].t().contiguous()
            sd[f"conv{i}.lin_r.weight"] = sd[f"conv{i}.lin_l.weight"]            # PyG's alias of lin_l
            sd[f"lin{i}.weight"] = full[:, self.Kft[l] + self._cols(l)].t().contiguous()
            sd[f"lin{i}.bias"] = b_lin[l][self._cols(l)].clone()
        return sd

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys and shapes of the reference module's state_dict (StudentNet / TeacherNet on PyG 1.7 GATConv)."""
        return self._export(self.W, self.att_l, self.att_r, self.b_lin, self.b_conv)

    def named_gradients(self) -> Dict[str, torch.Tensor]:
        """The last backward's parameter gradients under the state_dict keys."""
        return self._export(self.gW, self.g_att_l, self.g_att_r, self.g_b_lin, self.g_b_conv)

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for l in range(self.L):
            i = l + 1
            self._store_w(l, sd[f"conv{i}.lin_l.weight"], sd[f"lin{i}.weight"])
            self._load_vec(self.att_l[l], self._cols(l, "ft"), sd[f"conv{i}.att_l"])
            self._load_vec(self.att_r[l], self._cols(l, "ft"), sd[f"conv{i}.att_r"])
            self._load_vec(self.b_lin[l], self._cols(l), sd[f"lin{i}.bias"])
            self._load_vec(self.b_conv[l], self._cols(l), sd[f"conv{i}.bias"])

    # ------------------------------------------------------------------ forward
    def _forward(self, g: _Graph, b: _Bufs, x: torch.Tensor, y=None, t=None):
        """Every layer; the tail writes the logits and, given labels, the loss and the last layer's seed gradients."""
        L_, s = lib.load(), lib.stream_ptr()
        G = g.G
        for l in range(self.L):
            H, Dp, Kft, last = self.Hl[l], self.Dp[l], self.Kft[l], l == self.L - 1
            hi, lo = self.Wt_split[l]
            for (c0, nb), blk in zip(self.blocks[l], self.W[l]):
                ops.split_tf32(blk, transpose=True, hi=hi[c0:c0 + nb], lo=lo[c0:c0 + nb])
            h = x if l == 0 else b.A[l - 1]
            ops.gemm_tf32x3(h, hi, lo, bias=None if last else self.gemm_bias[l], out=b.cat[l])
            ft, res = b.cat[l][:, :Kft], b.cat[l][:, Kft:]
            ops.gat_scores(ft, self.att_l[l], self.att_r[l], None, H, el=b.el[l], er=b.er[l])
            lib.check(L_.b200gnn_gat_edge_softmax_f32(G.rowptr.data_ptr(), G.col.data_ptr(), b.el[l].data_ptr(), b.er[l].data_ptr(),
                                                      g.n, H, self.slope, 1e-16, b.a[l].data_ptr(), None, s),
                      "gat_edge_softmax_f32")
            if not last:
                ops.gat_aggregate_elu(G, b.a[l], ft, b.Z[l], b.A[l], H, res=res, bias=self.b_conv[l])
                continue
            ops.gat_aggregate_epi(G, None, b.a[l], ft, b.agg, H)
            train = y is not None
            ops.ppi_logits_loss(b.agg, res, self.b_conv[l], self.b_lin[l], H, self.C, b.logits, labels=y, teacher_logits=t,
                                alpha=self.alpha, T=self.kd_T, d_agg=b.dagg if train else None,
                                d_res=b.gcat[l][:, Kft:] if train else None, loss_out=self.loss_out if train else None,
                                partial=self.tail_part if train else None)

    # ------------------------------------------------------------------ backward
    def _wgrad(self, l: int, h: torch.Tensor, gcat: torch.Tensor):
        """[dW_lin | dW_skip] = h^T [d ft | d res], block by block, straight into the flat gradient buffer."""
        L_, s = lib.load(), lib.stream_ptr()
        for (c0, nb), out in zip(self.blocks[l], self.gW[l]):
            gb = gcat[:, c0:c0 + nb]
            lib.check(L_.b200gnn_gemm_wgrad_tf32x3_f32(h.data_ptr(), h.stride(0), gb.data_ptr(), gb.stride(0), out.data_ptr(),
                                                       h.shape[0], self.Kin[l], nb, self.wgrad_ws.data_ptr(), s),
                      "gemm_wgrad_tf32x3")

    def _backward(self, g: _Graph, b: _Bufs, x: torch.Tensor, d_out_feat: Optional[torch.Tensor] = None):
        """Consumes the tail's d agg / d res (and optionally d loss / d out_feat, copied into b.dA[L-2] unless it is that
        buffer already); fills self.grads."""
        L_, s = lib.load(), lib.stream_ptr()
        G, Gt, n = g.G, g.Gt, g.n
        for l in range(self.L - 1, -1, -1):
            H, Dp, Kft, last = self.Hl[l], self.Dp[l], self.Kft[l], l == self.L - 1
            ft, gcat = b.cat[l][:, :Kft], b.gcat[l]
            dres = gcat[:, Kft:]
            if not last:          # d Z = elu'(Z) d A into the d res half; d agg = d res for a concat layer
                ops.elu_bwd(b.dA[l], b.Z[l], out=dres)
            dout = b.dagg if last else dres
            lib.check(L_.b200gnn_gat_bwd_rows_f32(
                G.rowptr.data_ptr(), G.col.data_ptr(), b.a[l].data_ptr(), ft.data_ptr(), ft.stride(0), dout.data_ptr(), dout.stride(0),
                b.el[l].data_ptr(), b.er[l].data_ptr(), n, H, Dp, self.slope, b.dpre[l].data_ptr(), b.d_er[l].data_ptr(),
                G.chunk_rowptr.data_ptr(), G.n_chunks, *_hub_args(G, H), None, s), "gat_bwd_rows_f32")
            dft = gcat[:, :Kft]
            ops.gat_aggregate_epi(Gt, g.perm, b.a[l], dout, dft, H)
            lib.check(L_.b200gnn_segment_sum_heads_f32(Gt.rowptr.data_ptr(), g.perm.data_ptr(), b.dpre[l].data_ptr(), n, H,
                                                       b.d_el[l].data_ptr(), s), "segment_sum_heads_f32")
            ops.gat_scores_bwd(ft, self.att_l[l], self.att_r[l], None, b.d_el[l], b.d_er[l], H, dft, self.g_att_l[l],
                               self.g_att_r[l], partial=self.score_part)
            if l > 0:             # d A[l-1] (+)= [d ft | d res] [W_lin | W_skip], inner dimension Ktot
                hi, lo = self.W_split[l]
                if len(self.blocks[l]) == 1:
                    ops.split_tf32(self.W[l][0], transpose=False, hi=hi, lo=lo)
                else:
                    for src, dst in zip(self.Wt_split[l], (hi, lo)):
                        lib.check(L_.b200gnn_transpose_f32(src.data_ptr(), self.Ktot[l], self.Kin[l], dst.data_ptr(), s),
                                  "transpose_f32")
                seeded = d_out_feat is not None and l == self.L - 1
                out = b.dA[l - 1]
                if seeded and d_out_feat is not out:
                    out.copy_(d_out_feat)
                ops.gemm_tf32x3(gcat, hi, lo, out=out, accumulate=seeded)
            self._ev_fork.record(torch.cuda.current_stream())     # weight gradients only feed Adam: side stream
            self._side.wait_event(self._ev_fork)
            with torch.cuda.stream(self._side):
                self._wgrad(l, x if l == 0 else b.A[l - 1], gcat)
            ops.col_sum_ld(dres, self.g_b_lin[l], partial=self.col_part)
            ops.col_sum_ld(dres, self.g_b_conv[l], partial=self.col_part)   # the same sum: two parameters, two Adam states
        self._ev_join.record(self._side)
        torch.cuda.current_stream().wait_event(self._ev_join)

    # ------------------------------------------------------------------ step
    def _teacher(self, i: int) -> Optional[torch.Tensor]:
        return None if self.teacher_logits is None else self.teacher_logits[i]

    def _step_impl(self, i: int, aux=None, beta: float = 1.0, sample=None):
        g = self.graphs[i]
        b = self.bufs.view(g.n, g.nnz)
        self._forward(g, b, self.x[i], self.y[i], self._teacher(i))
        self._last = (g, b)
        d_feat = None
        if aux is not None:
            d, loss_aux = aux_grad(self.out_feat(), aux, beta)
            d_feat = torch.zeros(g.n, self.Kout[-2], device=self.device)        # into the stored columns, padding zero
            d_feat[:, self._cols(self.L - 2)] = d
        elif self.lsp is not None:       # out_feat is A[L-2] unpadded; its gradient is the seed the input-gradient GEMM adds to
            d_feat = b.dA[self.L - 2]
            self.lsp.forward_backward(i, b.A[self.L - 2], d_feat, self.loss_out)
            self.loss_out[2].copy_(self.lsp.loss_aux[0])
        elif self.gcrd is not None:      # the student head's input gradient is stored over all n rows of that seed
            d_feat = b.dA[self.L - 2]
            self.gcrd.forward_backward(i, self, b.A[self.L - 2], d_feat, sample)
            self.loss_out[2].copy_(self.gcrd.loss_aux[0])
        elif self.gsp is not None:       # beta * d loss / d out_feat is stored straight into that seed
            d_feat = b.dA[self.L - 2]
            self.gsp.forward_backward(i, self, b.A[self.L - 2], d_feat, sample)
            self.loss_out[2].copy_(self.gsp.loss_aux[0])
        self._backward(g, b, self.x[i], d_out_feat=d_feat)
        self.store.adam(self.lr)
        if self.gcrd is not None:
            self.gcrd.optimizer_step(self.lr)
        if aux is not None:
            self.loss_out[0].add_(loss_aux * beta)
            self.loss_out[2].copy_(loss_aux)

    def train_step(self, i: int, aux=None, beta: float = 1.0, sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One step on training graph i: BCE, or kd_criterion when teacher logits were given.  ``aux(out_feat)`` (the [n, hidden]
        activation of layer L-2, requires_grad) returns an auxiliary loss that enters as loss + beta * aux and seeds the backward
        at out_feat (gnn.py:213-265); the teacher's out_feat for graph i is ``self.teacher_feat[i]``.  Returns the device tensor
        [loss, loss_cls, loss_aux] (loss_aux: the kd term, or aux's / the lsp= / gcrd= / gsp= object's value when given); no
        host sync.  ``sample`` (positions into graph i's nodes, [S]) replaces the gcrd= or gsp= object's on-device row
        draw."""
        if aux is not None and self.lsp is not None:
            raise ValueError("aux= and the trainer's lsp= objective are two auxiliary losses; pass one")
        if aux is not None and self.gcrd is not None:
            raise ValueError("aux= and the trainer's gcrd= objective are two auxiliary losses; pass one")
        if aux is not None and self.gsp is not None:
            raise ValueError("aux= and the trainer's gsp= objective are two auxiliary losses; pass one")
        if sample is not None and self.gcrd is None and self.gsp is None:
            raise ValueError("sample= is the G-CRD row sample; this trainer has no gcrd= objective")
        if sample is not None and self.gsp is not None:
            self.gsp.check_sample(i, sample)
        self._step_impl(i, aux, beta, sample)
        return self.loss_out

    def logits(self) -> torch.Tensor:
        """Logits [n, C] of the last training forward."""
        return self._last[1].logits

    def out_feat(self) -> torch.Tensor:
        """The reference's ``model.out_feat`` of the last forward: the last hidden activation, padding removed."""
        A = self._last[1].A[self.L - 2]
        return A if self.Dp[-2] == self.Dl[-2] else A[:, self._cols(self.L - 2)].contiguous()

    # ------------------------------------------------------------------ CUDA graphs
    def capture(self, warmup: int = 1):
        """Record one CUDA graph per training graph.  Warm-up steps run on a saved copy of the parameters and Adam state (and
        of the gcrd= heads' state), which is restored afterwards: capturing does not train."""
        heads = self.gcrd.preserved() if self.gcrd is not None else contextlib.nullcontext()
        with self.store.preserved(), heads:
            for i in range(len(self.graphs)):
                self._graph[i] = capture_graph(lambda: self._step_impl(i), warmup)
        return self

    def replay(self, i: int) -> torch.Tensor:
        self._graph[i].replay()
        g = self.graphs[i]
        if self.gcrd is not None:
            self.gcrd._last = i
        if self.gsp is not None:
            self.gsp._last = i
        self._last = (g, self.bufs.view(g.n, g.nnz))
        return self.loss_out

    def epoch_order(self, epoch: int) -> List[int]:
        """The training graphs in the epoch's shuffled order: a CPU permutation drawn from (seed, epoch).  Like
        DataLoader(shuffle=True) every graph comes once per epoch; the order is not torch's DataLoader stream."""
        g = torch.Generator().manual_seed((self.seed * 1_000_003 + epoch) & 0x7FFFFFFFFFFFFFFF)
        return torch.randperm(len(self.graphs), generator=g).tolist()

    def train_epoch(self, epoch: Optional[int] = None) -> torch.Tensor:
        """One pass over the training graphs in ``epoch_order(epoch)``, replaying the captured graphs (eager steps when
        nothing is captured).  Returns the per-step losses [n_graphs, 3] in that order (device, no sync)."""
        epoch = self.epoch if epoch is None else int(epoch)
        self.epoch = epoch + 1
        out = torch.empty(len(self.graphs), 3, device=self.device)
        for k, i in enumerate(self.epoch_order(epoch)):
            out[k].copy_(self.replay(i) if i in self._graph else self.train_step(i))
        return out

    # ------------------------------------------------------------------ eval
    def _predict_graph(self, edge_index: torch.Tensor, n: int) -> _Graph:
        """The plans of an input graph, cached per edge_index tensor: the entry keeps the caller's tensor alive (its address
        cannot be handed to another tensor while cached) and is keyed by its in-place version, so an edited or a new graph
        gets new plans.  At most 8 graphs are kept (test() predicts the same few graphs every epoch)."""
        key = (edge_index.data_ptr(), tuple(edge_index.shape), edge_index._version, str(edge_index.device), n)
        g = self._predict_cache.get(key)
        if g is not None and g.edge_index is not edge_index:
            g = None
        if g is None:
            if len(self._predict_cache) >= 8:
                self._predict_cache.clear()
            g = self._predict_cache[key] = _Graph(edge_index, n, self.device)
            g.edge_index = edge_index
        return g

    @torch.no_grad()
    def predict(self, x: torch.Tensor, edge_index: torch.Tensor, return_feat: bool = False):
        """Eval forward on any graph or disjoint union (a PyG ``Batch``'s x / edge_index): logits [n, C], and with
        ``return_feat`` also out_feat (for a teacher: the student's KD and auxiliary inputs, computed once per graph).
        Plans are cached per edge_index tensor (see _predict_graph)."""
        n = int(x.shape[0])
        g = self._predict_graph(edge_index, n)
        b = _Bufs(self, n, g.nnz, training=False)
        self._forward(g, b, self._pad_x(x))
        logits = b.logits
        if not return_feat:
            return logits
        A = b.A[self.L - 2]
        return logits, (A if self.Dp[-2] == self.Dl[-2] else A[:, self._cols(self.L - 2)].contiguous())

    # ------------------------------------------------------------------ accounting
    def launches_per_step(self, i: int = 0) -> int:
        """b200gnn kernel launches in one training step on graph i (counted); advances the state by one step."""
        before = lib.launch_count()
        self._step_impl(i)
        return lib.launch_count() - before


def student(graphs, in_channels: int = 50, out_channels: int = 121, **kw) -> PPIGATTrainer:
    """ppi_pyg/gnn.py StudentNet: 4 x elu(GATConv(68, heads=2) + Linear(136)), then GATConv(121, heads=2, concat=False) +
    Linear(121) (scripts/run.sh: --num_layers 5 --hidden_channels 68)."""
    layers = [(h, out_channels if d == 121 else d, c) for h, d, c in STUDENT_LAYERS]
    return PPIGATTrainer(graphs, layers, in_channels, out_channels, **kw)


def teacher(graphs, in_channels: int = 50, out_channels: int = 121, **kw) -> PPIGATTrainer:
    """ppi_pyg/gnn.py TeacherNet (also train_teacher.py): 2 x elu(GATConv(256, heads=4) + Linear(1024)), then
    GATConv(121, heads=6, concat=False) + Linear(121)."""
    layers = [(h, out_channels if d == 121 else d, c) for h, d, c in TEACHER_LAYERS]
    return PPIGATTrainer(graphs, layers, in_channels, out_channels, **kw)
