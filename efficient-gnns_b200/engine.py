"""Fused full-batch training step for the GCN student (+ logit-KD) — BASELINE.json configs[1].

Mirrors what one call of the reference's ``train()`` does for ``--gnn gcn --training kd|supervised``
(arxiv_pyg/gnn.py:102-195 with ``GCN.forward`` :45-53, ``kd_criterion`` criterion.py:8-21, Adam :308-315):

    for each layer:  H = X W            (dense GEMM; cuBLAS fp32 through torch.mm — a plain library GEMM)
                     Y = Â H + b        (b200gnn SpMM, bias + BatchNorm statistics fused in the epilogue)
                     X = dropout(relu(BN(Y)))   (formed inside the GEMMs that read X, from Y and packed keep bits)
    loss, dlogits = fused CE/KD row kernel over logits[train_idx]
    backward: dH = Âᵀ dY (same SpMM kernel), dW = Xᵀ dH, dX = dH Wᵀ, fused BN/ReLU/dropout backward
    Adam over one flat parameter buffer.

No autograd tape: activations live in preallocated buffers and the whole step (≈40 launches) is captured
into one CUDA graph.  Everything except the three GEMM shapes is hand-written sm_90a code behind the C ABI.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional

import torch

from . import lib, ops
from .sparse import CsrGraph, SparseTensor
from .trainer import FlatParams, FullBatchStudent, one_objective


def gcn_norm(adj: SparseTensor) -> SparseTensor:
    """PyG gcn_norm for a SparseTensor (SURVEY Appendix A.2): Â = D^-1/2 (A + I) D^-1/2, A value-less => ones."""
    if not adj.has_value():
        adj = adj.fill_value(1.0)
    adj = adj.fill_diag(1.0)
    deg = adj.sum(dim=1)
    dis = deg.pow(-0.5)
    dis.masked_fill_(dis == float("inf"), 0.0)
    row, col, val = adj.coo()
    return adj.set_value(dis[row] * val * dis[col])


def _is_symmetric(adj: SparseTensor) -> bool:
    st = adj.storage
    if st.sparse_sizes()[0] != st.sparse_sizes()[1]:
        return False
    perm = st.csr2csc()
    same = torch.equal(st.col()[perm], st.row()) and torch.equal(st.row()[perm], st.col())
    if same and st.value() is not None:
        same = torch.equal(st.value()[perm], st.value())
    return bool(same)


class GCNStudentTrainer(FullBatchStudent):
    """State + fused step of an L-layer GCN student on one GPU."""

    def __init__(self, adj: SparseTensor, dims: List[int], dropout: float = 0.5, lr: float = 0.01, seed: int = 0,
                 alpha: float = 0.9, kd_T: float = 4.0, bn_eps: float = 1e-5, bn_momentum: float = 0.1,
                 aggregate_first: Optional[bool] = None, tensor_core_gemm: bool = True, overlap_wgrad: bool = True,
                 fuse_row_passes: bool = True, fuse_activations: bool = True, _prebuilt_graph: Optional[CsrGraph] = None, _rows_alloc: Optional[int] = None,
                 gcrd=None, lsp=None, gsp=None):
        """gcrd: a gcrd.GCRD whose projection heads and InfoNCE loss run inside this trainer's step (kd or supervised + beta *
        G-CRD, one CUDA graph); lsp: an lsp.LSP run the same way (kd or supervised + beta * LSP); gsp: a gsp.GSP, the
        projection heads of G-CRD with the pairwise-similarity loss (kd or supervised + beta * GSP); at most one of the three,
        and None for all leaves the step as it is."""
        self.objective = one_objective(gcrd, lsp, gsp)
        assert adj.is_cuda(), "the engine runs on a CUDA device"
        self.device = adj.device
        self.dims, self.L = list(dims), len(dims) - 1
        self.p, self.lr, self.alpha, self.kd_T = float(dropout), float(lr), float(alpha), float(kd_T)
        self.bn_eps, self.bn_momentum = bn_eps, bn_momentum
        self.seed = int(seed)
        self.tc_gemm = bool(tensor_core_gemm) and all(d % 4 == 0 for d in dims)
        for d in dims[1:]:
            assert d % 4 == 0 and d <= 1024, "layer widths must be multiples of 4 (128-bit rows)"
        self.N = adj.size(0)
        # Layer 0 may aggregate BEFORE its GEMM: Â(XW) = (ÂX)W.  When the input is narrower than the hidden width
        # the gather runs at the narrow width, and because X needs no gradient the backward aggregation of layer 0
        # disappears altogether: dW0 = (ÂX)ᵀ dY0.  Same mathematics as the reference (PyG transforms first and
        # pays a 256-wide backward SpMM whose result is only used as an intermediate); fp32 reassociation only.
        self.agg_first = (dims[0] < dims[1] and dims[0] % 4 == 0) if aggregate_first is None else bool(aggregate_first)
        if self.L < 2:
            self.agg_first = False

        if _prebuilt_graph is not None:          # a row shard of the normalised adjacency (dist.ShardedGCNTrainer)
            self.G = self.Gt = _prebuilt_graph
            self.N = _prebuilt_graph.n_rows
        else:
            norm = gcn_norm(adj)                 # cached=True semantics: normalise once (arxiv_pyg/gnn.py:28)
            self.G: CsrGraph = norm.storage.engine_csr()
            self.Gt: CsrGraph = self.G if _is_symmetric(norm) else norm.storage.engine_csc("value")
        self.nnz = self.G.nnz

        # ---- flat parameters: per layer W [in,out], b [out]; per hidden layer gamma, beta
        shapes = []
        for l in range(self.L):
            shapes += [(dims[l], dims[l + 1]), (dims[l + 1],)]
            if l < self.L - 1:
                shapes += [(dims[l + 1],), (dims[l + 1],)]
        dev = self.device
        self.store = FlatParams(shapes, dev).attach(self)
        self.W, self.b, self.gamma, self.beta = [], [], [], []
        self.gW, self.gb, self.ggamma, self.gbeta = [], [], [], []
        views = iter(self.store.views)
        for l in range(self.L):
            (w, gw), (b, gb) = next(views), next(views)
            self.W.append(w); self.gW.append(gw); self.b.append(b); self.gb.append(gb)
            if l < self.L - 1:
                (g, gg), (be, gbe) = next(views), next(views)
                self.gamma.append(g); self.ggamma.append(gg); self.beta.append(be); self.gbeta.append(gbe)
        # tf32 hi/lo splits of the weights for the wgmma GEMM: W^T [out,in] feeds the forward (C = X W),
        # W [in,out] feeds the input gradient (dX = dH W^T); refreshed every step (a few KB).
        self.Wt_split = [(torch.empty(dims[l + 1], dims[l], device=dev), torch.empty(dims[l + 1], dims[l], device=dev))
                         for l in range(self.L)]
        self.W_split = [(torch.empty(dims[l], dims[l + 1], device=dev), torch.empty(dims[l], dims[l + 1], device=dev))
                        for l in range(self.L)]
        wg = [ops.wgrad_supported(dims[l], dims[l + 1]) for l in range(self.L)]
        self.wgrad_ws = (torch.empty(max(ops.wgrad_workspace_floats(dims[l], dims[l + 1]) for l in range(self.L) if wg[l]), device=dev)
                         if self.tc_gemm and any(wg) else None)
        self.running_mean = [torch.zeros(d, device=dev) for d in dims[1:-1]]
        self.running_var = [torch.ones(d, device=dev) for d in dims[1:-1]]
        self.reset_parameters(seed)

        # ---- activations / gradients (preallocated; CUDA-graph friendly)
        N = self.N
        rows_alloc = N if _rows_alloc is None else _rows_alloc   # shards over-allocate to the common block size
        self._blocks = []

        def buf(k):
            blk = torch.zeros(rows_alloc, k, device=dev)
            self._blocks.append(blk)
            return blk[:N]
        self.H = [buf(dims[l + 1]) for l in range(self.L)]            # X W
        self.Y = [buf(dims[l + 1]) for l in range(self.L)]            # Â H + b  (last = logits)
        self._A = [buf(dims[l + 1]) for l in range(self.L - 1)]       # dropout(relu(BN(Y))): see the A property
        self.dY = [buf(dims[l + 1]) for l in range(self.L)]
        self.dH = [buf(dims[l + 1]) for l in range(self.L)]
        self.dA = [buf(dims[l + 1]) for l in range(self.L - 1)]
        self.AX = buf(dims[0]) if self.agg_first else None              # Â X (layer 0, aggregate-first)
        slots_spmm = ops.stat_slots(self.G)
        self.stat_part = [torch.empty(slots_spmm, 2, dims[l + 1], device=dev) for l in range(self.L - 1)]
        self.bn = [torch.empty(4, dims[l + 1], device=dev) for l in range(self.L - 1)]   # mean, invstd, scale, shift
        self.rs = ops.rows_slots(N)
        # Row passes fused into GEMM epilogues (SURVEY §8 f1): the layer-0 BatchNorm statistics come out of the layer-0 GEMM
        # and pass 1 of every BatchNorm/ReLU/dropout backward out of the input-gradient GEMM that produces its dOut.
        self.fuse_rows = bool(fuse_row_passes) and self.tc_gemm
        self._gemm_part = {k: torch.empty(ops.gemm_stat_slots(N, k), 2, k, device=dev)
                           for k in set(dims[1:-1]) if self.fuse_rows and ops.gemm_stats_supported(k)}
        # Activations not materialised in training (the default where the fused kernels apply): the step draws the dropout
        # keep decisions of all hidden layers as packed bits (one launch, on the side stream next to the layer-0
        # aggregation), and every reader of A[l] (the next layer's GEMM, the weight-gradient GEMM, the BatchNorm-backward
        # epilogue) recomputes it from Y[l], bn[l] scale / shift and the bits: the two [N, K] sweeps of the activation
        # pass disappear.  The A property materialises the last training step's activations on first read.
        hid = dims[1:-1]
        self.fuse_act = (bool(fuse_activations) and self.fuse_rows and self.L >= 2 and len(set(hid)) == 1
                         and ops.gemm_stats_supported(hid[0]) and hid[0] <= 2048
                         and all(ops.wgrad_supported(dims[l], dims[l + 1]) for l in range(1, self.L)))
        self.keep_bits = (torch.zeros(self.L - 1, N, (hid[0] + 31) // 32, dtype=torch.int32, device=dev)
                          if self.fuse_act else None)
        self._act_stale = False            # A[l] not yet materialised for the last forward
        self._fwd_fused = False            # the last forward left its activations to the fused kernels
        self._ev_bits = torch.cuda.Event()
        self.kd_part = torch.empty(2 * int(lib.load().b200gnn_kd_partials(N)), device=dev)
        # weight gradients only feed Adam: they run on a side stream next to the BN/ReLU backward passes and the next
        # aggregation (parallel branches of the captured graph)
        self.overlap_wgrad = overlap_wgrad
        self._side = torch.cuda.Stream(device=dev) if overlap_wgrad else None
        self._ev_fork, self._ev_join = torch.cuda.Event(), torch.cuda.Event()
        self._static: Dict[str, torch.Tensor] = {}
        for k in set(dims[1:]):
            self._part(k); self._coef(k)
        if self.objective is not None:
            self.objective.bind(self)

    # ------------------------------------------------------------------ parameters
    def reset_parameters(self, seed: int = 0):
        """GCNConv: glorot weight, zero bias; BatchNorm1d: ones / zeros (SURVEY A.2, A.8)."""
        g = torch.Generator().manual_seed(seed)
        for l in range(self.L):
            fan_in, fan_out = self.dims[l], self.dims[l + 1]
            a = math.sqrt(6.0 / (fan_in + fan_out))
            self.W[l].copy_((torch.rand(fan_in, fan_out, generator=g) * 2 - 1) * a)
            self.b[l].zero_()
        for l in range(self.L - 1):
            self.gamma[l].fill_(1.0); self.beta[l].zero_()
            self.running_mean[l].zero_(); self.running_var[l].fill_(1.0)
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_count.zero_()

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys of the reference's GCN module under PyG 1.x (convs.i.weight / bias, bns.i.*)."""
        sd = {}
        for l in range(self.L):
            sd[f"convs.{l}.weight"] = self.W[l].detach().clone()
            sd[f"convs.{l}.bias"] = self.b[l].detach().clone()
        for l in range(self.L - 1):
            sd[f"bns.{l}.weight"] = self.gamma[l].detach().clone()
            sd[f"bns.{l}.bias"] = self.beta[l].detach().clone()
            sd[f"bns.{l}.running_mean"] = self.running_mean[l].clone()
            sd[f"bns.{l}.running_var"] = self.running_var[l].clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for l in range(self.L):
            self.W[l].copy_(sd[f"convs.{l}.weight"]); self.b[l].copy_(sd[f"convs.{l}.bias"])
        for l in range(self.L - 1):
            self.gamma[l].copy_(sd[f"bns.{l}.weight"]); self.beta[l].copy_(sd[f"bns.{l}.bias"])
            if f"bns.{l}.running_mean" in sd:
                self.running_mean[l].copy_(sd[f"bns.{l}.running_mean"]); self.running_var[l].copy_(sd[f"bns.{l}.running_var"])

    # ------------------------------------------------------------------ forward / backward
    @property
    def A(self) -> List[torch.Tensor]:
        """Hidden activations dropout(relu(BN(Y))) of the last forward, [N, dims[l+1]] per hidden layer."""
        if self._act_stale:
            self._act_stale = False
            for l in range(self.L - 1):
                ops.affine_relu_bits(self.Y[l], self.keep_bits[l], self.bn[l][2], self.bn[l][3], self.p, out=self._A[l])
        return self._A

    def _act(self, l: int):
        """(Y, scale, shift, keep bits) from which the fused kernels form hidden activation l."""
        return self.Y[l], self.bn[l][2], self.bn[l][3], self.keep_bits[l]

    def activation_pattern(self, l: int) -> torch.Tensor:
        """bool [N, dims[l+1]]: ReLU-active AND kept by dropout in the last training forward of hidden layer l."""
        return self.A[l] > 0

    def out_feat(self) -> torch.Tensor:
        """The reference's ``model.out_feat`` (arxiv_pyg/gnn.py:51): output of the last hidden layer."""
        return self.A[-1]

    def forward(self, x: torch.Tensor, training: bool = True) -> torch.Tensor:
        """Returns logits [N,C]; hidden activations stay in self.A (self.A[-1] is the reference's model.out_feat)."""
        fused = training and self.fuse_act
        self._act_stale = False
        if fused:
            # the keep bits need no input: drawn next to the first aggregation, joined before the first reader
            if self._side is not None:
                self._ev_fork.record(torch.cuda.current_stream())
                self._side.wait_event(self._ev_fork)
                with torch.cuda.stream(self._side):
                    ops.dropout_bits(self.keep_bits, self.p, self.seed, 0, step_dev=self.step_count, step_mul=self.L)
                self._ev_bits.record(self._side)
            else:
                ops.dropout_bits(self.keep_bits, self.p, self.seed, 0, step_dev=self.step_count, step_mul=self.L)
        A = self._A
        inp = x
        for l in range(self.L):
            last = l == self.L - 1
            if l == 0 and self.agg_first:
                ops.spmm_csr(self.G, x, "sum", out=self.AX)
                if training:
                    gp = self._gemm_part.get(self.dims[1])
                    if gp is not None:                               # statistics of Y0 from the GEMM epilogue
                        hi, lo = ops.split_tf32(self.W[0], transpose=True, hi=self.Wt_split[0][0], lo=self.Wt_split[0][1])
                        ops.gemm_tf32x3_stats(self.AX, hi, lo, self.b[0], self.Y[0], gp)
                        part = gp
                    else:
                        self._linear(0, self.AX, self.Y[0], bias=self.b[0])
                        part = ops.col_stats(self.Y[0], partial=self._part(self.dims[1]))
                    ops.bn_finalize(part, self.N, self.gamma[0], self.beta[0], self.bn_eps,
                                    self.bn_momentum, self.running_mean[0], self.running_var[0], out=self.bn[0])
                    if not fused:
                        ops.affine_relu_dropout(self.Y[0], self.bn[0][2], self.bn[0][3], True, self.p, self.seed, 0,
                                                out=A[0], step_dev=self.step_count, step_mul=self.L)
                else:
                    self._linear(0, self.AX, self.Y[0], bias=self.b[0])
                    scale = self.gamma[0] * torch.rsqrt(self.running_var[0] + self.bn_eps)
                    shift = self.beta[0] - self.running_mean[0] * scale
                    ops.affine_relu_dropout(self.Y[0], scale, shift, True, 0.0, out=A[0])
                inp = A[0]
                continue
            if fused and l > 0:
                if l == 1 and self._side is not None:
                    torch.cuda.current_stream().wait_event(self._ev_bits)
                self._linear(l, None, self.H[l], act=self._act(l - 1))
            else:
                self._linear(l, inp, self.H[l])
            if last:
                ops.spmm_csr(self.G, self.H[l], "sum", bias=self.b[l], out=self.Y[l])
            elif training:
                ops.spmm_csr(self.G, self.H[l], "sum", bias=self.b[l], out=self.Y[l], stat_partial=self.stat_part[l])
                ops.bn_finalize(self.stat_part[l], self.N, self.gamma[l], self.beta[l], self.bn_eps, self.bn_momentum,
                                self.running_mean[l], self.running_var[l], out=self.bn[l])
                if not fused:
                    ops.affine_relu_dropout(self.Y[l], self.bn[l][2], self.bn[l][3], True, self.p, self.seed, l,
                                            out=A[l], step_dev=self.step_count, step_mul=self.L)
                inp = A[l]
            else:
                ops.spmm_csr(self.G, self.H[l], "sum", bias=self.b[l], out=self.Y[l])
                scale = self.gamma[l] * torch.rsqrt(self.running_var[l] + self.bn_eps)
                shift = self.beta[l] - self.running_mean[l] * scale
                ops.affine_relu_dropout(self.Y[l], scale, shift, True, 0.0, out=A[l])
                inp = A[l]
        self._act_stale = self._fwd_fused = fused
        return self.Y[-1]

    def backward(self, x: torch.Tensor, d_out_feat: Optional[torch.Tensor] = None):
        """Consumes self.dY[-1] (d loss / d logits) and, for the auxiliary distillation losses, d loss / d out_feat
        ([N, H], added to the gradient arriving at the last hidden activation); fills self.grads."""
        fused = self._fwd_fused
        for l in range(self.L - 1, -1, -1):
            act = self._act(l - 1) if fused and l > 0 else None
            inp = x if l == 0 else (None if act else self._A[l - 1])
            if l == self.L - 1:
                ops.col_sum(self.dY[l], out=self.gb[l], partial=self._part(self.dims[l + 1]))
            if l == 0 and self.agg_first:
                self._wgrad_async(0, self.AX, self.dY[0])              # dW0 = (ÂX)ᵀ dY0, no backward aggregation
                continue
            ops.spmm_csr(self.Gt, self.dY[l], "sum", out=self.dH[l])
            d_prev = self.dA[l - 1] if l > 0 else None
            gp = self._gemm_part.get(self.dims[l]) if l > 0 else None
            if l > 0:
                acc = d_out_feat is not None and l == self.L - 1
                if acc:
                    # the auxiliary loss's gradient w.r.t. out_feat is the starting value the input-gradient GEMM adds to
                    d_prev = d_out_feat
                if gp is not None:
                    # dgrad GEMM whose epilogue masks by the ReLU/dropout pattern, stores dz and reduces the two BatchNorm
                    # backward column sums: pass 1 of the block's backward costs no sweep of its own
                    hi, lo = ops.split_tf32(self.W[l], transpose=False, hi=self.W_split[l][0], lo=self.W_split[l][1])
                    if act:
                        ops.gemm_tf32x3_bnbwd_bits(self.dH[l], hi, lo, d_prev, act[3], self.Y[l - 1], self.bn[l - 1][0],
                                                   self.bn[l - 1][1], act[1], act[2], self.p, gp, accumulate=acc)
                    else:
                        ops.gemm_tf32x3_bnbwd(self.dH[l], hi, lo, d_prev, self._A[l - 1], self.Y[l - 1], self.bn[l - 1][0],
                                              self.bn[l - 1][1], self.p, gp, accumulate=acc)
                else:
                    self._linear_dgrad(l, self.dH[l], d_prev, accumulate=acc)
            self._wgrad_async(l, inp, self.dH[l], act=act)             # forks after the dgrad GEMM (both want the whole SM)
            if l > 0:
                k = self.dims[l]
                part = self._part(k)
                if gp is not None:
                    ops.bn_act_bwd_apply(d_prev, None, self.Y[l - 1], self.bn[l - 1][0], self.bn[l - 1][1], self.gamma[l - 1],
                                         gp, self.N, self.p, self.dY[l - 1], self.ggamma[l - 1], self.gbeta[l - 1],
                                         self.gb[l - 1], part, self._coef(k))
                else:
                    ops.bn_act_bwd(d_prev, self._A[l - 1], self.Y[l - 1], self.bn[l - 1][0], self.bn[l - 1][1],
                                   self.gamma[l - 1], self.p, d_y=self.dY[l - 1], d_gamma=self.ggamma[l - 1],
                                   d_beta=self.gbeta[l - 1], d_bias=self.gb[l - 1], partial=part, coef=self._coef(k))
        self._wgrad_join()

    def _wgrad_async(self, l: int, inp: Optional[torch.Tensor], d_out: torch.Tensor, act=None):
        """grad W_l on the side stream, ordered after everything enqueued so far on the current stream."""
        if self._side is None:
            return self._linear_wgrad(l, inp, d_out, act)
        self._ev_fork.record(torch.cuda.current_stream())
        self._side.wait_event(self._ev_fork)
        with torch.cuda.stream(self._side):
            self._linear_wgrad(l, inp, d_out, act)

    def _wgrad_join(self):
        if self._side is not None:
            self._ev_join.record(self._side)
            torch.cuda.current_stream().wait_event(self._ev_join)

    def _linear(self, l: int, inp: Optional[torch.Tensor], out: torch.Tensor, bias: Optional[torch.Tensor] = None, act=None):
        """out = inp @ W_l (+bias): wgmma 3xTF32 kernel, or cuBLAS fp32 when disabled.  act = (Y, scale, shift, bits): inp is
        the activation formed from those inside the GEMM."""
        if act is not None:
            hi, lo = ops.split_tf32(self.W[l], transpose=True, hi=self.Wt_split[l][0], lo=self.Wt_split[l][1])
            ops.gemm_tf32x3_act(*act, self.p, hi, lo, bias=bias, out=out)
        elif self.tc_gemm:
            hi, lo = ops.split_tf32(self.W[l], transpose=True, hi=self.Wt_split[l][0], lo=self.Wt_split[l][1])
            ops.gemm_tf32x3(inp, hi, lo, bias=bias, out=out)
        elif bias is not None:
            torch.addmm(bias, inp, self.W[l], out=out)
        else:
            torch.mm(inp, self.W[l], out=out)

    def _linear_dgrad(self, l: int, d_out: torch.Tensor, d_inp: torch.Tensor, accumulate: bool = False):
        """d_inp (+)= d_out @ W_l^T."""
        if self.tc_gemm:
            hi, lo = ops.split_tf32(self.W[l], transpose=False, hi=self.W_split[l][0], lo=self.W_split[l][1])
            ops.gemm_tf32x3(d_out, hi, lo, out=d_inp, accumulate=accumulate)
        elif accumulate:
            d_inp.addmm_(d_out, self.W[l].t())
        else:
            torch.mm(d_out, self.W[l].t(), out=d_inp)

    def _linear_wgrad(self, l: int, inp: Optional[torch.Tensor], d_out: torch.Tensor, act=None):
        """grad W_l = inp^T @ d_out: split-K wgmma kernel where the tiling allows, cuBLAS fp32 otherwise; act as in _linear."""
        if act is not None:
            ops.gemm_wgrad_tf32x3_act(*act, self.p, d_out, out=self.gW[l], workspace=self.wgrad_ws)
        elif self.tc_gemm and ops.wgrad_supported(self.dims[l], self.dims[l + 1]):
            ops.gemm_wgrad_tf32x3(inp, d_out, out=self.gW[l], workspace=self.wgrad_ws)
        else:
            torch.mm(inp.t(), d_out, out=self.gW[l])

    def replay(self, key: int = 0) -> torch.Tensor:
        super().replay(key)
        self._act_stale = self.fuse_act
        return self.loss_out

    # ------------------------------------------------------------------ accounting
    def aggregations_per_step(self) -> Dict[int, int]:
        """width -> number of SpMM launches of that width in one training step."""
        out: Dict[int, int] = {}
        for l in range(self.L):
            if l == 0 and self.agg_first:
                out[self.dims[0]] = out.get(self.dims[0], 0) + 1
            else:
                out[self.dims[l + 1]] = out.get(self.dims[l + 1], 0) + 2
        return out

    def spmm_algorithmic_bytes(self) -> Dict[int, int]:
        """Compulsory HBM bytes of one aggregation per feature width (SURVEY.md §8d):
        2*N*K*4 (read X, write Y) + nnz*(4 col + 4 val) + (N+1)*4."""
        return {k: 2 * self.N * k * 4 + self.nnz * 8 + (self.N + 1) * 4 for k in set(self.dims)}
