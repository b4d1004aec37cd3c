"""GAT teacher layer across P GPUs (BASELINE.json configs[3] "GAT teacher 8-head edge-softmax ... 1→8×H100"; SURVEY.md §8e).

SURVEY §8e sketched a node-parallel scheme with a source-side halo of ``ft`` and ``el`` and a non-symmetric backward.  The
hybrid layout of hybrid.py makes all of that unnecessary: attention is computed PER HEAD, so with the columns of the projected
features split head-aligned (rank p owns heads [p·H/P, (p+1)·H/P) of ALL nodes, "C layout") the whole attention block of
arxiv_dgl/models.py:196-217 — ``el``/``er``, LeakyReLU, edge softmax over incoming edges, the weighted multi-head aggregation,
the symmetric degree scaling, and their hand-written backward (csrc/gat.cu) — runs on each rank for its own heads over the
whole (replicated, 30 MB) graph with NO halo and no cross-rank reduction.  Only the dense projections stay node-parallel
("R layout"), and the two layouts are connected by the same R<->C exchanges as the GCN engine:

    feat_R ──fc (wgmma)──▶ ft_R [n_p, H·D] ──R→C──▶ ft_C [N, (H/P)·D] ──attention + aggregation on own heads──▶ rst_C ──C→R──▶ rst_R
    rst_R += res_fc(feat_R)                                                                       (models.py:228-230)

Exchanged per layer and direction: N·H·D·4·(P−1)/P² bytes per rank (8× less than gathering ``ft`` at P = 8).  Autograd:
the backward of an R→C exchange is the C→R exchange of the gradient and vice versa.  Parameters are replicated; ``attn_l`` /
``attn_r`` receive gradients only for the rank's own heads and the dense weights only from the rank's own rows, so gradients
are summed over ranks (``allreduce_grads``) before the optimizer step, as for any data-parallel replica.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from . import nn as bnn
from .hybrid import DensePlan, PeerExchange, TorchExchange
from .sparse import SparseTensor


class _Exchange(torch.autograd.Function):
    """direction 0: R->C forward (C->R backward); direction 1: C->R forward (R->C backward)."""

    @staticmethod
    def forward(ctx, src, layer, direction: int):
        ctx.layer, ctx.direction = layer, direction
        return layer._run(src.contiguous(), direction, grad=False)

    @staticmethod
    def backward(ctx, g):
        return ctx.layer._run(g.contiguous(), 1 - ctx.direction, grad=True), None, None


class HeadParallelGATConv(torch.nn.Module):
    """The reference's DGL GATConv (arxiv_dgl/models.py:95-236) on P GPUs: same parameters and state_dict keys as
    nn.DGLGATConv (fc, attn_l, attn_r, res_fc); ``forward(adj_rel, feat_R)`` takes the RELABELLED full adjacency
    (hybrid.relabel) and this rank's rows of the input, returns this rank's rows of the output [n_p, H, D]."""

    _count = 0

    def __init__(self, in_feats: int, out_feats: int, num_heads: int, plan: DensePlan, rank: int, exchange, negative_slope=0.2,
                 use_attn_dst=True, residual=False, activation=None, use_symmetric_norm=False):
        super().__init__()
        P = plan.world
        if num_heads % P:
            raise ValueError(f"head-parallel GAT needs num_heads ({num_heads}) divisible by the world size ({P})")
        if (num_heads // P) * out_feats % 4:
            raise ValueError("per-rank column slice must be a multiple of 4 floats")
        self.plan, self.rank, self.ex = plan, rank, exchange
        self._num_heads, self._out_feats, self._slope = num_heads, out_feats, negative_slope
        self._h_loc = num_heads // P
        self._use_symmetric_norm, self._activation = use_symmetric_norm, activation
        self.fc = bnn.Linear(in_feats, out_feats * num_heads, bias=False)
        self.attn_l = torch.nn.Parameter(torch.empty(1, num_heads, out_feats))
        self.attn_r = torch.nn.Parameter(torch.empty(1, num_heads, out_feats)) if use_attn_dst else None
        self.res_fc = bnn.Linear(in_feats, num_heads * out_feats, bias=False) if residual else None
        gain = torch.nn.init.calculate_gain("relu")
        torch.nn.init.xavier_normal_(self.fc.weight, gain=gain)
        torch.nn.init.xavier_normal_(self.attn_l, gain=gain)
        if self.attn_r is not None:
            torch.nn.init.xavier_normal_(self.attn_r, gain=gain)
        if self.res_fc is not None:
            torch.nn.init.xavier_normal_(self.res_fc.weight, gain=gain)
        HeadParallelGATConv._count += 1
        self._tag = f"gat{HeadParallelGATConv._count}"
        self._bufs = {}

    # -- exchange plumbing (destination buffers are allocated once; peer exchanges need them inside the arena)
    def _buffer(self, key: str, shape, device):
        b = self._bufs.get(key)
        if b is None:
            b = self._bufs[key] = self.ex.buffer(f"{self._tag}_{key}", shape, device)
        return b

    def _run(self, src: torch.Tensor, direction: int, grad: bool) -> torch.Tensor:
        N, K = self.plan.n, self._num_heads * self._out_feats
        kc, n_p, B = K // self.plan.world, self.plan.counts[self.rank], self.plan.block
        key = ("g" if grad else "f") + ("r2c" if direction == 0 else "c2r")
        if direction == 0:
            dst = self._buffer(key, (N, kc), src.device)
            self.ex.r2c(src, dst, f"{self._tag}_{key}")
            return dst.clone()           # the exchange buffer is reused by the next call: hand autograd its own copy
        dst = self._buffer(key, (B, K), src.device)[:n_p]
        self.ex.c2r(src, dst, f"{self._tag}_{key}")
        return dst.clone()

    def forward(self, adj_rel: SparseTensor, feat_R: torch.Tensor):
        H, D, HL = self._num_heads, self._out_feats, self._h_loc
        h0 = self.rank * HL
        ft_R = self.fc(feat_R)                                                   # [n_p, H*D]   node-parallel GEMM
        ft_C = _Exchange.apply(ft_R, self, 0).view(-1, HL, D)                    # [N, HL, D]   my heads, all nodes
        ft_dst = ft_C                                                            # models.py:187-188: er from the raw projection
        st = adj_rel.storage
        if self._use_symmetric_norm:
            out_deg = torch.bincount(st.col(), minlength=adj_rel.size(1)).float().clamp(min=1)
            ft_C = ft_C * out_deg.pow(-0.5).view(-1, 1, 1)
        el = (ft_C * self.attn_l[:, h0:h0 + HL]).sum(-1)
        er = (ft_dst * self.attn_r[:, h0:h0 + HL]).sum(-1) if self.attn_r is not None else None
        rst_C = bnn.gat_aggregate(ft_C.reshape(-1, HL * D), el, er, adj_rel, HL, self._slope, 0.0)
        if self._use_symmetric_norm:
            rst_C = rst_C * st.rowcount().float().clamp(min=1).pow(0.5).view(-1, 1)
        rst = _Exchange.apply(rst_C, self, 1).view(-1, H, D)                     # [n_p, H, D]  my nodes, all heads
        if self.res_fc is not None:
            rst = rst + self.res_fc(feat_R).view(feat_R.shape[0], -1, D)
        return self._activation(rst) if self._activation is not None else rst

    def allreduce_grads(self, group=None):
        """Sum the parameter gradients over the ranks (own rows / own heads contribute; everything else is zero)."""
        for p in self.parameters():
            if p.grad is None:
                p.grad = torch.zeros_like(p)
            dist.all_reduce(p.grad, group=group)
