"""Full-batch R-GCN engine — ``RGCN.inference`` of the reference (mag_pyg/gnn.py:140-171), BASELINE.json configs[4]
("R-GCN teacher ... MAG-shape heterogeneous ... node-parallel 2/4/8×H100").

Per layer and node type t (the reference's loop, :153-169):

    out[t]  = root_lins[t](x[t])                                          one GEMM per node type
    out[t] += rel_lins[r]( mean_{j in N_r(i)} x[src(r)][j] )              per relation r = (src, ·, t): rectangular mean-SpMM,
                                                                          then a GEMM that ACCUMULATES into out[t]
    x = relu(out)  between layers

What differs from the reference's execution (not from its arithmetic): the per-relation CSR is built ONCE by the device
ingestion kernels (the reference re-sorts every relation on every call, :149-151); the relation GEMMs add into ``out[t]``
through the accumulating wgmma epilogue (``b200gnn_gemm_tf32x3_acc_f32``) instead of materialising ``rel_lins(tmp)`` and
an ``add_``; aggregation runs before the transform, as in the reference's inference (its training path transforms per EDGE).

Multi-GPU (``exchange`` given): same hybrid layout as hybrid.py, per node type — activations live node-parallel ("R": rank p
owns rows [off_t[p], off_t[p+1]) of every type, contiguous blocks, no relabelling: column-split aggregations are balanced by
construction), every aggregation runs feature-parallel ("C": rank p owns columns [p·F/P, (p+1)·F/P) of ALL nodes of the
source type) on the whole replicated relation graph, one R→C exchange per node type and one C→R exchange per relation per
layer; the GEMMs see only local rows.  Results equal the single-GPU engine up to fp32 reassociation of the column split.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch

from . import lib, ops
from .hybrid import DensePlan
from .sparse import SparseTensor


def _block_plan(n: int, world: int) -> DensePlan:
    """Contiguous equal row blocks of one node type (identity relabelling)."""
    base, rem = divmod(n, world)
    counts = [base + (1 if q < rem else 0) for q in range(world)]
    offs = [0]
    for c in counts:
        offs.append(offs[-1] + c)
    ar = torch.arange(n)
    return DensePlan(world, n, counts, offs, ar, ar)


class RGCNInference:
    """state: the reference module's state_dict (``convs.{i}.rel_lins.{r}.weight`` [out,in], ``convs.{i}.root_lins.{t}.weight``
    / ``.bias``, ``emb_dict.{t}``); edge_index_dict: {(src_key, name, dst_key): [2, E] (row 0 = source)}; key2int as the
    reference builds it (node-type keys and relation triples -> ints)."""

    def __init__(self, state: Dict[str, torch.Tensor], num_nodes: Dict[int, int], edge_index_dict, key2int, device="cuda",
                 exchange_factory=None, rank: int = 0, world: int = 1):
        self.dev = torch.device(device)
        self.key2int = key2int
        self.num_nodes = {int(k): int(v) for k, v in num_nodes.items()}
        self.n_layers = 1 + max(int(k.split(".")[1]) for k in state if k.startswith("convs."))
        self.rank, self.world = rank, world
        f32 = lambda t: t.detach().to(self.dev, torch.float32).contiguous()
        self.emb = {int(k.split(".")[1]): f32(v) for k, v in state.items() if k.startswith("emb_dict.")}
        self.layers = []
        for i in range(self.n_layers):
            rel = {int(k.split(".")[3]): f32(v) for k, v in state.items() if k.startswith(f"convs.{i}.rel_lins.") and k.endswith(".weight")}
            root_w = {int(k.split(".")[3]): f32(v) for k, v in state.items() if k.startswith(f"convs.{i}.root_lins.") and k.endswith(".weight")}
            root_b = {int(k.split(".")[3]): f32(v) for k, v in state.items() if k.startswith(f"convs.{i}.root_lins.") and k.endswith(".bias")}
            self.layers.append((rel, root_w, root_b))
        # relation graphs: rows = destination nodes, cols = source nodes, built once (device ingestion kernels)
        self.rels: List[Tuple[int, int, int, SparseTensor]] = []
        for keys, ei in edge_index_dict.items():
            s, d, r = key2int[keys[0]], key2int[keys[-1]], key2int[keys]
            ei = ei.to(self.dev)
            adj = SparseTensor(row=ei[1], col=ei[0], sparse_sizes=(self.num_nodes[d], self.num_nodes[s]), is_sorted=False)
            adj.storage.engine_csr_unweighted()
            self.rels.append((s, d, r, adj))
        self.nnz = sum(a.nnz() for *_, a in self.rels)
        # multi-GPU plumbing
        self.plans = {t: _block_plan(n, world) for t, n in self.num_nodes.items()}
        self.ex = {t: exchange_factory(self.plans[t]) for t in self.num_nodes} if (world > 1 and exchange_factory) else None
        self._bufs: Dict[str, torch.Tensor] = {}

    # ------------------------------------------------------------------ helpers
    def _gemm(self, x: torch.Tensor, w: torch.Tensor, out: torch.Tensor, bias=None, accumulate=False):
        """out (+)= x @ w^T (+bias) on the wgmma GEMM; K not a multiple of 4 is zero-padded (exact)."""
        k = x.shape[1]
        if k % 4:
            pad = 4 - k % 4
            x = torch.nn.functional.pad(x, (0, pad)).contiguous()
            w = torch.nn.functional.pad(w, (0, pad)).contiguous()
        hi, lo = ops.split_tf32(w)
        if accumulate:
            ops.gemm_tf32x3(x, hi, lo, out=out, accumulate=True)
        else:
            ops.gemm_tf32x3(x, hi, lo, bias=bias, out=out)

    def _buf(self, key: str, shape, ex=None) -> torch.Tensor:
        b = self._bufs.get(key)
        if b is None or tuple(b.shape) != tuple(shape):
            b = self._bufs[key] = (ex.buffer(key, shape, self.dev) if ex is not None else torch.empty(*shape, device=self.dev))
        return b

    def rows_of(self, t: int):
        return self.plans[t].rows_of(self.rank)

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def __call__(self, x_dict: Dict[int, torch.Tensor]) -> Dict[int, torch.Tensor]:
        """x_dict: features of the node types that have them (int keys), FULL matrices; embedding tables fill the rest
        (mag_pyg/gnn.py:145-147).  Returns {type: [n_t, out]} on one GPU, this rank's row blocks on several."""
        x = {int(k): v.to(self.dev, torch.float32).contiguous() for k, v in x_dict.items()}
        x.update(self.emb)
        if self.world > 1:
            x = {t: v[self.rows_of(t)[0]:self.rows_of(t)[1]].contiguous() for t, v in x.items()}
        for i, (rel_w, root_w, root_b) in enumerate(self.layers):
            f_out = next(iter(root_w.values())).shape[0]
            out = {}
            for t, xt in x.items():
                o = self._buf(f"out{i}_{t}", (xt.shape[0], f_out))
                self._gemm(xt, root_w[t], o, bias=root_b[t])
                out[t] = o
            if self.world == 1:
                for s, d, r, adj in self.rels:
                    agg = adj.matmul(x[s], reduce="mean")                            # [n_d, F]
                    self._gemm(agg, rel_w[r], out[d], accumulate=True)
            else:
                P = self.world
                f_in = next(iter(x.values())).shape[1]
                if f_in % (4 * P):
                    raise lib.B200GnnError(f"feature width {f_in} must be a multiple of 4*world for the column layout")
                kc = f_in // P
                xc = {}
                for t, xt in x.items():                                              # R -> C, once per node type
                    dst = self._buf(f"xc{i}_{t}", (self.num_nodes[t], kc), self.ex[t])
                    self.ex[t].r2c(xt, dst, f"xc{i}_{t}")
                    xc[t] = dst
                for s, d, r, adj in self.rels:
                    agg_c = adj.matmul(xc[s], reduce="mean")                         # [n_d, F/P]: my columns, all destinations
                    n_p = self.plans[d].counts[self.rank]
                    dst = self._buf(f"agg{i}_{r}", (self.plans[d].block, f_in), self.ex[d])[:n_p]
                    self.ex[d].c2r(agg_c, dst, f"agg{i}_{r}")                        # C -> R: my destinations, all columns
                    self._gemm(dst, rel_w[r], out[d], accumulate=True)
            if i != self.n_layers - 1:
                for o in out.values():
                    o.relu_()
            x = out
        return x

    def gather(self, x_loc: Dict[int, torch.Tensor]) -> Dict[int, torch.Tensor]:
        """All ranks' row blocks -> full matrices (evaluation / tests; torch.distributed)."""
        import torch.distributed as dist
        if self.world == 1:
            return x_loc
        full = {}
        for t, v in x_loc.items():
            f = torch.empty(self.num_nodes[t], v.shape[1], device=v.device)
            dist.all_to_all_single(f, v.contiguous().repeat(self.world, 1), output_split_sizes=self.plans[t].counts,
                                   input_split_sizes=[v.shape[0]] * self.world)
            full[t] = f
        return full
