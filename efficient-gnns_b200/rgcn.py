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

import math
from typing import Dict, List, Optional, Tuple

import torch

from . import lib, ops
from .hybrid import DensePlan
from .sparse import SparseTensor, csr_graph_from, device_argsort
from .trainer import FlatParams, aux_grad, one_objective


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


# ============================================================================ training on GraphSAINT batches
def relation_types(edge_index_dict, key2int) -> Dict[int, Tuple[int, int]]:
    """relation id -> (source node type, destination node type), from the keys main() builds (mag_pyg/gnn.py:320-347)."""
    return {int(key2int[k]): (int(key2int[k[0]]), int(key2int[k[-1]])) for k in edge_index_dict}


class BatchPlan:
    """Aggregation plan of one sampled batch (built on the batch's device; torch glue around the radix argsort).

    * ``perm`` [N]: internal row r holds batch node perm[r]; node types are contiguous, type t at rows [off[t], off[t]+cnt[t])
      (stable within a type); ``pos`` is the inverse.
    * Virtual rows: type t owns rows [vbase[t], vbase[t] + cnt[t]·(1+R_t)) of one arena; row vbase[t] + a·(1+R_t) + k is
      slot k of the a-th node of type t: slot 0 = the node itself, slot k >= 1 = the in-edges of the k-th relation into t
      (relations of t in increasing id).  Read as [cnt[t], (1+R_t)·F] the arena block of type t is Acat_t = [X_t | mean_r1 | ...].
    * Forward CSR (rows = virtual rows, cols = internal rows, no values: mean reduce).  Duplicate edges are kept: the
      reference's scatter-mean counts them.  Entries of a row keep the batch's edge order.
    * Backward CSR: its transpose (rows = internal rows, cols = virtual rows, sorted by column), values 1/deg of the
      virtual row (1 for slot 0)."""

    def __init__(self, edge_index, edge_type, node_type, rel_src, rel_dst, n_types: int):
        dev = node_type.device
        N = int(node_type.numel())
        R = int(rel_src.numel())
        nt = node_type.view(-1).long()
        et = edge_type.view(-1).long()
        src, dst = edge_index[0].long(), edge_index[1].long()
        if et.numel():
            bad = (et < 0) | (et >= R)
            ok_et = et.clamp(0, max(R - 1, 0))
            bad |= (nt[src] != rel_src[ok_et]) | (nt[dst] != rel_dst[ok_et])
            if bool(bad.any()):
                raise lib.B200GnnError("R-GCN batch plan: an edge's type does not match its relation's fixed (source type, "
                                       "destination type) pair (aggregating before the transform needs one pair per relation)")
        if nt.numel() and (int(nt.min()) < 0 or int(nt.max()) >= n_types):
            raise lib.B200GnnError("R-GCN batch plan: node type out of range")
        # slot of every relation within its destination type (1-based), relations per type
        dst_of = rel_dst.tolist()
        self.rels_of = [[r for r in range(R) if dst_of[r] == t] for t in range(n_types)]
        slot = torch.zeros(max(R, 1), dtype=torch.long)
        for rels in self.rels_of:
            for k, r in enumerate(rels):
                slot[r] = k + 1
        width = torch.tensor([1 + len(r) for r in self.rels_of], dtype=torch.long)
        slot, width_d = slot.to(dev), width.to(dev)

        self.N, self.n_types = N, n_types
        self.perm = device_argsort(nt, torch.zeros_like(nt), n_types, 1)
        self.pos = torch.empty_like(self.perm)
        self.pos[self.perm] = torch.arange(N, device=dev)
        cnt = torch.bincount(nt, minlength=n_types)
        self.cnt = [int(c) for c in cnt.tolist()]
        self.off = [0]
        for c in self.cnt:
            self.off.append(self.off[-1] + c)
        self.width = width.tolist()
        self.vbase = [0]
        for t in range(n_types):
            self.vbase.append(self.vbase[-1] + self.cnt[t] * self.width[t])
        self.V = self.vbase[-1]
        off_d = torch.tensor(self.off[:-1], dtype=torch.long, device=dev)
        vbase_d = torch.tensor(self.vbase[:-1], dtype=torch.long, device=dev)

        # virtual row of every self entry (internal row i) and every edge
        nt_int = nt[self.perm]
        ar = torch.arange(N, device=dev)
        v_self = vbase_d[nt_int] + (ar - off_d[nt_int]) * width_d[nt_int]
        dt = nt[dst]
        v_edge = vbase_d[dt] + (self.pos[dst] - off_d[dt]) * width_d[dt] + slot[et]
        vrow = torch.cat([v_self, v_edge])
        col = torch.cat([ar, self.pos[src]])
        order = device_argsort(vrow, torch.zeros_like(vrow), max(self.V, 1), 1)
        f_row, self.f_col = vrow[order], col[order]
        deg = torch.bincount(f_row, minlength=self.V)
        self.f_rowptr = torch.zeros(self.V + 1, dtype=torch.long, device=dev)
        torch.cumsum(deg, 0, out=self.f_rowptr[1:])
        # transpose: sorted by (internal column, virtual row)
        order_t = device_argsort(self.f_col, f_row, max(N, 1), max(self.V, 1))
        self.b_col = f_row[order_t]
        self.b_val = 1.0 / deg[self.b_col].to(torch.float32)
        self.b_rowptr = torch.zeros(N + 1, dtype=torch.long, device=dev)
        torch.cumsum(torch.bincount(self.f_col, minlength=N), 0, out=self.b_rowptr[1:])
        # the rows of each type, internal order (typed gather / embedding gradient)
        self.node_type_int = nt_int.contiguous()

    def graphs(self):
        """Engine CSR views (device): forward (mean, no values) and backward (sum, 1/deg values)."""
        fwd = csr_graph_from(self.f_rowptr, self.f_col, None, self.V, self.N)
        bwd = csr_graph_from(self.b_rowptr, self.b_col, self.b_val, self.N, self.V)
        return fwd, bwd


class RGCNTrainer:
    """Fused training step of the reference's ``RGCN`` (mag_pyg/gnn.py:26-137) on GraphSAINT batches — the loop body of
    ``train()`` (:174-268): R-GCN teacher (3 x 512) or student (2 x 32) on ogbn-mag, supervised or logit-KD.

    Per layer, aggregation runs before the transform (mean is linear: mean_j(W x_j) = W mean_j(x_j)): ONE mean-SpMM over
    the batch plan writes Acat_t = [X_t | mean_r1 | mean_r2 | ...] for every node type t, then one wgmma GEMM per type
    ``out_t = Acat_t · [Wroot_t | W_r1 | ...]^T + b_t``.  Backward: per type the bias column sum, the split-K weight gradient
    dWcat_t = Acat_t^T dOut_t and the input gradient dAcat_t = dOut_t Wcat_t into one arena, then ONE SpMM over the
    transposed plan gives dX of every node.  Layer-0 dX feeds the embedding tables through an Adam that consumes the batch's
    rows directly (no dense gradient of the 154 M embedding parameters).

    Parameters other than the embeddings live in one flat buffer; per (layer, type) the block Wcat_t^T [(1+R_t)·F_in, F_out']
    (F_out' = F_out rounded up to 4 — 349 classes are stored as 352 with zero columns) and b_t [F_out'].
    Dropout: Philox masks of ``affine_relu_dropout`` indexed by the batch's node order, offset ``layer + step·L`` (the
    reference's forward hard-codes p = 0.5; its callers pass dropout = 0.5)."""

    def __init__(self, in_channels: int, hidden_channels: int, out_channels: int, num_layers: int, dropout: float,
                 num_nodes_dict: Dict[int, int], x_types, num_edge_types: int, relations: Dict[int, Tuple[int, int]],
                 lr: float = 0.01, seed: int = 0, alpha: float = 0.9, kd_T: float = 4.0, device="cuda", lsp=None,
                 gcrd=None, gsp=None):
        """lsp: an lsp.BatchLSP run inside every step (the reference's ``--training lpw``); gcrd: a gcrd.BatchGCRD, the same
        way (``--training nce``); gsp: a gsp.BatchGSP (``--training gpw``).  At most one of them; their steps take
        ``teacher=``."""
        one_objective(gcrd=gcrd, lsp=lsp, gsp=gsp)
        self.dev = torch.device(device)
        self.F_in, self.H, self.C, self.L = int(in_channels), int(hidden_channels), int(out_channels), int(num_layers)
        self.p, self.lr, self.alpha, self.kd_T, self.seed = float(dropout), float(lr), float(alpha), float(kd_T), int(seed)
        self.num_nodes = {int(k): int(v) for k, v in num_nodes_dict.items()}
        self.T = len(self.num_nodes)
        if sorted(self.num_nodes) != list(range(self.T)):
            raise lib.B200GnnError("node types must be 0..T-1 (key2int order)")
        self.x_types = sorted(int(t) for t in x_types)
        self.R = int(num_edge_types)
        if sorted(int(r) for r in relations) != list(range(self.R)):
            raise lib.B200GnnError("relations must map every edge type 0..R-1 to its (source type, destination type)")
        self.relations = tuple((int(relations[r][0]), int(relations[r][1])) for r in range(self.R))
        self.rel_src = torch.tensor([int(relations[r][0]) for r in range(self.R)], dtype=torch.long, device=self.dev)
        self.rel_dst = torch.tensor([int(relations[r][1]) for r in range(self.R)], dtype=torch.long, device=self.dev)
        self.rels_of = [[r for r in range(self.R) if int(relations[r][1]) == t] for t in range(self.T)]
        self.dims = [self.F_in] + [self.H] * (self.L - 1) + [self.C]
        self.dims_pad = [d + (-d) % 4 for d in self.dims]
        if any(d % 4 for d in self.dims[:-1]):
            raise lib.B200GnnError("input and hidden widths must be multiples of 4")

        # ---- flat parameters: per layer, per node type, WcatT [(1+R_t)·F_in, F_out'] then b [F_out']
        shapes = []
        for i in range(self.L):
            fi, fo = self.dims_pad[i], self.dims_pad[i + 1]
            for t in range(self.T):
                shapes += [((1 + len(self.rels_of[t])) * fi, fo), (fo,)]
        self.store = FlatParams(shapes, self.dev).attach(self)
        params = iter(p for p, _ in self.store.views)
        self._wcat, self._b = [], []               # [layer][type] -> view of params
        for i in range(self.L):
            row = [(next(params), next(params)) for _ in range(self.T)]
            self._wcat.append([w for w, _ in row]); self._b.append([b for _, b in row])
        # embedding tables of the types without features, with their Adam moments and the row-head scratch
        self.emb = {t: torch.zeros(n, self.F_in, device=self.dev) for t, n in self.num_nodes.items() if t not in self.x_types}
        self.emb_m = {t: torch.zeros_like(e) for t, e in self.emb.items()}
        self.emb_v = {t: torch.zeros_like(e) for t, e in self.emb.items()}
        self._head = torch.full((max([e.shape[0] for e in self.emb.values()] + [1]),), -1, dtype=torch.int32, device=self.dev)
        self.wgrad_ws = torch.empty(max(ops.wgrad_workspace_floats(*w.shape) for row in self._wcat for w in row), device=self.dev)
        self.reset_parameters(seed)
        self._fwd = None
        self._training = False
        self.lsp, self.gcrd, self.gsp = lsp, gcrd, gsp
        for o in (lsp, gcrd, gsp):
            if o is not None:
                o.bind(self)

    # ------------------------------------------------------------------ parameters
    def _wcatT(self, i: int, t: int, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        w = self._wcat[i][t]
        return w if buf is None else self.store.like(buf, w)

    def _bias(self, i: int, t: int, buf: Optional[torch.Tensor] = None) -> torch.Tensor:
        b = self._b[i][t]
        return b if buf is None else self.store.like(buf, b)

    def _blocks(self, i: int, t: int, buf=None):
        """(root weight [F_out, F_in], {relation: weight [F_out, F_in]}, bias [F_out]) as views of the flat buffer."""
        w = self._wcatT(i, t, buf)
        fi, fo = self.dims_pad[i], self.dims[i + 1]
        root = w[:fi, :fo].t()
        rel = {r: w[(k + 1) * fi:(k + 2) * fi, :fo].t() for k, r in enumerate(self.rels_of[t])}
        return root, rel, self._bias(i, t, buf)[:fo]

    def reset_parameters(self, seed: int = 0):
        """The reference's reset_parameters: xavier_uniform_ embeddings, nn.Linear defaults (kaiming_uniform_(a=sqrt(5)) weights,
        U(±1/sqrt(fan_in)) biases) for rel_lins and root_lins."""
        g = torch.Generator().manual_seed(int(seed))
        for t in sorted(self.emb):
            n = self.emb[t].shape[0]
            a = math.sqrt(6.0 / (n + self.F_in))
            self.emb[t].copy_((torch.rand(n, self.F_in, generator=g) * 2 - 1) * a)
        self.params.zero_()
        for i in range(self.L):
            fi, fo = self.dims[i], self.dims[i + 1]
            bound = 1.0 / math.sqrt(fi)
            ws = {}
            for r in range(self.R):
                ws[("rel", r)] = (torch.rand(fo, fi, generator=g) * 2 - 1) * bound
            for t in range(self.T):
                ws[("root", t)] = ((torch.rand(fo, fi, generator=g) * 2 - 1) * bound, (torch.rand(fo, generator=g) * 2 - 1) * bound)
            for t in range(self.T):
                root, rel, b = self._blocks(i, t)
                root.copy_(ws[("root", t)][0]); b.copy_(ws[("root", t)][1])
                for r, w in rel.items():
                    w.copy_(ws[("rel", r)])
        self.exp_avg.zero_(); self.exp_avg_sq.zero_(); self.step_count.zero_()
        for t in self.emb:
            self.emb_m[t].zero_(); self.emb_v[t].zero_()

    def state_dict(self) -> Dict[str, torch.Tensor]:
        """Keys of the reference's RGCN module: emb_dict.{t}, convs.{i}.rel_lins.{r}.weight, convs.{i}.root_lins.{t}.weight|bias."""
        return self._named(None, {t: e for t, e in self.emb.items()})

    def _named(self, buf, emb) -> Dict[str, torch.Tensor]:
        sd = {f"emb_dict.{t}": e.detach().clone() for t, e in emb.items()}
        for i in range(self.L):
            for t in range(self.T):
                root, rel, b = self._blocks(i, t, buf)
                sd[f"convs.{i}.root_lins.{t}.weight"] = root.clone()
                sd[f"convs.{i}.root_lins.{t}.bias"] = b.clone()
                for r, w in rel.items():
                    sd[f"convs.{i}.rel_lins.{r}.weight"] = w.clone()
        return sd

    def load_state_dict(self, sd: Dict[str, torch.Tensor]):
        for t, e in self.emb.items():
            e.copy_(sd[f"emb_dict.{t}"])
        for i in range(self.L):
            for t in range(self.T):
                root, rel, b = self._blocks(i, t)
                root.copy_(sd[f"convs.{i}.root_lins.{t}.weight"]); b.copy_(sd[f"convs.{i}.root_lins.{t}.bias"])
                for r, w in rel.items():
                    w.copy_(sd[f"convs.{i}.rel_lins.{r}.weight"])

    # ------------------------------------------------------------------ batch plan
    def plan(self, batch) -> BatchPlan:
        return BatchPlan(batch.edge_index, batch.edge_attr, batch.node_type, self.rel_src, self.rel_dst, self.T)

    # ------------------------------------------------------------------ forward / backward
    def forward(self, batch, x_dict: Dict[int, torch.Tensor], training: bool = True,
                plan: Optional[BatchPlan] = None) -> torch.Tensor:
        """Logits [n_batch, C] in the batch's node order; ``training=False``: no dropout (the teacher's eval forward).
        ``plan``: the batch's BatchPlan when the caller already has it (a teacher running on its student's plan)."""
        self._training = bool(training)
        P = self.plan(batch) if plan is None else plan
        G, Gt = P.graphs()
        li_int = batch.local_node_idx.view(-1).long()[P.perm].contiguous()
        tables = {int(t): v for t, v in x_dict.items()}
        tables.update(self.emb)
        x = torch.empty(P.N, self.F_in, device=self.dev)
        ops.typed_gather(tables, self.T, P.node_type_int, li_int, x)
        rowmap = P.perm.to(torch.int32)
        xs, arenas, ys = [x], [], []
        for i in range(self.L):
            fi, fo = self.dims_pad[i], self.dims_pad[i + 1]
            arena = torch.empty(P.V, fi, device=self.dev)
            ops.spmm_csr(G, x, "mean", out=arena)
            y = torch.empty(P.N, fo, device=self.dev)
            for t in range(self.T):
                n = P.cnt[t]
                if n == 0:
                    continue
                acat = arena[P.vbase[t]:P.vbase[t + 1]].view(n, -1)
                hi, lo = ops.split_tf32(self._wcatT(i, t), transpose=True)
                ops.gemm_tf32x3(acat, hi, lo, bias=self._bias(i, t), out=y[P.off[t]:P.off[t + 1]])
            arenas.append(arena)
            if i < self.L - 1:
                x = ops.affine_relu_dropout_mapped(y, None, None, True, self.p if training else 0.0, self.seed, i,
                                                   step_dev=self.step_count if training else None, step_mul=self.L,
                                                   rowmap=rowmap, k_global=fo)
                xs.append(x)
            ys.append(y)
        self._fwd = dict(P=P, Gt=Gt, li_int=li_int, xs=xs, arenas=arenas, ys=ys)
        return ys[-1][P.pos, :self.C]

    def out_feat(self) -> torch.Tensor:
        """The reference's ``model.out_feat``: the last hidden layer's output after ReLU and dropout, batch node order."""
        f = self._fwd
        return f["xs"][-1][f["P"].pos]

    def backward(self, d_logits_int: torch.Tensor, d_out_feat: Optional[torch.Tensor] = None,
                 d_out_feat_int: Optional[torch.Tensor] = None) -> torch.Tensor:
        """d loss / d logits [N, C'] in INTERNAL row order -> self.grads (flat) and the returned layer-0 input gradient [N, F_in]
        (internal order).  d_out_feat (batch order) or d_out_feat_int (internal order) is added to the gradient arriving at
        the last hidden activation."""
        f = self._fwd
        P = f["P"]
        self.grads.zero_()
        dy = d_logits_int
        dx = None
        need_dx0 = bool(self.emb)
        for i in range(self.L - 1, -1, -1):
            fi = self.dims_pad[i]
            darena = torch.empty(P.V, fi, device=self.dev) if (i > 0 or need_dx0) else None
            for t in range(self.T):
                n = P.cnt[t]
                if n == 0:
                    continue
                rows = slice(P.off[t], P.off[t + 1])
                d_t = dy[rows]
                ops.col_sum(d_t, out=self._bias(i, t, self.grads))
                acat = f["arenas"][i][P.vbase[t]:P.vbase[t + 1]].view(n, -1)
                ops.gemm_wgrad_tf32x3(acat, d_t, out=self._wcatT(i, t, self.grads), workspace=self.wgrad_ws, wide=True)
                if darena is not None:
                    hi, lo = ops.split_tf32(self._wcatT(i, t), transpose=False)
                    ops.gemm_tf32x3(d_t, hi, lo, out=darena[P.vbase[t]:P.vbase[t + 1]].view(n, -1))
            if darena is None:
                break
            dx = ops.spmm_csr(f["Gt"], darena, "sum")
            if i > 0:
                if i == self.L - 1 and d_out_feat is not None:
                    dx.add_(d_out_feat[P.perm])
                if i == self.L - 1 and d_out_feat_int is not None:
                    dx.add_(d_out_feat_int)
                dy = ops.relu_dropout_bwd(dx, f["xs"][i], self.p if self._training else 0.0, out=dx)
        return dx

    def _loss(self, P, batch, teacher_logits, teacher_int: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Fused CE / KD over the train_mask rows on the padded logits (ld = C'); returns d logits (internal order).
        teacher_int: the teacher's padded logits in internal row order, read in place (a teacher run on this plan)."""
        y_int = batch.y.view(-1).long()[P.perm].contiguous()
        train_b = batch.train_mask.view(-1).nonzero().view(-1)
        train_int = P.pos[train_b].contiguous()
        self._fwd["train_int"] = train_int
        logits = self._fwd["ys"][-1]
        d = torch.zeros_like(logits)
        teacher = teacher_int
        if teacher_logits is not None:
            teacher = torch.zeros(P.N, self.C, device=self.dev)
            teacher[train_int] = teacher_logits.to(torch.float32)
        n_train = train_int.numel()
        L = lib.load()
        part = torch.empty(2 * int(L.b200gnn_kd_partials(max(n_train, 1))), device=self.dev)
        lib.check(L.b200gnn_kd_loss_fwd_bwd_f32(
            logits.data_ptr(), logits.stride(0), train_int.data_ptr(), n_train, y_int.data_ptr(),
            None if teacher is None else teacher.data_ptr(), 0 if teacher is None else teacher.stride(0), self.C, self.alpha,
            self.kd_T, 0, d.data_ptr(), d.stride(0), self.loss_out.data_ptr(), part.data_ptr(), lib.stream_ptr()),
            "kd_loss_fwd_bwd_f32")
        return d

    def check_teacher(self, teacher: "RGCNTrainer") -> None:
        """ValueError unless ``teacher`` can run on this trainer's batch plans and feed its loss: the same node types and
        table sizes, feature types, relations (source, destination), input width, classes and device."""
        if not isinstance(teacher, RGCNTrainer):
            raise ValueError("teacher= must be an RGCNTrainer")
        for what, mine, theirs in (("node types and counts", self.num_nodes, teacher.num_nodes),
                                   ("node types with features", self.x_types, teacher.x_types),
                                   ("relations (source type, destination type)", self.relations, teacher.relations),
                                   ("input width", self.F_in, teacher.F_in), ("classes", self.C, teacher.C),
                                   ("device", self.dev, teacher.dev)):
            if mine != theirs:
                raise ValueError(f"teacher= has other {what} than the student ({theirs} vs {mine}): it cannot run on the "
                                 "student's batch plan")

    def train_step(self, batch, x_dict: Dict[int, torch.Tensor], teacher_logits: Optional[torch.Tensor] = None, aux=None,
                   beta: float = 1.0, teacher: Optional["RGCNTrainer"] = None,
                   sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One iteration of the reference ``train()`` loop body: logit-KD if ``teacher_logits`` ([n_train, C], the teacher's
        logits on the train_mask rows in batch order) or ``teacher`` is given, else cross-entropy, over the train_mask rows;
        then Adam over every parameter and embedding row.  ``aux(out_feat)`` as in ``GCNStudentTrainer.train_step``.

        ``teacher``: another RGCNTrainer (the reference's ``teacher_model``), run in eval mode on this step's batch plan (one
        plan per batch, no second sort); the KD loss reads its padded logits in place, and nothing of the teacher changes.
        The trainer's ``lsp=``, ``gcrd=`` and ``gsp=`` objectives need it: the teacher's last hidden layer (ReLU, no dropout)
        is their feature side.  ``sample`` (positions into the batch's train rows, in batch order, [S]) replaces the gcrd= or
        gsp= object's on-device row sample (tests).  Returns the device tensor [loss, loss_cls, loss_kd] ([kd + beta * lsp,
        loss_cls, lsp] with lsp=, [kd + beta * nce, loss_cls, nce] with gcrd=, [kd + beta * gsp, loss_cls, gsp] with gsp=)."""
        objective = one_objective(gcrd=self.gcrd, lsp=self.lsp, gsp=self.gsp)
        name = "lsp=" if self.lsp is not None else "gcrd=" if self.gcrd is not None else "gsp="
        if teacher is not None and teacher_logits is not None:
            raise ValueError("teacher= and teacher_logits= are two teachers; pass one")
        if objective is not None and aux is not None:
            raise ValueError(f"aux= and the trainer's {name} objective are two auxiliary losses; pass one")
        if objective is not None and teacher is None:
            raise ValueError(f"the {name} objective compares with the teacher's features: pass teacher=")
        if sample is not None and self.gcrd is None and self.gsp is None:
            raise ValueError("sample= is the G-CRD / GSP row sample; this trainer has no gcrd= objective and no gsp= "
                             "objective")
        if teacher is not None:
            self.check_teacher(teacher)
        if self.gcrd is not None:
            self.gcrd.check_teacher(teacher)
            # the one host read of the train rows' count (the step reads the host anyway): refusals before any launch
            self.gcrd.check_batch(int(batch.train_mask.sum()), sample)
        if self.gsp is not None:
            self.gsp.check_teacher(teacher)
            self.gsp.check_batch(int(batch.train_mask.sum()), sample)
        self.forward(batch, x_dict, training=True)
        P = self._fwd["P"]
        teacher_int = None
        if teacher is not None:
            teacher.forward(batch, x_dict, training=False, plan=P)
            teacher_int = teacher._fwd["ys"][-1]
        d_logits = self._loss(P, batch, teacher_logits, teacher_int)
        d_feat = d_feat_int = None
        if aux is not None:
            d_feat, self.loss_aux = aux_grad(self.out_feat(), aux, beta)
        elif self.lsp is not None:
            d_feat_int = self.lsp.forward_backward(self, teacher, batch)
        elif self.gcrd is not None:
            d_feat_int = self.gcrd.forward_backward(self, teacher, sample)
        elif self.gsp is not None:
            d_feat_int = self.gsp.forward_backward(self, teacher, sample)
        dx0 = self.backward(d_logits, d_feat, d_feat_int)
        if self.emb:
            li = self._fwd["li_int"]
            order = device_argsort(P.node_type_int, li, self.T, max(self.num_nodes.values()))
            for t, e in self.emb.items():
                ops.embedding_adam(dx0, P.node_type_int, li, order, t, e, self.emb_m[t], self.emb_v[t], self._head,
                                   self.step_count, self.lr)
        ops.adam_step(self.params, self.grads, self.exp_avg, self.exp_avg_sq, self.step_count, self.lr)
        if self.gcrd is not None:
            self.gcrd.optimizer_step(self.lr)
        if aux is not None:
            self.loss_out[0].add_(self.loss_aux * beta)
        elif objective is not None:
            self.loss_out[2].copy_(objective.loss_aux[0])
        return self.loss_out

    def gradients(self, batch, x_dict, d_logits: torch.Tensor) -> Dict[str, torch.Tensor]:
        """Gradients of sum(logits * d_logits) under the state_dict names (embedding gradients as dense tables) after an
        evaluation-mode forward; no parameter changes (checks against autograd)."""
        self.forward(batch, x_dict, training=False)
        P = self._fwd["P"]
        d = torch.zeros(P.N, self.dims_pad[-1], device=self.dev)
        d[:, :self.C] = d_logits.to(self.dev, torch.float32)[P.perm]
        dx0 = self.backward(d)
        emb = {t: torch.zeros_like(e) for t, e in self.emb.items()}
        if emb:
            li = self._fwd["li_int"]
            order = device_argsort(P.node_type_int, li, self.T, max(self.num_nodes.values()))
            ops.typed_scatter(dx0, P.node_type_int, li, order, emb, self.T)
        return self._named(self.grads, emb)
