"""LSP inside the students' captured training step: the teacher's edge similarities once, the student side in one kernel.

The reference's ``train()`` with ``--training lpw`` (arxiv_pyg/gnn.py:139-145: CE + beta * lpw; gnn_kd_and_aux.py:149-155:
KD + beta * lpw) compares, over the train-induced edge list (gnn_kd_and_aux.py:240-243), the PyG softmax per destination of
the student's and the teacher's edge similarities (criterion.py:95-126, criterion kld):

    edge_index  = subgraph(train_idx, stack(adj_t.coo()[:2]), relabel_nodes=True)[0]
    sim_s[e]    = k(out_feat[train_idx][src], out_feat[train_idx][dst])       k: cosine, poly, l2 or rbf
    sim_t[e]    = k(teacher_out_feat[train_idx][src], ... [dst])              a constant of the run
    loss_aux    = kl_div(log softmax(sim_s, dst), softmax(sim_t, dst))

``LSP`` holds the dst-sorted plan (criterion.LspPlan), its backward matrix, ``sim_t`` (formed once with the edge_sim kernel
from the gathered teacher rows, which are then dropped) and every buffer of the step.  ``GCNStudentTrainer(..., lsp=o)`` /
``SAGEStudentTrainer(..., lsp=o)`` call it from inside their step, so ``capture()`` / ``replay()`` run it in the same CUDA
graph:

    gather       out_feat[train_idx] -> G_s [n_train, H] (GCN: formed from Y, BN scale/shift and the keep bits)
    student      b200gnn_lsp_student_f32: sim_s, the KL loss and the backward matrix's values in one kernel (+ its diagonal
                 and the loss reduction), bit-identical to edge_sim -> lsp_segment -> lsp_bwd_values
    backward     d = C . G_s (the row-segmented SpMM), then d out_feat[train_idx] = d * beta, zero elsewhere, and
                 loss[0] += beta * loss_aux (b200gnn_scatter_rows_scaled_f32)

Every float equals the eager ``train_step(aux=lambda f: lpw_criterion(..., f[idx], t[idx], edge_index, kernel, 1)[2],
beta=beta)``: the same kernels' arithmetic, the same SpMM, and beta applied as its autograd applies it.

``PerGraphLSP`` is the same loss for engine_ppi's PPI student: one raw edge list per training graph, every node a row, the
constants of each graph built once by the helpers ``LSP`` uses and the step's buffers shared by all graphs.

``BatchLSP`` is the same loss for rgcn's MAG student on GraphSAINT batches, where nothing is a constant of the run: each
batch has its own train-induced edge list (built on the device, sampling.induced_edges) and the teacher runs inside the
student's step, so the plan, the backward matrix and sim_t are built per batch by the same helpers.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from . import criterion, lib, ops, sampling

_KERNELS = criterion._KERNELS             # PerGraphLSP's criterion= argument shadows the module


def _checked_edges(edge_index: torch.Tensor, n: int, rows: str) -> torch.Tensor:
    """edge_index as a [2, E] int64 tensor on its own device; ValueError if it has no edge or an index outside [0, n)."""
    if edge_index.dim() != 2 or edge_index.shape[0] != 2:
        raise ValueError("edge_index must be [2, E]")
    if edge_index.shape[1] == 0:
        raise ValueError("edge_index has no edges: the LSP loss would average over none")
    ei = edge_index.to(torch.int64)
    if int(ei.min()) < 0 or int(ei.max()) >= n:
        raise ValueError(f"edge_index refers to a row outside the {n} {rows}")
    return ei


def _edge_constants(G_t: torch.Tensor, ei: torch.Tensor, n: int, kernel_id: int):
    """What one edge list fixes for the whole run: the dst-sorted plan (criterion.LspPlan), its backward matrix for n feature
    rows (C, pos_dst, pos_src, diag_pos, selfc) and the teacher's edge similarities sim_t [E] from its rows G_t [n, F_t]."""
    plan = criterion.LspPlan(ei)
    bwd = plan.backward_matrix(n)
    sim_t = torch.empty(plan.E, dtype=torch.float32, device=ei.device)
    lib.check(lib.load().b200gnn_edge_sim_f32(lib.dptr(G_t, torch.float32, "teacher"), G_t.shape[1], plan.src.data_ptr(),
                                              plan.dst.data_ptr(), plan.E, kernel_id, sim_t.data_ptr(), lib.stream_ptr()),
              "edge_sim_f32")
    return plan, bwd, sim_t


class LSP:
    def __init__(self, teacher_feat: torch.Tensor, train_idx: torch.Tensor, edge_index: torch.Tensor, hidden: int,
                 kernel: str = "rbf", beta: float = 0.5):
        """teacher_feat: the teacher's [N, F_t] features (the GAT teacher's ``features/`` file); train_idx: the training rows,
        the same tensor the trainer's step receives; edge_index [2, E]: the train-induced edge list, relabelled to positions
        in train_idx (the reference's ``subgraph(train_idx, ..., relabel_nodes=True)[0]``); hidden: the student's last
        hidden width, at most lib.LSP_MAX_F.  kernel: 'cosine', 'poly', 'l2' or 'rbf' (the reference's default);
        beta: the weight of the loss (the scripts use cosine with beta 100)."""
        if kernel not in criterion._KERNELS:
            raise ValueError(f"kernel {kernel!r}: LSP kernels are {sorted(criterion._KERNELS)}")
        if not 0 < int(hidden) <= lib.LSP_MAX_F:
            raise ValueError(f"hidden width {hidden}: the LSP kernel holds a student row in registers, at most {lib.LSP_MAX_F}")
        dev = teacher_feat.device
        self.device = dev
        self.train_idx = train_idx.to(dev, torch.int64).contiguous()
        self.n = n = self.train_idx.numel()
        self.H, self.kernel, self.kernel_id, self.beta = int(hidden), kernel, criterion._KERNELS[kernel], float(beta)
        ei = _checked_edges(edge_index, n, "training rows").to(dev)
        self.E = E = ei.shape[1]
        # the teacher side is a constant of the run: its similarities once, from rows gathered for this call only
        G_t = teacher_feat.detach().to(torch.float32)[self.train_idx].contiguous()
        self.plan, (self.C, self.pos_dst, self.pos_src, self.diag_pos, self.selfc), self.sim_t = \
            _edge_constants(G_t, ei, n, self.kernel_id)
        del G_t

        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        self.G_s = e(n, self.H)                                # out_feat[train_idx]
        self.sim_s, self.scratch = e(E), e(2 * E)
        self.partial = e(int(lib.load().b200gnn_lsp_partials(self.plan.n_seg)))
        self.loss_aux = torch.zeros(1, dtype=torch.float32, device=dev)
        self.d = e(n, self.H)                                  # C . G_s
        self.d_feat: Optional[torch.Tensor] = None

    def bind(self, trainer):
        """Called by the trainer that owns this object: the [N, H] gradient of out_feat the step writes."""
        if trainer.dims[-2] != self.H:
            raise ValueError(f"LSP built for hidden width {self.H}, the student's last hidden layer is {trainer.dims[-2]}")
        self.d_feat = torch.zeros(trainer.N, self.H, device=self.device)
        self.trainer = trainer

    def forward_backward(self, tr, sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Everything between the trainer's loss and its backward: returns d (beta * loss_aux) / d out_feat [N, H] and adds
        beta * loss_aux to tr.loss_out[0].  Enqueues launches only (capturable)."""
        if sample is not None:
            raise ValueError("sample= is the G-CRD row sample; LSP draws no sample")
        if getattr(tr, "_fwd_fused", False):
            l = tr.L - 2
            ops.gather_rows_act(tr.Y[l], self.train_idx, self.G_s, bits=tr.keep_bits[l], scale=tr.bn[l][2],
                                shift=tr.bn[l][3], p=tr.p)
        else:
            ops.gather_rows_act(tr.out_feat(), self.train_idx, self.G_s)
        p = self.plan
        ops.lsp_student(self.G_s, p.src, p.dst, p.rowptr, self.sim_t, self.kernel_id, self.pos_dst, self.pos_src, self.C.rowptr,
                        self.diag_pos, self.sim_s, self.scratch, self.C.val, self.selfc, self.loss_aux, self.partial)
        ops.spmm_csr(self.C, self.G_s, "sum", out=self.d)
        # the GCN backward reuses this buffer as its dz, so it is cleared every step
        self.d_feat.zero_()
        ops.scatter_rows_scaled(self.d, self.train_idx, self.beta, self.d_feat, loss_aux=self.loss_aux, loss_total=tr.loss_out)
        return self.d_feat

    def optimizer_step(self, lr: float):
        """LSP has no parameters of its own."""


class _GraphConstants:
    """One training graph's share of PerGraphLSP: n rows, E edges, the plan, the backward matrix and sim_t."""

    def __init__(self, n: int, G_t: torch.Tensor, ei: torch.Tensor, kernel_id: int):
        self.n = n
        self.plan, (self.C, self.pos_dst, self.pos_src, self.diag_pos, self.selfc), self.sim_t = \
            _edge_constants(G_t, ei, n, kernel_id)
        self.E = self.plan.E


class PerGraphLSP:
    """LSP inside engine_ppi's captured step: the reference's PPI ``train()`` with ``--training lpw`` (ppi_pyg/gnn.py:240-249)
    computes ``lpw_criterion(out, labels, model.out_feat, teacher_model.out_feat, batch.edge_index, kernel, beta)`` on each
    training graph, over the graph's raw edge list and every one of its nodes.

    Per graph the plan, the backward matrix and sim_t are built once (as LSP builds them for its one edge list); the
    per-step buffers are sized for the largest graph and sliced per graph, so that one CUDA graph per training graph
    (``PPIGATTrainer.capture``) records the student side with that graph's constants:

        student      b200gnn_lsp_student_f32 on out_feat [n, H] (no gather: every node is a row)
        backward     d = C . out_feat, then d out_feat = d * beta into the trainer's seed buffer and
                     loss[0] += beta * loss_aux (b200gnn_scatter_rows_scaled_f32)

    Every float equals the eager ``train_step(i, aux=lambda f: criterion_ppi.lpw_criterion(..., f, teacher_feat[i],
    edge_index[i], kernel, 1)[2], beta=beta)``."""

    def __init__(self, teacher_feat: Sequence[torch.Tensor], edge_index: Sequence[torch.Tensor], hidden: int,
                 kernel: str = "rbf", beta: float = 100.0, criterion: str = "kld", device="cuda"):
        """teacher_feat: per training graph the teacher's [n_i, F_t] ``out_feat`` (``predict(..., return_feat=True)``; F_t =
        1024 for TeacherNet); edge_index: per training graph its [2, E_i] edge list exactly as ``batch.edge_index`` holds it
        (self-loops and duplicate edges are terms of the loss like any other edge); hidden: the student's out_feat width, at
        most lib.LSP_MAX_F (136 for StudentNet).  kernel: 'cosine', 'poly', 'l2' or 'rbf' (the argparse default of
        ppi_pyg/gnn.py); beta: the weight of the loss (scripts/run.sh: 100).  Only the kld criterion (the reference's
        default) is built.  The teacher features are dropped once sim_t is formed."""
        if len(teacher_feat) != len(edge_index):
            raise ValueError(f"{len(teacher_feat)} teacher feature matrices for {len(edge_index)} edge lists")
        if len(edge_index) == 0:
            raise ValueError("no training graphs")
        if kernel not in _KERNELS:
            raise ValueError(f"kernel {kernel!r}: LSP kernels are {sorted(_KERNELS)}")
        if criterion != "kld":
            raise ValueError(f"criterion {criterion!r}: the fused LSP step is the kld form (the reference's default)")
        if not 0 < int(hidden) <= lib.LSP_MAX_F:
            raise ValueError(f"hidden width {hidden}: the LSP kernel holds a student row in registers, at most {lib.LSP_MAX_F}")
        # every graph is checked before any work on the device
        edges = []
        for k, (t, ei) in enumerate(zip(teacher_feat, edge_index)):
            if t.dim() != 2:
                raise ValueError(f"graph {k}: teacher features must be [n, F_t]")
            edges.append(_checked_edges(ei, int(t.shape[0]), f"nodes of training graph {k}"))
        self.device = dev = torch.device(device)
        self.H, self.kernel, self.kernel_id, self.beta = int(hidden), kernel, _KERNELS[kernel], float(beta)
        self.graphs = [_GraphConstants(int(t.shape[0]), t.detach().to(dev, torch.float32).contiguous(), ei.to(dev), self.kernel_id)
                       for t, ei in zip(teacher_feat, edges)]
        n_max, E_max = max(g.n for g in self.graphs), max(g.E for g in self.graphs)
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)    # noqa: E731
        self.sim_s, self.scratch = e(E_max), e(2 * E_max)
        self.partial = e(max(int(lib.load().b200gnn_lsp_partials(g.plan.n_seg)) for g in self.graphs))
        self.loss_aux = torch.zeros(1, dtype=torch.float32, device=dev)
        self.d = e(n_max, self.H)                                                  # C . out_feat
        self.rows = torch.arange(n_max, dtype=torch.int64, device=dev)              # the identity scatter of d * beta

    def bind(self, trainer):
        """Called by the PPIGATTrainer that owns this object: its graphs and out_feat width must be the ones built for."""
        if len(trainer.graphs) != len(self.graphs):
            raise ValueError(f"LSP built for {len(self.graphs)} training graphs, the trainer has {len(trainer.graphs)}")
        if trainer.Kout[-2] != self.H:
            raise ValueError(f"LSP built for hidden width {self.H}, the student's out_feat is {trainer.Kout[-2]} wide")
        for k, (mine, theirs) in enumerate(zip(self.graphs, trainer.graphs)):
            if mine.n != theirs.n:
                raise ValueError(f"graph {k}: LSP built for {mine.n} nodes, the trainer's graph has {theirs.n}")

    def forward_backward(self, i: int, feat: torch.Tensor, d_feat: torch.Tensor, loss_out: torch.Tensor):
        """Graph i's loss and gradient: reads out_feat ``feat`` [n_i, H], writes d (beta * loss_aux) / d out_feat into d_feat
        [n_i, H] and adds beta * loss_aux to loss_out[0]; the value of loss_aux stays in self.loss_aux.  Enqueues launches
        only (capturable)."""
        g = self.graphs[i]
        p, n, E = g.plan, g.n, g.E
        ops.lsp_student(feat, p.src, p.dst, p.rowptr, g.sim_t, self.kernel_id, g.pos_dst, g.pos_src, g.C.rowptr, g.diag_pos,
                        self.sim_s[:E], self.scratch[:2 * E], g.C.val, g.selfc, self.loss_aux, self.partial)
        d = ops.spmm_csr(g.C, feat, "sum", out=self.d[:n])
        ops.scatter_rows_scaled(d, self.rows[:n], self.beta, d_feat, loss_aux=self.loss_aux, loss_total=loss_out)


class BatchLSP:
    """LSP inside rgcn.RGCNTrainer's step: the reference's MAG ``train()`` with ``--training lpw``
    (mag_pyg/gnn_kd_and_aux.py:232-245) on every GraphSAINT batch b:

        edge_index = subgraph(b.train_mask.nonzero().squeeze(1), b.edge_index, relabel_nodes=True)[0]
        loss_aux   = lpw_criterion(out, labels, model.out_feat[b.train_mask], teacher_model.out_feat[b.train_mask],
                                   edge_index, kernel, beta)[2]                    kld
        loss       = kd_criterion(out, labels, teacher_out, alpha, kd_T)[0] + beta * loss_aux

    Per batch, between the student's loss and its backward (``RGCNTrainer(..., lsp=o).train_step(b, x, teacher=t)``):

        edges      sampling.induced_edges (one host read sizes it), then the dst-sorted plan, the backward matrix for
                   n_train rows and the teacher's sim_t (_edge_constants, as LSP builds them once)
        gather     G_s = the student's last hidden layer (after ReLU and dropout) and G_t = the teacher's (eval: ReLU) at
                   the train rows, in the order of train_mask.nonzero()
        student    b200gnn_lsp_student_f32, then d = C . G_s (the row-segmented SpMM)
        backward   beta * d scattered straight into the internal-order gradient the trainer adds at its last hidden layer,
                   loss[0] += beta * loss_aux (b200gnn_scatter_rows_scaled_f32); loss[2] = loss_aux

    The train rows are relabelled by their rank in train_mask.nonzero() (batch order) and gathered at their internal rows
    BatchPlan.pos[train_mask.nonzero()], so row k of G_s is the k-th train row whatever the internal order.  (All train
    rows are papers and BatchPlan sorts types stably, so those internal rows also ascend.)

    Every float equals the eager ``train_step(b, x, teacher_logits=..., aux=lambda f: criterion.lpw_criterion(...,
    f[train_mask], t_feat[train_mask], edge_index, kernel, 1)[2], beta=beta)``.  A batch whose train rows induce no edge
    does what the reference does: kl_div's mean over no term is NaN, so loss[0] and loss[2] are NaN, and the step's
    gradients carry no LSP term."""

    def __init__(self, hidden: int, kernel: str = "rbf", beta: float = 1.0, criterion: str = "kld", device="cuda"):
        """hidden: the student's last hidden width (32 in the reference's MAG student), at most lib.LSP_MAX_F.  kernel:
        'cosine', 'poly', 'l2' or 'rbf' (scripts/run_kd_and_aux.sh runs rbf, cosine and poly); beta: the weight of the loss.
        Only the kld criterion (the reference's default) is built."""
        if kernel not in _KERNELS:
            raise ValueError(f"kernel {kernel!r}: LSP kernels are {sorted(_KERNELS)}")
        if criterion != "kld":
            raise ValueError(f"criterion {criterion!r}: the fused LSP step is the kld form (the reference's default)")
        if not 0 < int(hidden) <= lib.LSP_MAX_F:
            raise ValueError(f"hidden width {hidden}: the LSP kernel holds a student row in registers, at most {lib.LSP_MAX_F}")
        self.device = torch.device(device)
        self.H, self.kernel, self.kernel_id, self.beta = int(hidden), kernel, _KERNELS[kernel], float(beta)
        self.loss_aux = torch.zeros(1, dtype=torch.float32, device=self.device)
        self.edge_index: Optional[torch.Tensor] = None          # the last batch's train-induced edge list

    def bind(self, trainer):
        """Called by the RGCNTrainer that owns this object: its last hidden layer must be the width built for."""
        if trainer.L < 2 or trainer.dims[-2] != self.H:
            raise ValueError(f"LSP built for hidden width {self.H}, the student's last hidden layer is "
                             f"{trainer.dims[-2] if trainer.L >= 2 else 'absent'}")

    def forward_backward(self, tr, teacher, batch) -> Optional[torch.Tensor]:
        """After tr's loss on its forward and teacher's eval forward on the same plan: returns d (beta * loss_aux) / d out_feat
        [N, H] in internal row order (None when the batch induces no edge) and adds beta * loss_aux to tr.loss_out[0]."""
        f, ft = tr._fwd, teacher._fwd
        P, train_int = f["P"], f["train_int"]
        n = train_int.numel()
        ei = sampling.induced_edges(batch.edge_index, batch.train_mask.view(-1))
        self.edge_index = ei
        if ei.shape[1] == 0:
            self.loss_aux.fill_(float("nan"))
            tr.loss_out[:1].add_(self.loss_aux * self.beta)
            return None
        feat_t = ft["xs"][-1]
        G_t = ops.gather_rows_act(feat_t, train_int, torch.empty(n, feat_t.shape[1], device=self.device))
        plan, (C, pos_dst, pos_src, diag_pos, selfc), sim_t = _edge_constants(G_t, ei, n, self.kernel_id)
        del G_t
        G_s = ops.gather_rows_act(f["xs"][-1], train_int, torch.empty(n, self.H, device=self.device))
        E = plan.E
        e = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=self.device)    # noqa: E731
        ops.lsp_student(G_s, plan.src, plan.dst, plan.rowptr, sim_t, self.kernel_id, pos_dst, pos_src, C.rowptr, diag_pos,
                        e(E), e(2 * E), C.val, selfc, self.loss_aux, e(int(lib.load().b200gnn_lsp_partials(plan.n_seg))))
        d = ops.spmm_csr(C, G_s, "sum")
        d_feat = torch.zeros(P.N, self.H, device=self.device)
        ops.scatter_rows_scaled(d, train_int, self.beta, d_feat, loss_aux=self.loss_aux, loss_total=tr.loss_out)
        return d_feat
