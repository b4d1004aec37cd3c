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
"""
from __future__ import annotations

from typing import Optional

import torch

from . import criterion, lib, ops


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
        if edge_index.dim() != 2 or edge_index.shape[0] != 2:
            raise ValueError("edge_index must be [2, E]")
        ei = edge_index.to(dev, torch.int64)
        self.E = E = ei.shape[1]
        if E == 0:
            raise ValueError("edge_index has no edges: the train-induced subgraph is empty")
        if int(ei.min()) < 0 or int(ei.max()) >= n:
            raise ValueError(f"edge_index refers to a row outside the {n} training rows")
        self.plan = criterion.LspPlan(ei)
        self.C, self.pos_dst, self.pos_src, self.diag_pos, self.selfc = self.plan.backward_matrix(n)

        # the teacher side is a constant of the run: its similarities once, from rows gathered for this call only
        G_t = teacher_feat.detach().to(torch.float32)[self.train_idx].contiguous()
        self.sim_t = torch.empty(E, dtype=torch.float32, device=dev)
        lib.check(lib.load().b200gnn_edge_sim_f32(lib.dptr(G_t, torch.float32, "teacher"), G_t.shape[1], self.plan.src.data_ptr(),
                                                  self.plan.dst.data_ptr(), E, self.kernel_id, self.sim_t.data_ptr(),
                                                  lib.stream_ptr()), "edge_sim_f32")
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
