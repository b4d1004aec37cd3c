"""Host-side plumbing the fused trainers share: the flat parameter store, the autograd bridge of ``train_step(aux=)``,
CUDA-graph capture, and the (x, y, train_idx, teacher_logits) step of the full-batch students (GCN, SAGE, GAT)."""
from __future__ import annotations

import contextlib
import math
from typing import Callable, Optional, Sequence, Tuple

import torch

from . import lib, ops


class FlatParams:
    """Parameters, gradients and Adam state of one model as flat fp32 buffers, laid out in declaration order.

    The gradients are the front of one buffer padded to 16 bytes and followed by a 4-float tail whose first three floats
    are the step's losses (``loss_out``): the multi-GPU engines exchange and reduce both with a single launch."""

    def __init__(self, shapes: Sequence[Tuple[int, ...]], device):
        sizes = [math.prod(s) for s in shapes]
        n = sum(sizes)
        self.n_par_pad = (n + 3) // 4 * 4
        self.params = torch.zeros(n, device=device)
        self._grads_buf = torch.zeros(self.n_par_pad + 4, device=device)
        self.grads = self._grads_buf[:n]
        self.loss_out = self._grads_buf[self.n_par_pad:self.n_par_pad + 3]
        self.exp_avg = torch.zeros(n, device=device)
        self.exp_avg_sq = torch.zeros(n, device=device)
        self.step_count = torch.zeros(1, dtype=torch.int32, device=device)
        self.views = []                  # (param, grad) per shape
        off = 0
        for k, s in zip(sizes, shapes):
            self.views.append((self.params[off:off + k].view(s), self.grads[off:off + k].view(s)))
            off += k

    def attach(self, owner) -> "FlatParams":
        """Publishes the buffers as owner.params, .grads, ...: the names bench.py, the multi-GPU engines and the tests read."""
        for k in ("params", "grads", "_grads_buf", "n_par_pad", "loss_out", "exp_avg", "exp_avg_sq", "step_count"):
            setattr(owner, k, getattr(self, k))
        return self

    @staticmethod
    def offset(view: torch.Tensor) -> int:
        """Element offset of a view of params (or of grads) in its flat buffer."""
        return view.storage_offset()

    def like(self, buf: torch.Tensor, view: torch.Tensor) -> torch.Tensor:
        """The view of ``buf``, a flat buffer laid out like params, at the place of parameter view ``view``."""
        o = self.offset(view)
        return buf[o:o + view.numel()].view(view.shape)

    def adam(self, lr: float):
        ops.adam_step(self.params, self.grads, self.exp_avg, self.exp_avg_sq, self.step_count, lr)

    @contextlib.contextmanager
    def preserved(self):
        """Parameters, Adam state and the step counter are put back on exit as they were on entry."""
        state = (self.params, self.exp_avg, self.exp_avg_sq, self.step_count)
        saved = [t.clone() for t in state]
        yield
        for t, v in zip(state, saved):
            t.copy_(v)


def aux_grad(out_feat: torch.Tensor, aux: Callable, beta: float):
    """The autograd bridge of ``train_step(aux=)``: (d (beta * aux(out_feat)) / d out_feat, aux(out_feat) detached).  The
    gradient is zeros when aux does not depend on its input; parameters inside aux keep their gradients in autograd."""
    feat = out_feat.detach().requires_grad_(True)
    with torch.enable_grad():
        loss_aux = aux(feat)
        (loss_aux * beta).backward()
    d_feat = feat.grad if feat.grad is not None else torch.zeros_like(feat)
    return d_feat.contiguous(), loss_aux.detach()


def capture_graph(step: Callable[[], None], warmup: int) -> torch.cuda.CUDAGraph:
    """Runs ``step()`` ``warmup`` times on a side stream, joins, synchronises and returns ``step`` captured as a CUDA graph
    (the capture itself runs nothing)."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(warmup):
            step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    return g


def one_objective(gcrd=None, lsp=None, gsp=None):
    """The auxiliary loss a student runs inside its step: at most one of G-CRD, LSP and GSP."""
    if gcrd is not None and lsp is not None:
        raise ValueError("gcrd= and lsp= are two auxiliary losses; pass one")
    if gsp is not None and (gcrd is not None or lsp is not None):
        raise ValueError("gsp= and the gcrd= / lsp= objective are two auxiliary losses; pass one")
    return next((o for o in (gcrd, lsp, gsp) if o is not None), None)


class FullBatchStudent:
    """The step GCNStudentTrainer, SAGEStudentTrainer and GATTrainer share.  A subclass provides ``forward(x, training)``,
    ``out_feat()``, ``backward(x, d_out_feat)``, the FlatParams ``store`` and ``_static`` (a dict), and extends ``replay``
    with the host state a replayed step leaves stale."""

    objective = None                 # G-CRD / LSP / GSP run inside the step (one_objective)
    _graph = None                    # key -> captured step

    def dropout_offset(self, layer: int, step: int) -> int:
        return layer + step * self.L

    def _part(self, k: int) -> torch.Tensor:
        key = f"part{k}"
        if key not in self._static:
            self._static[key] = torch.empty(self.rs, 2, k, device=self.device)
        return self._static[key]

    def _coef(self, k: int) -> torch.Tensor:
        key = f"coef{k}"
        if key not in self._static:
            self._static[key] = torch.empty(3, k, device=self.device)
        return self._static[key]

    def _loss(self, x, y, train_idx, teacher_logits):
        """Training forward, then the fused CE / logit-KD loss with d loss / d logits into dY[-1]."""
        logits = self.forward(x, training=True)
        self.dY[-1].zero_()
        ops.kd_loss_fwd_bwd(logits, y, train_idx, teacher_logits, self.alpha, self.kd_T, d_logits=self.dY[-1],
                            loss_out=self.loss_out, partial=self.kd_part)

    def _step_impl(self, x, y, train_idx, teacher_logits, sample=None, aux=None, beta: float = 1.0):
        """Forward and loss, d loss / d out_feat from aux (through autograd) or the objective, backward, Adam, the objective's
        Adam.  Enqueues launches only when aux is None (capturable)."""
        self._loss(x, y, train_idx, teacher_logits)
        d_feat = None
        if aux is not None:
            d_feat, self.loss_aux = aux_grad(self.out_feat(), aux, beta)
        elif self.objective is not None:
            d_feat = self.objective.forward_backward(self, sample)
        self.backward(x, d_out_feat=d_feat)
        self.store.adam(self.lr)
        if self.objective is not None:
            self.objective.optimizer_step(self.lr)
        if aux is not None:
            self.loss_out[0].add_(self.loss_aux * beta)

    def train_step(self, x, y, train_idx, teacher_logits=None, aux=None, beta: float = 1.0,
                   sample: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One reference ``train()`` call: kd if teacher_logits is given, else supervised (arxiv_pyg/gnn.py:102-195), and
        with ``aux`` the kd + beta*aux form of gnn_kd_and_aux.py:100-189 — ``aux(out_feat)`` receives the [N, H] output
        of the last hidden layer (the reference's ``model.out_feat``, requires_grad) and returns the auxiliary loss, e.g.
        ``lambda f: criterion.lpw_criterion(z, y, f[idx], t_feat[idx], edge_index, "cosine", 1)[2]`` or a projection head +
        ``nce_criterion``; parameters of such heads get their gradients through torch autograd and stay with the caller's
        optimizer.  Returns the device tensor [loss, loss_cls, loss_kd] (+ beta*aux folded into loss); no host sync.
        With a G-CRD, LSP or GSP object (constructor) the step includes it (loss[0] += beta * loss_aux, value in its loss_aux);
        ``sample`` (positions into train_idx, [S]) then replaces the G-CRD / GSP on-device row draw."""
        if sample is not None and self.objective is None:
            raise ValueError("sample= is the G-CRD row sample; this trainer has no G-CRD head")
        if aux is not None and self.objective is not None:
            raise ValueError("aux= and the trainer's G-CRD / LSP objective are two auxiliary losses; pass one")
        # the multi-GPU engines override _step_impl with the four step inputs only
        self._step_impl(x, y, train_idx, teacher_logits, *(() if sample is None and aux is None else (sample, aux, beta)))
        return self.loss_out

    def capture(self, x, y, train_idx, teacher_logits=None, warmup: int = 2, key: int = 0):
        """Capture the step on static input buffers (after ``warmup`` training steps on them); afterwards ``replay(key)`` runs
        one full step.  Several input-buffer sets can be captured (key = 0, 1, ...) so that uploads of the next step's inputs
        overlap the current step (activations and parameters are shared between the graphs)."""
        self._static.update(x=x, y=y, train_idx=train_idx, teacher=teacher_logits)
        if self._graph is None:
            self._graph = {}
        self._graph[key] = capture_graph(lambda: self._step_impl(x, y, train_idx, teacher_logits), warmup)
        return self

    def replay(self, key: int = 0) -> torch.Tensor:
        self._graph[key].replay()
        return self.loss_out

    def launches_per_step(self) -> int:
        """b200gnn kernel launches in one training step on the captured inputs (counted, not estimated); advances the state
        by one step."""
        before = lib.launch_count()
        st = self._static
        self._step_impl(st["x"], st["y"], st["train_idx"], st["teacher"])
        return lib.launch_count() - before
