"""The arxiv GAT teacher's training recipe (arxiv_dgl/gat.py, the flags of scripts/gat-teachers.sh) on the fused GAT step.

One epoch of the reference (gat.py:203-222) is ``adjust_learning_rate`` -> ``train`` -> ``evaluate`` -> keep the prediction
and ``model.feat`` of the epoch with the lowest validation loss.  Here it is, with no host read:

    train_step   label_inputs      the random label mask (a Philox stream of the step), roles, the one-hot label block of
                                   the persistent [N, F + C] input and the device count of loss rows, in one launch
                 forward           training mode (fresh dropout / input-drop / edge-drop streams per forward)
                 n_label_iters x   label_softmax of the prediction into the label block of the loss / val / test rows, forward
                 logce             log(eps + CE) over the loss rows, its gradient, the accuracy over train_idx
                 backward, rmsprop RMSprop with the linear warm-up read from the step counter, which it then increments
    evaluate     label_inputs (every training label), eval-mode forwards, split_eval (losses / accuracies of three splits)
    snapshot     if val loss < best: copy the logits and the last hidden layer's eval-mode state (pre-BatchNorm output and
                 scale / shift), from which ``feat`` is formed once in save()

``capture()`` records one epoch as one CUDA graph; ``run()`` replays it and keeps the reference's eight learning-curve
values per epoch.  ``save()`` writes the reference's four artefacts (output / logits / features / checkpoints).
"""
from __future__ import annotations

import argparse
from collections import OrderedDict
from pathlib import Path
from typing import Dict, Optional

import torch

from . import ops
from .engine_gat import GATTrainer
from .sparse import SparseTensor
from .trainer import capture_graph

HISTORY_COLUMNS = ("acc", "train_acc", "val_acc", "test_acc", "loss", "train_loss", "val_loss", "test_loss")
WARMUP_EPOCHS = 50          # adjust_learning_rate, gat.py:110-113
RMSPROP_ALPHA, RMSPROP_EPS = 0.99, 1e-8


class GATTeacherTrainer(GATTrainer):
    """GAT teacher of arxiv_dgl/gat.py on one GPU; the defaults are the teacher preset of scripts/gat-teachers.sh
    (--use-norm --use-labels --n-label-iters=1 --no-attn-dst --edge-drop=0.3 --input-drop=0.25, dropout 0.75, lr 0.002,
    3 layers of 3 heads x 250).  adj: bidirected with self-loops, rows = destinations."""

    def __init__(self, adj: SparseTensor, x: torch.Tensor, labels: torch.Tensor, split_idx: Dict[str, torch.Tensor],
                 n_classes: Optional[int] = None, use_labels: bool = True, n_label_iters: int = 1, mask_rate: float = 0.5,
                 n_hidden: int = 250, n_layers: int = 3, n_heads: int = 3, dropout: float = 0.75, input_drop: float = 0.25,
                 attn_drop: float = 0.0, edge_drop: float = 0.3, no_attn_dst: bool = True, use_norm: bool = True,
                 lr: float = 0.002, wd: float = 0.0, seed: int = 0):
        if not use_labels and n_label_iters > 0:
            raise ValueError("'--use-labels' must be enabled when n_label_iters > 0")      # gat.py:337-338
        if not 0.0 <= mask_rate < 1.0:
            raise ValueError("mask_rate must be in [0, 1)")
        dev = adj.device
        labels = labels.reshape(-1).to(dev, torch.int64)
        C = int(labels.max().item()) + 1 if n_classes is None else int(n_classes)
        F = x.shape[1]
        self.n_node_feats, self.use_labels, self.n_label_iters = F, bool(use_labels), int(n_label_iters)
        self.mask_rate, self.wd = float(mask_rate), float(wd)
        self.n_fwd = self.n_label_iters + 1
        L = int(n_layers)
        # Philox streams of one step: 2 L per training forward, then the label mask
        super().__init__(adj, F + C if use_labels else F, C, n_hidden, n_layers, n_heads, dropout=dropout,
                         input_drop=input_drop, edge_drop=edge_drop, use_attn_dst=not no_attn_dst, use_symmetric_norm=use_norm,
                         lr=lr, seed=seed, attn_drop=attn_drop, step_streams=self.n_fwd * 2 * L + 1)
        self.no_attn_dst, self.use_norm, self.p_attn = bool(no_attn_dst), bool(use_norm), float(attn_drop)
        N = self.N
        self.square_avg = self.exp_avg_sq                                    # RMSprop's one moment (exp_avg stays zero)
        self.X = torch.zeros(N, self.in_feats, device=dev)                   # [x | label block], persistent
        self.X[:, :F] = x.to(dev, torch.float32)
        self.labels = labels
        self.train_idx, self.val_idx, self.test_idx = (split_idx[k].reshape(-1).to(dev, torch.int64) for k in ("train", "valid", "test"))
        self.sizes = (self.train_idx.numel(), self.val_idx.numel(), self.test_idx.numel())
        self.idx_all = torch.cat([self.train_idx, self.val_idx, self.test_idx])
        self.row_pos = torch.full((N,), -2, dtype=torch.int32, device=dev)
        self.row_pos[torch.cat([self.val_idx, self.test_idx])] = -1
        self.row_pos[self.train_idx] = torch.arange(self.sizes[0], dtype=torch.int32, device=dev)
        self.role = torch.zeros(N, dtype=torch.uint8, device=dev)
        self.cnt_part = torch.zeros(ops.teacher_slots(N), dtype=torch.int32, device=dev)
        self.part_train = torch.empty(6 * ops.teacher_slots(self.sizes[0]), dtype=torch.float64, device=dev)
        self.part_eval = torch.empty(6 * ops.teacher_slots(sum(self.sizes)), dtype=torch.float64, device=dev)
        self.row = torch.zeros(len(HISTORY_COLUMNS), device=dev)             # this epoch's learning-curve values
        self.best = torch.full((1,), float("inf"), device=dev)               # best validation loss so far
        h = L - 2
        self.best_logits = torch.zeros_like(self.Y[-1])
        self.best_Y = torch.zeros_like(self.Y[h])
        self.best_bn = torch.zeros_like(self.bn_eval[h])
        self._epoch_graph: Optional[torch.cuda.CUDAGraph] = None

    # ------------------------------------------------------------------ the epoch
    def mask_offset(self, step: int) -> int:
        """Philox offset of the label mask of training step ``step`` (b200gnn_dropout_mask_u8 at p = mask_rate)."""
        return self.n_fwd * 2 * self.L + step * self.step_mul

    def _label_block(self) -> torch.Tensor:
        return self.X[:, self.n_node_feats:]

    def train_step(self, mask: Optional[torch.Tensor] = None):
        """gat.py:116-148 after adjust_learning_rate.  mask (bool [n_train], optional) replaces the step's label-mask draw,
        e.g. to replay a recorded torch.rand draw.  Returns the device scalars (acc, loss); no host sync."""
        F, C, L = self.n_node_feats, self.n_classes, self.L
        ops.label_inputs(self.X, F, C, self.row_pos, self.labels, self.role, self.cnt_part, eval=False,
                         use_labels=self.use_labels, mask_rate=self.mask_rate, seed=self.seed, offset=self.mask_offset(0),
                         step_dev=self.step_count, step_mul=self.step_mul,
                         mask=None if mask is None else mask.to(self.device, torch.uint8).contiguous())
        self.forward(self.X, training=True)
        for it in range(self.n_label_iters):
            ops.label_softmax(self.Y[-1], C, self._label_block(), self.role, (1 << ops.ROLE_PRED) | (1 << ops.ROLE_EVAL))
            self.forward(self.X, training=True, stream_base=(it + 1) * 2 * L)
        self.dY[-1].zero_()
        ops.logce_fwd_bwd(self.Y[-1], C, self.train_idx, self.labels, self.role, self.cnt_part, self.dY[-1], self.row[4:5],
                          self.row[0:1], self.part_train)
        self.backward(self.X)
        ops.rmsprop_step(self.params, self.grads, self.square_avg, self.step_count, self.lr, WARMUP_EPOCHS, RMSPROP_ALPHA,
                         RMSPROP_EPS, self.wd)
        return self.row[0], self.row[4]

    def evaluate(self):
        """gat.py:151-183: eval-mode prediction from every training label.  Returns the device vectors
        ([train, val, test] accuracies, [train, val, test] losses); no host sync."""
        F, C = self.n_node_feats, self.n_classes
        ops.label_inputs(self.X, F, C, self.row_pos, self.labels, self.role, self.cnt_part, eval=True, use_labels=self.use_labels)
        self.forward(self.X, training=False)
        for _ in range(self.n_label_iters):
            ops.label_softmax(self.Y[-1], C, self._label_block(), self.role, 1 << ops.ROLE_EVAL)
            self.forward(self.X, training=False)
        ops.split_eval(self.Y[-1], C, self.idx_all, self.sizes, self.labels, self.row[5:8], self.row[1:4], self.part_eval)
        return self.row[1:4], self.row[5:8]

    def snapshot(self):
        """Keep the last evaluate()'s logits and hidden state if its validation loss is strictly the lowest so far."""
        h = self.L - 2
        ops.snapshot_if_better(self.row[6:7], self.best, [(self.Y[-1], self.best_logits), (self.Y[h], self.best_Y),
                                                          (self.bn_eval[h], self.best_bn)])

    def _epoch_impl(self):
        self.train_step()
        self.evaluate()
        self.snapshot()

    def epoch(self) -> torch.Tensor:
        """One epoch, eagerly: the device vector of HISTORY_COLUMNS."""
        self._epoch_impl()
        return self.row

    def capture(self):
        """Record one epoch (train, evaluate, snapshot, history row) as one CUDA graph.  Capturing runs nothing."""
        self._epoch_graph = capture_graph(self._epoch_impl, warmup=0)
        return self

    def replay(self) -> torch.Tensor:
        self._epoch_graph.replay()
        self._training = False
        return self.row

    def run(self, n_epochs: int, log_every: int = 20) -> torch.Tensor:
        """n_epochs graph replays; the host reads the history every log_every epochs (0: only at the end).  Returns the
        [n_epochs, 8] history of HISTORY_COLUMNS (the reference's accs, train_accs, ..., test_losses lists), on the CPU."""
        if self._epoch_graph is None:
            self.capture()
        hist = torch.empty(n_epochs, len(HISTORY_COLUMNS), device=self.device)
        for e in range(n_epochs):
            self.replay()
            hist[e].copy_(self.row)
            if log_every and ((e + 1) % log_every == 0 or e + 1 == n_epochs):
                v = dict(zip(HISTORY_COLUMNS, hist[e].tolist()))
                print(f"Epoch: {e + 1}/{n_epochs}, Loss: {v['loss']:.4f}, Acc: {v['acc']:.4f}, "
                      f"Train/Val/Test loss: {v['train_loss']:.4f}/{v['val_loss']:.4f}/{v['test_loss']:.4f}, "
                      f"Train/Val/Test acc: {v['train_acc']:.4f}/{v['val_acc']:.4f}/{v['test_acc']:.4f}")
        return hist.cpu()

    # ------------------------------------------------------------------ reference-format state
    def _reference_order(self, sd: Dict[str, torch.Tensor], buffers: bool) -> "OrderedDict[str, torch.Tensor]":
        """Keys in the order of the reference module's state_dict() (parameters() when buffers is False): per GATConv its own
        attn_l, attn_r, then fc.weight, res_fc.weight; per BatchNorm weight, bias (, running statistics, batch count)."""
        out = OrderedDict()
        for l in range(self.L):
            for k in ("attn_l", "attn_r", "fc.weight", "res_fc.weight"):
                if f"convs.{l}.{k}" in sd:
                    out[f"convs.{l}.{k}"] = sd[f"convs.{l}.{k}"]
        for l in range(self.L - 1):
            for k in ("weight", "bias") + (("running_mean", "running_var", "num_batches_tracked") if buffers else ()):
                out[f"norms.{l}.{k}"] = sd[f"norms.{l}.{k}"]
        out["bias_last.bias"] = sd["bias_last.bias"]
        return out

    def steps_taken(self) -> int:
        return int(self.step_count.item())

    def named_parameters(self) -> "OrderedDict[str, torch.Tensor]":
        """The reference module's named_parameters(), in its order (padding removed)."""
        return self._reference_order(self._export(self.Wfc, self.Wres, self.attn_l, self.attn_r, self.gamma, self.beta,
                                                  self.bias_last), buffers=False)

    def named_square_avg(self) -> "OrderedDict[str, torch.Tensor]":
        """RMSprop's square_avg under the parameter names, in parameters() order."""
        lk = lambda t: None if t is None else self.store.like(self.square_avg, t)          # noqa: E731
        return self._reference_order(self._export([[lk(t) for t in W] for W in self.Wfc], [[lk(t) for t in W] for W in self.Wres],
                                                  [lk(t) for t in self.attn_l], [lk(t) for t in self.attn_r],
                                                  [lk(t) for t in self.gamma], [lk(t) for t in self.beta], lk(self.bias_last)),
                                     buffers=False)

    def model_state_dict(self) -> "OrderedDict[str, torch.Tensor]":
        """The reference module's state_dict() on the CPU, num_batches_tracked included (one per training forward)."""
        sd = {k: v.cpu() for k, v in self.state_dict().items()}
        n_batches = torch.tensor(self.steps_taken() * self.n_fwd, dtype=torch.int64)
        for l in range(self.L - 1):
            sd[f"norms.{l}.num_batches_tracked"] = n_batches.clone()
        return self._reference_order(sd, buffers=True)

    def current_lr(self) -> float:
        """The optimizer's rate as adjust_learning_rate last set it."""
        s = self.steps_taken()
        return self.lr * min(s, WARMUP_EPOCHS) / WARMUP_EPOCHS if s > 0 else self.lr

    def optimizer_state_dict(self) -> dict:
        """torch.optim.RMSprop(model.parameters(), lr, weight_decay=wd).state_dict() of the reference after these steps."""
        params = [torch.nn.Parameter(v.detach().cpu().clone()) for v in self.named_parameters().values()]
        opt = torch.optim.RMSprop(params, lr=self.current_lr(), alpha=RMSPROP_ALPHA, eps=RMSPROP_EPS, weight_decay=self.wd)
        step = float(self.steps_taken())
        for p, sq in zip(params, self.named_square_avg().values()):
            opt.state[p] = {"step": torch.tensor(step), "square_avg": sq.detach().cpu().clone()}
        return opt.state_dict()

    def args(self, expt_name: str, n_epochs: int) -> argparse.Namespace:
        """gat.py's argparse namespace (its field names) for this configuration."""
        return argparse.Namespace(cpu=False, gpu=0, seed=self.seed, n_runs=1, n_epochs=n_epochs, use_labels=self.use_labels,
                                  n_label_iters=self.n_label_iters, mask_rate=self.mask_rate, no_attn_dst=self.no_attn_dst,
                                  use_norm=self.use_norm, lr=self.lr, n_layers=self.L, n_heads=self.H, n_hidden=self.n_hidden,
                                  dropout=self.p, input_drop=self.p_in, attn_drop=self.p_attn, edge_drop=self.p_edge,
                                  wd=self.wd, log_every=20, plot_curves=False, save_pred=True, expt_name=expt_name)

    # ------------------------------------------------------------------ artefacts
    def final_pred(self) -> torch.Tensor:
        """Logits [N, n_classes] of the best epoch (gat.py:217-221)."""
        if not bool(torch.isfinite(self.best).all()):
            raise RuntimeError("no evaluation with a finite validation loss has been snapshotted yet")
        return self.best_logits[:, :self.n_classes]

    def final_feat(self) -> torch.Tensor:
        """``model.feat`` of the best epoch: the last hidden activation in eval mode, [N, n_heads * n_hidden]."""
        self.final_pred()
        a = ops.affine_relu_bits(self.best_Y, self.ones_bits, self.best_bn[0], self.best_bn[1], 0.0)
        return a if self.Dp[0] == self.Dl[0] else a[:, self._cols(self.L - 2)].contiguous()

    def save(self, root, expt_name: str, run: int, n_epochs: Optional[int] = None) -> Dict[str, Path]:
        """gat.py:243-258: output/<expt>/<run>.pt = softmax(final_pred), logits/, features/, checkpoints/ = {'args',
        'model_state_dict', 'optimizer_state_dict'}; CPU fp32 tensors at the true widths."""
        logits = self.final_pred()
        prob = ops.label_softmax(logits, self.n_classes, torch.empty(self.N, self.n_classes, device=self.device))
        objs = {"output": prob.cpu(), "logits": logits.contiguous().cpu(), "features": self.final_feat().cpu(),
                "checkpoints": {"args": self.args(expt_name, self.steps_taken() if n_epochs is None else n_epochs),
                                "model_state_dict": self.model_state_dict(),
                                "optimizer_state_dict": self.optimizer_state_dict()}}
        paths = {}
        for d, obj in objs.items():
            p = Path(root) / d / expt_name / f"{run}.pt"
            p.parent.mkdir(parents=True, exist_ok=True)
            torch.save(obj, p)
            paths[d] = p
        return paths

    def n_parameters(self) -> int:
        """count_parameters (gat.py:299-301)."""
        return sum(v.numel() for v in self.named_parameters().values())
