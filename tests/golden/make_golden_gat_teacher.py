"""Generate tests/golden/gat_teacher_arxiv.pt by running the REFERENCE's own arxiv_dgl/gat.py (``adjust_learning_rate``,
``train``, ``evaluate``) and models.py, unmodified, with torch.optim.RMSprop, on the ``dgl`` stand-in of make_golden.py.

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_gat_teacher.py   (not run by the suite)

designed_graph() of make_golden_gat_model.py (symmetric + self-loops, a hub, degree-1 rows), F = 16 features, C = 8
classes, 3 layers of 3 heads x 10, use_norm, no attn_dst, all dropouts and edge drop 0 (their draws cannot be shared).
Three epochs per case: use_labels with one label iteration, and no labels with none.  The label mask of each epoch is
recorded by drawing it once more between a save and a restore of the CPU generator state; ``train`` itself draws it.
To keep the file small, evaluate()'s prediction and ``feat`` are kept for the last epoch only (the losses and accuracies
of every epoch are kept) and the graph indices are stored as int32."""
from __future__ import annotations

import argparse
import importlib
import sys
import types
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as mg  # noqa: E402
from make_golden_gat_model import designed_graph  # noqa: E402

N_EPOCHS = 3


def install_gat_script_stubs():
    na = lambda *a, **k: (_ for _ in ()).throw(NotImplementedError("stub"))  # noqa: E731
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    mpl.ticker = types.ModuleType("matplotlib.ticker")
    mpl.ticker.AutoMinorLocator = mpl.ticker.MultipleLocator = na
    sys.modules.update({"matplotlib": mpl, "matplotlib.pyplot": mpl.pyplot, "matplotlib.ticker": mpl.ticker})
    sys.modules["ogb.nodeproppred"].DglNodePropPredDataset = na


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
    mg.install_stubs()
    mg.install_dgl_stubs()
    install_gat_script_stubs()
    sys.path.insert(0, str(mg.REF / "arxiv_dgl"))
    gat = importlib.import_module("gat")
    n, F_in, C, D, H, L = 700, 16, 8, 10, 3, 3
    row, col = designed_graph(n)
    g = torch.Generator().manual_seed(23)
    x = torch.randn(n, F_in, generator=g)
    y = torch.randint(0, C, (n,), generator=g)
    perm = torch.randperm(n, generator=g)
    train_idx, val_idx, test_idx = perm[:350].sort().values, perm[350:520].sort().values, perm[520:].sort().values
    graph = mg._DGLGraph(col, row, n)
    graph.ndata["feat"] = x
    gat.device = torch.device("cpu")
    gat.n_node_feats, gat.n_classes = F_in, C
    labels = y.view(-1, 1)

    def evaluator(pred, lab):                                                   # gat.py:187-189 with ogb's accuracy
        return (pred.argmax(dim=-1, keepdim=True) == lab).float().mean().item()

    out = {}
    for name, use_labels, iters in (("labels", True, 1), ("no_labels", False, 0)):
        args = argparse.Namespace(use_labels=use_labels, n_label_iters=iters, mask_rate=0.5, no_attn_dst=True, use_norm=True,
                                  lr=0.002, n_layers=L, n_heads=H, n_hidden=D, dropout=0.0, input_drop=0.0, attn_drop=0.0,
                                  edge_drop=0.0, wd=0.0)
        torch.manual_seed(11)
        model = gat.gen_model(args)
        optimizer = torch.optim.RMSprop(model.parameters(), lr=args.lr, weight_decay=args.wd)
        names = [k for k, _ in model.named_parameters()]
        case = dict(names=names, state0={k: v.detach().clone() for k, v in model.state_dict().items()}, epochs=[])
        for epoch in range(1, N_EPOCHS + 1):
            gat.adjust_learning_rate(optimizer, args.lr, epoch)
            rng = torch.get_rng_state()
            mask = torch.rand(train_idx.shape) < args.mask_rate                # the draw train() is about to make
            torch.set_rng_state(rng)
            acc, loss = gat.train(args, model, graph, labels, train_idx, val_idx, test_idx, optimizer, evaluator)
            res = gat.evaluate(args, model, graph, labels, train_idx, val_idx, test_idx, evaluator)
            train_acc, val_acc, test_acc, train_loss, val_loss, test_loss, pred, feat = res
            case["epochs"].append(dict(
                mask=mask, lr=optimizer.param_groups[0]["lr"], acc=acc, loss=loss, train_acc=train_acc, val_acc=val_acc,
                test_acc=test_acc, train_loss=train_loss.item(), val_loss=val_loss.item(), test_loss=test_loss.item(),
                pred=pred.clone() if epoch == N_EPOCHS else None, feat=feat.clone() if epoch == N_EPOCHS else None,
                params={k: v.detach().clone() for k, v in model.named_parameters()},
                square_avg={k: optimizer.state[v]["square_avg"].clone() for k, v in model.named_parameters()},
                running={k: v.clone() for k, v in model.state_dict().items() if "running" in k or "num_batches" in k}))
        out[name] = case
    torch.save(dict(row=row.int(), col=col.int(), x=x, y=y, train_idx=train_idx, val_idx=val_idx, test_idx=test_idx, n_layers=L, n_heads=H,
                    n_hidden=D, n_classes=C, cases=out), mg.OUT / "gat_teacher_arxiv.pt")
    print("wrote gat_teacher_arxiv.pt")


if __name__ == "__main__":
    main()
