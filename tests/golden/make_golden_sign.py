"""SIGN model fixture: the reference's OWN `SIGN` class (arxiv_dgl/sign.py:105-157), unmodified.

    python tests/golden/make_golden_sign.py        REFERENCE=<checkout of the reference repository>   (not run by the test suite)

Same method as make_golden.py (whose stand-in modules are reused so that sign.py imports): the reference file computes.
  * sign_model_arxiv.pt — 3 hops of 16 features, hidden 32, 8 classes, for n_layers (ff_layer) 1, 2, 3 with non-default
                          PReLU slopes: the state, eval-mode logits / out_feat of every node, and a train-mode forward /
                          backward with dropout and input dropout set to 0 (cross-entropy over a batch): loss and every
                          parameter gradient, the slopes included.
oracle/sign.py (tests, -m "not gpu") and SIGNStudentTrainer (tests, -m gpu) must reproduce it.
"""
from __future__ import annotations

import importlib
import sys
import types

import torch

import make_golden as mg


def sign_model_fixture(sign):
    g = torch.Generator().manual_seed(31)
    n, f_in, hid, n_cls, hops = 70, 16, 32, 8, 3
    feats = [torch.randn(n, f_in, generator=g) for _ in range(hops)]
    labels = torch.randint(0, n_cls, (n,), generator=g)
    batch = torch.randperm(n, generator=g)[:45]
    models = {}
    for ff in (1, 2, 3):
        torch.manual_seed(40 + ff)
        m = sign.SIGN(f_in, hid, n_cls, hops, ff, 0.5, 0.1)
        slopes = [mod for mod in m.modules() if isinstance(mod, torch.nn.PReLU)]
        with torch.no_grad():
            for i, mod in enumerate(slopes):
                mod.weight.fill_((-0.35, 0.1, 0.6, 0.0, -0.05)[i % 5])
        m.eval()
        with torch.no_grad():
            logits_eval = m(feats)
            out_feat_eval = m.out_feat.clone()
        m0 = sign.SIGN(f_in, hid, n_cls, hops, ff, 0.0, 0.0)
        m0.load_state_dict(m.state_dict())
        m0.train()
        logits = m0([x[batch] for x in feats])
        loss = torch.nn.functional.cross_entropy(logits, labels[batch])
        loss.backward()
        models[ff] = dict(state={k: v.detach().clone() for k, v in m.state_dict().items()}, logits_eval=logits_eval,
                          out_feat_eval=out_feat_eval, logits_train=logits.detach(), out_feat_train=m0.out_feat.detach(),
                          loss=loss.detach(), grads={k: q.grad.detach().clone() for k, q in m0.named_parameters()})
    torch.save(dict(feats=feats, labels=labels, batch=batch, hidden=hid, n_classes=n_cls, models=models),
               mg.OUT / "sign_model_arxiv.pt")


def main():
    mg.install_stubs()
    mg.install_dgl_stubs()
    sys.modules["ogb.nodeproppred"].DglNodePropPredDataset = None
    if "torch.utils.tensorboard" not in sys.modules:
        try:
            importlib.import_module("torch.utils.tensorboard")
        except Exception:                                    # tensorboard is not installed everywhere: sign.py only names it
            tb = types.ModuleType("torch.utils.tensorboard")
            tb.SummaryWriter = None
            sys.modules["torch.utils.tensorboard"] = tb
    sys.path.insert(0, str(mg.REF / "arxiv_dgl"))
    sign_model_fixture(importlib.import_module("sign"))
    print("wrote", mg.OUT / "sign_model_arxiv.pt")


if __name__ == "__main__":
    main()
