"""Generate tests/golden/sign_gcrd.pt by running the REFERENCE's own ``train_kd_and_aux`` of arxiv_dgl/sign.py (:293-383)
with ``--training nce`` for one step: the SIGN student and its projection head learning from teacher features through the
teacher's projection head and ``kd_criterion + beta * nce_criterion(...)[2]`` (criterion.py:95-115), one Adam over the model
and both heads (:421-438).

    REFERENCE=<checkout of the reference repository> python tests/golden/make_golden_sign_gcrd.py   (not run by the suite)

The stubs are make_golden_sign.py's.  Designed input: 70 nodes, 3 hops of 16 features, hidden 32, 8 classes, one batch of
45 nodes, teacher logits and 22-wide teacher features (750 in the scripts; 22 keeps the file small and still needs the
engine's zero padding to a 16-byte pitch).  Every nn.Dropout of the model multiplies by a recorded keep mask, the one
SIGNStudentTrainer(seed=0) itself draws at step 0 (oracle.sign_gcrd.engine_masks, the CPU restatement of its Philox keep
decisions), so that the engine's step is compared with the fixture directly.  The heads are built as the reference's run()
builds them, nn.Sequential(Linear, BatchNorm1d, ReLU), and start from ``oracle.ppi_gcrd.seeded_heads`` (seed 404), so no
head state is stored.  Hyper-parameters are the SIGN script's (scripts/run_all_kd_and_aux.sh: beta 0.1, nce_T 0.075,
lr 0.001, dropout 0.5, input dropout 0.1; alpha 0.9, kd_T 4 from argparse) with proj_dim 64.  Cases, for ff_layer 1 and 2:

    ff{1,2}/all       max_samples 16384 >= 45: every row, no draw
    ff{1,2}/sampled   max_samples 12: numpy is seeded before the step and the draw np.random.choice makes inside
                      nce_criterion is recorded by wrapping it

Recorded per case: the three losses, every gradient of the model and of both heads, every parameter after Adam, and the
heads' running statistics and num_batches_tracked."""
from __future__ import annotations

import argparse
import importlib
import sys
import types
from pathlib import Path

import numpy as np
import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; the stub modules have no __spec__ to scan)

sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(__file__).resolve().parents[2]))
import make_golden as mg  # noqa: E402

from oracle import ppi_gcrd as opg, sign_gcrd as osg  # noqa: E402

N, F_IN, HID, C, HOPS, B, F_T = 70, 16, 32, 8, 3, 45, 22
BETA, NCE_T, PROJ, LR, ALPHA, KD_T, P, P_IN = 0.1, 0.075, 64, 0.001, 0.9, 4.0, 0.5, 0.1
SEEDS = dict(data=51, model=60, heads=404, numpy=13, dropout=0)
CASES = {f"ff{ff}/{kind}": (ff, ms) for ff in (1, 2) for kind, ms in (("all", 16384), ("sampled", 12))}


class _Recorded(torch.nn.Module):
    """nn.Dropout(p) in training that multiplies by the next of its recorded keep masks."""

    def __init__(self, p, masks):
        super().__init__()
        self.p, self.masks = p, list(masks)

    def forward(self, x):
        return x * self.masks.pop(0).to(x.dtype) / (1 - self.p)


def inject_masks(model, masks, ff):
    model.input_drop = _Recorded(P_IN, masks["input"])
    model.dropout = _Recorded(P, [masks["cat"]])
    if ff > 1:
        for h, f in enumerate(model.inception_ffs):
            f.dropout = _Recorded(P, masks["hidden"][h])
        model.project.dropout = _Recorded(P, masks["project"])


def heads():
    s_sd, t_sd = opg.seeded_heads(HOPS * HID, F_T, PROJ, SEEDS["heads"])
    sp = torch.nn.Sequential(torch.nn.Linear(HOPS * HID, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    tp = torch.nn.Sequential(torch.nn.Linear(F_T, PROJ), torch.nn.BatchNorm1d(PROJ), torch.nn.ReLU())
    sp.load_state_dict(s_sd)
    tp.load_state_dict(t_sd)
    return sp, tp


def main():
    assert mg.REF.exists(), "set REFERENCE to a checkout of the reference repository"
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
    sign = importlib.import_module("sign")

    # the draw np.random.choice makes inside nce_criterion
    seen = {}
    choice = np.random.choice

    def choice_rec(*a, **k):
        seen["sample"] = r = choice(*a, **k)
        return r

    np.random.choice = choice_rec

    g = torch.Generator().manual_seed(SEEDS["data"])
    feats = [torch.randn(N, F_IN, generator=g) for _ in range(HOPS)]
    labels = torch.randint(0, C, (N,), generator=g)
    t_logits = torch.randn(N, C, generator=g) * 2
    t_feat = torch.randn(N, F_T, generator=g)
    batch = torch.randperm(N, generator=g)[:B]
    out = dict(feats=feats, labels=labels, teacher_logits=t_logits, teacher_feat=t_feat, batch=batch, hidden=HID,
               n_classes=C, beta=BETA, nce_T=NCE_T, proj_dim=PROJ, lr=LR, alpha=ALPHA, kd_T=KD_T, dropout=P,
               input_drop=P_IN, seeds=SEEDS, states={}, cases={})
    for ff in (1, 2):
        torch.manual_seed(SEEDS["model"] + ff)
        m = sign.SIGN(F_IN, HID, C, HOPS, ff, P, P_IN)
        with torch.no_grad():                                # slopes of both signs
            for i, mod in enumerate(mm for mm in m.modules() if isinstance(mm, torch.nn.PReLU)):
                mod.weight.fill_((-0.3, 0.2, 0.45, -0.1)[i % 4])
        out["states"][ff] = {k: v.detach().clone() for k, v in m.state_dict().items()}
    for name, (ff, max_samples) in CASES.items():
        m = sign.SIGN(F_IN, HID, C, HOPS, ff, P, P_IN)
        m.load_state_dict(out["states"][ff])
        inject_masks(m, osg.engine_masks(HOPS, F_IN, HID, ff, B, P, P_IN, SEEDS["dropout"], 0), ff)
        sp, tp = heads()
        opt = torch.optim.Adam([{"params": m.parameters(), "lr": LR, "weight_decay": 0},
                                {"params": sp.parameters(), "lr": LR, "weight_decay": 0},
                                {"params": tp.parameters(), "lr": LR, "weight_decay": 0}])
        args = argparse.Namespace(training="nce", beta=BETA, nce_T=NCE_T, max_samples=max_samples, alpha=ALPHA, kd_T=KD_T)
        seen.clear()
        np.random.seed(SEEDS["numpy"])
        loss, loss_cls, loss_aux = sign.train_kd_and_aux(m, feats, labels, opt, [batch], args, t_feat, t_logits, sp, tp)
        sample = torch.from_numpy(seen["sample"]).to(torch.int64) if "sample" in seen else None
        groups = dict(model=m, sproj=sp, tproj=tp)
        out["cases"][name] = dict(
            ff=ff, max_samples=max_samples, sample=sample,
            loss=torch.tensor([loss, loss_cls, loss_aux], dtype=torch.float64),
            grads={g: {k: p.grad.detach().clone() for k, p in mod.named_parameters()} for g, mod in groups.items()},
            after={g: {k: p.detach().clone() for k, p in mod.named_parameters()} for g, mod in groups.items()},
            running={g: {k: v.clone() for k, v in mod.state_dict().items() if "running" in k or "num_batches" in k}
                     for g, mod in (("sproj", sp), ("tproj", tp))})
    np.random.choice = choice
    torch.save(out, mg.OUT / "sign_gcrd.pt")
    print("wrote sign_gcrd.pt", (mg.OUT / "sign_gcrd.pt").stat().st_size, "bytes")


if __name__ == "__main__":
    main()
