"""G-CRD on PPI without a GPU: the fp64 restatement (oracle.ppi_gcrd.gcrd_step: StudentNet, both projection heads, InfoNCE, one
Adam step) reproduces one step of the reference's own train() with --training nce (tests/golden/ppi_gcrd.pt,
make_golden_ppi_gcrd.py) with every row and with a recorded 128-row draw, and gcrd.PerGraphGCRD refuses malformed
per-graph inputs before it touches a device."""
from pathlib import Path

import pytest
import torch

from efficient_gnns_b200.criterion import nce_chunk_rows
from efficient_gnns_b200.gcrd import PerGraphGCRD
from oracle import ppi as oppi, ppi_gcrd as opg
from test_oracle_ppi_lsp import T_FEAT, after_entries

GOLD = torch.load(Path(__file__).resolve().parent / "golden" / "ppi_gcrd.pt")
CASES = ["full", "s128"]


def oracle_gcrd_step(case: str, dtype=torch.float64):
    """The fixture's step restated in ``dtype`` (oracle.ppi_gcrd.gcrd_step on the designed graph, seeded model and heads)."""
    c = GOLD["cases"][case]
    model = oppi.seeded_state(oppi.layers_of("student", GOLD["out_channels"]), GOLD["in_channels"], GOLD["seeds"]["student"])
    sproj, tproj = opg.seeded_heads(136, 1024, GOLD["proj_dim"], GOLD["seeds"]["heads"])
    return opg.gcrd_step(GOLD["x"], GOLD["y"].to(dtype), GOLD["edge_index"].long(), model, sproj, tproj, T_FEAT, c["sample"],
                          beta=GOLD["beta"], nce_T=GOLD["nce_T"], lr=GOLD["lr"], dtype=dtype)


def test_fixture_cases():
    n = GOLD["x"].shape[0]
    assert GOLD["cases"]["full"]["max_samples"] >= n and GOLD["cases"]["full"]["sample"] is None
    s = GOLD["cases"]["s128"]["sample"]
    assert s.numel() == 128 and s.unique().numel() == 128 and 0 <= int(s.min()) and int(s.max()) < n
    assert (Path(__file__).resolve().parent / "golden" / "ppi_gcrd.pt").stat().st_size < 1 << 20


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_nce_step(case):
    c = GOLD["cases"][case]
    got = oracle_gcrd_step(case)
    for a, b in zip(got["loss"], c["loss"]):
        assert abs(float(a) - float(b)) <= 1e-5 * abs(float(b)), (got["loss"], c["loss"])
    for group, fps in c["grads"].items():
        assert set(fps) == set(got["grads"][group]), group
        for k, fp_gold in fps.items():
            if group != "model" and k == "0.bias":
                # a bias in front of BatchNorm: its exact gradient is 0, the reference's carries rounding only
                scale = max(v.abs().max().item() for v in fps["0.weight"].values())
                assert got["grads"][group][k].abs().max() < 1e-12 * scale, group
                assert fp_gold["full"].abs().max() < 1e-6 * scale, group
                continue
            fp = oppi.fingerprint(got["grads"][group][k])
            for part, v in fp_gold.items():
                a, b = fp[part].double(), v.double()
                assert (a - b).abs().max() <= 1e-4 * max(b.abs().max().item(), 1e-30), (group, k, part)
    for group, entries in c["after"].items():
        for k, ref in entries.items():
            if group != "model" and k == "0.bias":
                continue          # Adam's first step moves it by lr * sign(rounding noise)
            # Adam's first step moves a parameter by lr * g / (|g| + eps): compared where the gradient is clearly nonzero
            g = got["grads"][group][k].reshape(-1)
            idx = after_entries(g.numel())
            keep = g[idx].abs() > 1e-2 * g.abs().max()
            assert keep.any(), (group, k)
            assert (got["after"][group][k].reshape(-1)[idx][keep] - ref[keep].double()).abs().max() <= 1e-5, (group, k)
    for group, sd in c["running"].items():
        for k in ("1.running_mean", "1.running_var"):
            ref = sd[k].double()
            assert (got["after"][group][k] - ref).abs().max() <= 1e-5 * max(ref.abs().max().item(), 1.0), (group, k)
        assert int(sd["1.num_batches_tracked"]) == 1


def test_the_draw_changes_the_loss():
    """The two cases differ only in the sample, so the recorded draw is what the 128-row case tests."""
    full, s128 = GOLD["cases"]["full"]["loss"], GOLD["cases"]["s128"]["loss"]
    assert full[1] == s128[1] and abs(float(full[2] - s128[2])) > 1e-3


def feats(sizes=(40, 55), width=24):
    gen = torch.Generator().manual_seed(0)
    return [torch.randn(n, width, generator=gen) for n in sizes]


def test_per_graph_gcrd_refuses_malformed_inputs():
    t = feats()
    for kw in (dict(teacher_feat=[]),                                           # no graphs
               dict(teacher_feat=[t[0], t[1][0]]),                              # not [n, F_t]
               dict(teacher_feat=[t[0], torch.randn(55, 28)]),                  # two teacher widths
               dict(teacher_feat=feats(width=2052)),                            # wider than the teacher head's GEMM takes
               dict(hidden=516),                                                # wider than the student head's GEMM takes
               dict(hidden=134),                                                # not a multiple of 4
               dict(proj_dim=100), dict(proj_dim=288), dict(proj_dim=32),       # not a multiple of 32 in (48, 256]
               dict(max_samples=0)):
        with pytest.raises(ValueError):
            PerGraphGCRD(**{"teacher_feat": t, "hidden": 136, "device": "cpu", **kw})


def test_per_graph_buffers_have_each_graphs_eager_geometry():
    """Every graph's InfoNCE buffers are views at its own pitch Sp with nce_chunk_rows(Sp) chunk rows, as the eager
    nce_criterion would allocate them (two chunks at n = 3,260, one below); the operands' padding rows follow the last
    real row of the largest sample, so no graph writes another's padding."""
    sizes = (3260, 1500, 3257, 700)
    obj = PerGraphGCRD(feats(sizes, 1024), 136, device="cpu")
    for r, n in zip(obj.graphs, sizes):
        Sp = (n + 3) // 4 * 4
        assert (r.n, r.S, r.Sp) == (n, n, Sp)
        assert tuple(r.nce.Z.shape) == (nce_chunk_rows(Sp), Sp) and tuple(r.nce.g_t.shape) == (Sp, 256)
        assert tuple(r.pre_s.shape) == (n, 256) and tuple(r.x_s.shape) == (Sp, 256)
        assert r.nce.Z.data_ptr() == obj.graphs[0].nce.Z.data_ptr()          # one flat buffer, viewed per graph
        assert r.loss_aux.data_ptr() == obj.loss_aux.data_ptr()
        end = (r.x_s.data_ptr() - obj.graphs[0].x_s.data_ptr()) // 4 + r.S * 256
        assert end == 3260 * 256                                                # real rows end where the largest ends
    assert -(-3260 // nce_chunk_rows(3260)) == 2 and nce_chunk_rows(1500) == 1500
    assert obj.sample_ws is None and all(torch.equal(r.inds, torch.arange(r.n, dtype=torch.int32)) for r in obj.graphs)
    drawn = PerGraphGCRD(feats(sizes, 1024), 136, max_samples=1000, device="cpu")
    assert [r.S for r in drawn.graphs] == [1000, 1000, 1000, 700] and drawn.sample_ws is not None
