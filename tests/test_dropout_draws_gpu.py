"""Every dropout keep-decision producer, through the C ABI / ops, against the CPU restatement oracle/dropout.py: bit for bit on
both decision paths, keep rates and independence of adjacent streams on 2^24 decisions, and a stream audit of every
training engine (no two draws of a run share Philox counters, eval forwards draw nothing, the layouts DESIGN §4.3 lists)."""
import numpy as np
import pytest
import scipy.stats
import torch

import efficient_gnns_b200  # noqa: F401
from efficient_gnns_b200 import lib, ops, sampling
from efficient_gnns_b200.sparse import SparseTensor
from efficient_gnns_b200.synthetic import skewed_edges
from oracle import dropout as od, graph as og
from oracle.sampling import philox4x32

pytestmark = pytest.mark.gpu

SEED = 0x9E3779B97F4A7C15                 # key k1 != 0
OFF = (1 << 32) + 7                       # counter c3 != 0
KS = [4, 12, 36, 40, 128, 256, 500]       # nvec_row 1, 3, 9, 10, 32, 64, 125: odd rows straddle P16 blocks; partial bit words


def _grid_p() -> float:
    """p = k·2⁻²⁴ with k the 24-bit uniform of one element at (SEED, OFF): that element sits exactly on the threshold."""
    u = philox4x32(SEED, OFF, np.arange(4, dtype=np.uint64)) >> 8
    k = next(int(v) for v in u.reshape(-1)[1:] if v % 256 and (v + 1) % 256)
    return k * 2.0 ** -24


PS = [0.5, 0.25, 2.0 ** -16, 1 - 2.0 ** -16, 0.1, 0.3, _grid_p()]
PS_IDS = ["p16-0.5", "p16-0.25", "p16-min", "p16-max", "24-0.1", "24-0.3", "24-grid"]


def _np(t):
    return t.cpu().numpy()


def _step(v):
    return torch.tensor([v], dtype=torch.int32, device="cuda")


# ------------------------------------------------------------------------------------------------ bit-exact producers
@pytest.mark.parametrize("p", PS, ids=PS_IDS)
@pytest.mark.parametrize("K", KS)
def test_dropout_mask_u8(K, p):
    n = 37
    assert np.array_equal(_np(ops.dropout_mask(n, K, p, SEED, OFF)).astype(bool), od.mask(n, K, p, SEED, OFF))
    assert np.array_equal(_np(ops.dropout_mask(n, K, p, 3, 1)).astype(bool), od.mask(n, K, p, 3, 1))


def test_grid_p_element_is_kept_on_the_threshold():
    """The element p was taken from is kept (u >= p); a `>` comparison would drop it."""
    p = _grid_p()
    m = _np(ops.dropout_mask(1, 16, p, SEED, OFF)).reshape(-1).astype(bool)
    u = (philox4x32(SEED, OFF, np.arange(4, dtype=np.uint64)) >> 8).reshape(-1)
    on = np.flatnonzero(u == round(p * 2 ** 24))
    assert on.size and m[on].all() and np.array_equal(m, od.mask(1, 16, p, SEED, OFF).reshape(-1))


@pytest.mark.parametrize("p", [0.5, 0.3], ids=["p16", "24"])
def test_dropout_mask_step_and_graph_replay(p):
    n = 1001 * 4
    mask = torch.empty(n, dtype=torch.uint8, device="cuda")
    step = _step(3)
    ops.dropout_mask_step(mask, p, SEED, OFF, step, 11)
    assert np.array_equal(_np(mask).astype(bool), od.mask(n // 4, 4, p, SEED, OFF + 33).reshape(-1))
    step.zero_()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.dropout_mask_step(mask, p, SEED, OFF, step, 11)
    for s in range(3):
        step.fill_(s)
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(_np(mask).astype(bool), od.mask(n // 4, 4, p, SEED, OFF + 11 * s).reshape(-1)), s


@pytest.mark.parametrize("p", PS, ids=PS_IDS)
@pytest.mark.parametrize("K", KS)
def test_dropout_bits(K, p):
    for L, n in ((1, 5), (2, 33), (3, 17)):
        words = (K + 31) // 32
        bits = torch.full((L, n, words), -1, dtype=torch.int32, device="cuda")
        ops.dropout_bits(bits, p, SEED, OFF, K=K)
        assert np.array_equal(_np(bits).view(np.uint32), od.bits(L, n, K, p, SEED, OFF)), (L, n)
    ops.dropout_bits(bits, p, SEED, OFF, step_dev=_step(2), step_mul=5, K=K)
    assert np.array_equal(_np(bits).view(np.uint32), od.bits(L, n, K, p, SEED, OFF + 10))


@pytest.mark.parametrize("p", PS, ids=PS_IDS)
@pytest.mark.parametrize("K", KS)
def test_affine_relu_dropout(K, p):
    n = 29
    g = torch.Generator(device="cuda").manual_seed(K)
    y = torch.rand(n, K, device="cuda", generator=g) + 0.5               # relu keeps everything: out != 0 iff kept
    for row_offset, step, mul in ((0, None, 0), (3, None, 0), (4, None, 0), ((1 << 31) + 1, None, 0), (5, 2, 7)):
        out = ops.affine_relu_dropout(y, None, None, True, p, SEED, OFF, step_dev=None if step is None else _step(step),
                                      step_mul=mul, row_offset=row_offset)
        want = od.mask(n, K, p, SEED, OFF + (step or 0) * mul, row_offset=row_offset)
        assert np.array_equal(_np(out != 0), want), row_offset


@pytest.mark.parametrize("p", [0.5, 2.0 ** -16, 0.3, _grid_p()], ids=["p16", "p16-min", "24", "24-grid"])
@pytest.mark.parametrize("K,Kg,col", [(8, 16, 8), (8, 32, 16), (4, 16, 4), (12, 40, 4), (12, 40, 28), (36, 36, 0),
                                      (500, 500, 0), (128, 256, 128), (40, 128, 60)])
def test_affine_relu_dropout_mapped(K, Kg, col, p):
    """Paired (nvec_l, nvec_g, cv_off all even) and unpaired P16 blocks, a permuting rowmap, row_offset >= 2^31."""
    n, N = 31, 97
    g = torch.Generator(device="cuda").manual_seed(K + Kg)
    y = torch.rand(n, K, device="cuda", generator=g) + 0.5
    rowmap = torch.randperm(N, generator=torch.Generator().manual_seed(col))[:n].to(torch.int32)
    out = ops.affine_relu_dropout_mapped(y, None, None, True, p, SEED, OFF, rowmap=rowmap.cuda(), k_global=Kg, col_offset=col)
    assert np.array_equal(_np(out != 0), od.mask_mapped(rowmap.numpy(), K, Kg, col, p, SEED, OFF))
    for r0 in (3, (1 << 31) + 1):
        out = ops.affine_relu_dropout_mapped(y, None, None, True, p, SEED, OFF, step_dev=_step(4), step_mul=3, row_offset=r0,
                                             k_global=Kg, col_offset=col)
        gid = np.arange(r0, r0 + n, dtype=np.uint64)
        assert np.array_equal(_np(out != 0), od.mask_mapped(gid, K, Kg, col, p, SEED, OFF + 12)), r0


@pytest.mark.parametrize("p", [0.5, 0.3], ids=["p16", "24"])
@pytest.mark.parametrize("Kg,cuts", [(40, (0, 12, 20, 40)), (256, (0, 128, 256)), (36, (0, 4, 16, 36))])
def test_sharded_blocks_reassemble_the_full_mask(Kg, cuts, p):
    """Row shards x column shards of a [N, Kg] matrix, each through the mapped pass (and one through the scatter form), put
    together equal the single-matrix mask."""
    N, rows = 53, (0, 17, 30, 53)
    y = torch.rand(N, Kg, device="cuda") + 0.5
    full = torch.zeros(N, Kg, dtype=torch.bool, device="cuda")
    for r0, r1 in zip(rows[:-1], rows[1:]):
        for c0, c1 in zip(cuts[:-1], cuts[1:]):
            blk = ops.affine_relu_dropout_mapped(y[r0:r1, c0:c1].contiguous(), None, None, True, p, SEED, OFF, row_offset=r0,
                                                 k_global=Kg, col_offset=c0)
            full[r0:r1, c0:c1] = blk != 0
    want = od.mask(N, Kg, p, SEED, OFF)
    assert np.array_equal(_np(full), want)
    assert np.array_equal(_np(ops.dropout_mask(N, Kg, p, SEED, OFF)).astype(bool), want)
    # the scatter form: a permuting rowmap, one column block, rows also stored to two destination buffers
    c0, c1 = cuts[0], cuts[1]
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(Kg)).to(torch.int32)
    yb = y[:, c0:c1].contiguous()
    out = torch.empty_like(yb)
    ld = Kg + 4
    dst = [torch.full((n_, ld), float("nan"), device="cuda") for n_ in (20, N - 20)]
    ops.affine_relu_dropout_scatter(yb, None, None, True, p, SEED, OFF, out, None, 0, perm.cuda(), Kg, c0,
                                    [d.data_ptr() for d in dst], [0, 20, N], ld)
    keep = od.mask_mapped(perm.numpy(), c1 - c0, Kg, c0, p, SEED, OFF)
    assert np.array_equal(_np(out != 0), keep)
    assert torch.equal(torch.cat(dst)[:, c0:c1], out)


@pytest.mark.parametrize("p", [0.5, 0.25, 0.1, _grid_p()], ids=["p16", "p16-0.25", "24", "24-grid"])
@pytest.mark.parametrize("F", [4, 12, 36, 128])
def test_sign_gather_hops(F, p):
    n, B = 300, 77
    feats = [torch.rand(n, F, device="cuda") + 0.5 for _ in range(3)]
    idx = torch.randperm(n, device="cuda")[:B]
    out = torch.empty(3, B, F, device="cuda")
    ops.sign_gather(feats, idx, p, SEED, OFF, out)
    assert np.array_equal(_np(out != 0), od.sign_hops(3, B, F, p, SEED, OFF))
    ops.sign_gather(feats, idx, p, SEED, OFF, out, step_dev=_step(2), step_mul=7)
    assert np.array_equal(_np(out != 0), od.sign_hops(3, B, F, p, SEED, OFF + 14))


def _label_masked(role, row_pos, use_labels):
    """masked (rand < mask_rate) of every training position, read back from the roles label_inputs wrote."""
    pos = _np(row_pos)
    r = _np(role)
    tr = np.flatnonzero(pos >= 0)
    out = np.zeros(int(pos.max()) + 1, dtype=bool)
    out[pos[tr]] = (r[tr] == ops.ROLE_INPUT) == use_labels
    return out


@pytest.mark.parametrize("p", [0.5, 0.25, 0.1, 0.3, _grid_p()], ids=["p16", "p16-0.25", "24-0.1", "24-0.3", "24-grid"])
@pytest.mark.parametrize("use_labels", [True, False])
def test_label_inputs_drop_decision(p, use_labels):
    N, n_train, C = 2000, 1203, 8
    gen = torch.Generator().manual_seed(1)
    perm = torch.randperm(N, generator=gen)
    row_pos = torch.full((N,), -2, dtype=torch.int32)
    row_pos[perm[:n_train]] = torch.arange(n_train, dtype=torch.int32)
    row_pos[perm[n_train:n_train + 300]] = -1
    row_pos = row_pos.cuda()
    labels = torch.randint(0, C, (N,), generator=gen).cuda()
    X = torch.zeros(N, 4 + C, device="cuda")
    role = torch.zeros(N, dtype=torch.uint8, device="cuda")
    cnt = torch.zeros(ops.teacher_slots(N), dtype=torch.int32, device="cuda")
    for step, mul in ((None, 0), (3, 13)):
        ops.label_inputs(X, 4, C, row_pos, labels, role, cnt, eval=False, use_labels=use_labels, mask_rate=p, seed=SEED,
                         offset=OFF, step_dev=None if step is None else _step(step), step_mul=mul)
        assert np.array_equal(_label_masked(role, row_pos, use_labels), od.label_drop(n_train, p, SEED, OFF + (step or 0) * mul))


# ------------------------------------------------------------------------------------------------ rates and independence
N_RATE, K_RATE = 1 << 16, 256                               # 2^24 decisions


ALPHA = 2 * scipy.stats.norm.sf(5.0)                        # two-sided 5 sigma


def _band(q, n):
    """The kept count's two-sided 5-sigma interval, from the binomial itself (exact also where n·q is a few units)."""
    return scipy.stats.binom.ppf(ALPHA / 2, n, q), scipy.stats.binom.isf(ALPHA / 2, n, q)


def _within(x, q, n, what):
    lo, hi = _band(q, n)
    assert lo <= round(x * n) <= hi, f"{what}: {x} vs {q} (5-sigma band [{lo / n:.6g}, {hi / n:.6g}])"


@pytest.mark.parametrize("p", [2.0 ** -16, 0.25, 0.5, 0.75, 1 - 2.0 ** -16, 0.1, 0.3],
                         ids=["p16-min", "p16-0.25", "p16-0.5", "p16-0.75", "p16-max", "24-0.1", "24-0.3"])
def test_keep_rate_and_flat_columns(p):
    m = ops.dropout_mask(N_RATE, K_RATE, p, SEED, OFF).float()
    q = od.expected_keep_rate(p)
    _within(m.mean().item(), q, m.numel(), "overall")
    col = m.sum(0).double().cpu().numpy()
    lo, hi = _band(q, N_RATE)
    assert ((col >= lo) & (col <= hi)).all(), (np.flatnonzero((col < lo) | (col > hi)), lo, hi)
    # the P16 pairing: even and odd float4s (columns 0-3 vs 4-7 of each 8) read different words of one block
    lo, hi = m.view(N_RATE, -1, 2, 4)[:, :, 0].mean().item(), m.view(N_RATE, -1, 2, 4)[:, :, 1].mean().item()
    _within(lo, q, m.numel() // 2, "even float4s"); _within(hi, q, m.numel() // 2, "odd float4s")


def _agree(a, b, p, what):
    q = od.expected_keep_rate(p)
    _within((a == b).float().mean().item(), q * q + (1 - q) * (1 - q), a.numel(), what)


@pytest.mark.parametrize("p", [0.5, 0.3], ids=["p16", "24"])
def test_adjacent_streams_are_independent(p):
    N, K = N_RATE, K_RATE
    bits = torch.empty(2, N, K // 32, dtype=torch.int32, device="cuda")
    ops.dropout_bits(bits, p, SEED, OFF, K=K)                  # layer l / l + 1
    u = [(bits[l].view(-1, 1) >> torch.arange(32, device="cuda", dtype=torch.int32)) & 1 for l in range(2)]
    _agree(u[0], u[1], p, "layers")
    m = torch.empty(N * K, dtype=torch.uint8, device="cuda")
    m2 = torch.empty_like(m)
    ops.dropout_mask_step(m, p, SEED, OFF, _step(0), 6)        # step s / s + 1
    ops.dropout_mask_step(m2, p, SEED, OFF, _step(1), 6)
    _agree(m, m2, p, "steps")
    f0 = ops.dropout_mask(N, K, p, SEED, OFF + 3)              # forward f / f + 1 (2L streams apart, L = 3)
    f1 = ops.dropout_mask(N, K, p, SEED, OFF + 3 + 6)
    _agree(f0, f1, p, "forwards")
    feats = [torch.ones(N, K, device="cuda")] * 2              # hop h / h + 1
    out = torch.empty(2, N, K, device="cuda")
    ops.sign_gather(feats, torch.arange(N, device="cuda"), p, SEED, OFF, out)
    _agree(out[0] != 0, out[1] != 0, p, "hops")
    _within((out != 0).float().mean().item(), od.expected_keep_rate(p), out.numel(), "hop rate")


# ------------------------------------------------------------------------------------------------ stream audit per engine
class Recorder:
    """Wraps the ops producers the engines call.  Every draw with p > 0 becomes a record (seed, effective offset, Philox
    blocks, step, phase); for the step ``check_step`` the output is compared with the restatement right after the call."""

    def __init__(self, monkeypatch, check_step=1):
        self.records, self.phase, self.check_step, self.checked = [], "train", check_step, []
        mp = monkeypatch
        for name in ("dropout_bits", "dropout_mask_step", "affine_relu_dropout", "affine_relu_dropout_mapped", "sign_gather",
                     "label_inputs"):
            mp.setattr(ops, name, getattr(self, "_" + name)(getattr(ops, name)))
        self._walk_fn = sampling.random_walk
        mp.setattr(sampling, "random_walk", self._random_walk)
        L = lib.load()
        self._sample_fn = L.b200gnn_gcrd_sample_i32
        mp.setattr(L, "b200gnn_gcrd_sample_i32", self._gcrd_sample)

    def add(self, kind, seed, off, g, p, step):
        self.records.append(dict(kind=kind, seed=int(seed), off=int(off), blocks=od.blocks_of(g, p), step=step,
                                 phase=self.phase))

    @staticmethod
    def _s(step_dev):
        return 0 if step_dev is None else int(step_dev.item())

    def _dropout_bits(self, fn):
        def w(bits, p, seed, offset, step_dev=None, step_mul=0, K=None):
            s = self._s(step_dev)
            L_, n, words = bits.shape
            K_ = 32 * words if K is None else K
            out = fn(bits, p, seed, offset, step_dev=step_dev, step_mul=step_mul, K=K)
            if p > 0:
                for l in range(L_):
                    self.add("bits", seed, offset + s * step_mul + l, np.arange(n * K_ // 4, dtype=np.uint64), p, s)
                if s == self.check_step and self.phase == "train":
                    torch.cuda.synchronize()
                    self.checked.append(np.array_equal(_np(bits).view(np.uint32),
                                                       od.bits(L_, n, K_, p, seed, offset + s * step_mul)))
            return out
        return w

    def _dropout_mask_step(self, fn):
        def w(mask, p, seed, offset, step_dev, step_mul):
            s = self._s(step_dev)
            out = fn(mask, p, seed, offset, step_dev, step_mul)
            if p > 0:
                nv = mask.numel() // 4
                self.add("mask_step", seed, offset + s * step_mul, np.arange(nv, dtype=np.uint64), p, s)
                if s == self.check_step and self.phase == "train":
                    torch.cuda.synchronize()
                    self.checked.append(np.array_equal(_np(mask).astype(bool),
                                                       od.mask(nv, 4, p, seed, offset + s * step_mul).reshape(-1)))
            return out
        return w

    def _affine_relu_dropout(self, fn):
        def w(y, scale=None, shift=None, relu=True, p=0.0, seed=0, offset=0, out=None, step_dev=None, step_mul=0, row_offset=0):
            s = self._s(step_dev)
            res = fn(y, scale, shift, relu, p, seed, offset, out=out, step_dev=step_dev, step_mul=step_mul, row_offset=row_offset)
            if p > 0:
                n, K = y.shape
                g = np.uint64(row_offset * (K // 4)) + np.arange(n * K // 4, dtype=np.uint64)
                self.add("affine", seed, offset + s * step_mul, g, p, s)
                if s == self.check_step and self.phase == "train":
                    act = fn(y, scale, shift, relu, 0.0)
                    vis = _np(act != 0)
                    want = od.mask(n, K, p, seed, offset + s * step_mul, row_offset=row_offset)
                    self.checked.append(np.array_equal(_np(res != 0)[vis], want[vis]))
            return res
        return w

    def _affine_relu_dropout_mapped(self, fn):
        def w(y, scale=None, shift=None, relu=True, p=0.0, seed=0, offset=0, out=None, step_dev=None, step_mul=0, rowmap=None,
              row_offset=0, k_global=None, col_offset=0):
            s = self._s(step_dev)
            res = fn(y, scale, shift, relu, p, seed, offset, out=out, step_dev=step_dev, step_mul=step_mul, rowmap=rowmap,
                     row_offset=row_offset, k_global=k_global, col_offset=col_offset)
            if p > 0:
                n, K = y.shape
                Kg = K if k_global is None else k_global
                gid = (_np(rowmap).astype(np.uint64) if rowmap is not None
                       else np.arange(row_offset, row_offset + n, dtype=np.uint64))
                g = (gid[:, None] * np.uint64(Kg // 4) + np.uint64(col_offset // 4)
                     + np.arange(K // 4, dtype=np.uint64)[None, :]).reshape(-1)
                self.add("mapped", seed, offset + s * step_mul, g, p, s)
                if s == self.check_step and self.phase == "train":
                    act = fn(y, scale, shift, relu, 0.0)
                    vis = _np(act != 0)
                    want = od.mask_mapped(gid, K, Kg, col_offset, p, seed, offset + s * step_mul)
                    self.checked.append(np.array_equal(_np(res != 0)[vis], want[vis]))
            return res
        return w

    def _sign_gather(self, fn):
        def w(feats, idx, p, seed, offset, out, step_dev=None, step_mul=0, **kw):
            s = self._s(step_dev)
            res = fn(feats, idx, p, seed, offset, out, step_dev=step_dev, step_mul=step_mul, **kw)
            if p > 0:
                H, B, F = out.shape
                for h in range(H):
                    self.add("sign_hop", seed, offset + s * step_mul + h, np.arange(B * F // 4, dtype=np.uint64), p, s)
                if s == self.check_step and self.phase == "train":
                    raw = torch.empty_like(out)
                    fn(feats, idx, 0.0, seed, offset, raw)
                    vis = _np(raw != 0)
                    want = od.sign_hops(H, B, F, p, seed, offset + s * step_mul)
                    self.checked.append(np.array_equal(_np(out != 0)[vis], want[vis]))
            return res
        return w

    def _label_inputs(self, fn):
        def w(X, col0, C, row_pos, labels, role, cnt_part, eval, use_labels, mask_rate=0.0, seed=0, offset=0, step_dev=None,
              step_mul=0, mask=None):
            s = self._s(step_dev)
            res = fn(X, col0, C, row_pos, labels, role, cnt_part, eval, use_labels, mask_rate, seed, offset, step_dev, step_mul,
                     mask)
            if not eval and mask is None and mask_rate > 0:
                n_train = int((row_pos >= 0).sum().item())
                self.add("label_mask", seed, offset + s * step_mul, np.arange((n_train + 3) // 4, dtype=np.uint64), mask_rate, s)
                if s == self.check_step and self.phase == "train":
                    self.checked.append(np.array_equal(_label_masked(role, row_pos, use_labels),
                                                       od.label_drop(n_train, mask_rate, seed, offset + s * step_mul)))
            return res
        return w

    def _random_walk(self, rowptr, col, start, walk_length, seed=0, offset=0):
        bpw = (walk_length + 3) // 4
        self.records.append(dict(kind="walk", seed=int(seed), off=int(offset), step=None, phase=self.phase,
                                 blocks=np.arange(start.numel() * bpw, dtype=np.uint64)))
        return self._walk_fn(rowptr, col, start, walk_length, seed, offset)

    def _gcrd_sample(self, n, seed, offset, step_ptr, perm, ws, stream):
        """The base offset only: the kernel adds the device step (the caller expands it)."""
        self.records.append(dict(kind="sample", seed=int(seed), off=int(offset), step=None, phase=self.phase,
                                 blocks=np.arange((n + 3) // 4, dtype=np.uint64)))
        return self._sample_fn(n, seed, offset, step_ptr, perm, ws, stream)

    # ---- checks
    def train_records(self):
        return [r for r in self.records if r["phase"] == "train"]

    def assert_disjoint(self, records=None):
        recs = self.train_records() if records is None else records
        clashes = od.disjoint([(r["seed"], r["off"], r["blocks"]) for r in recs])
        assert not clashes, [(recs[a]["kind"], recs[b]["kind"], o) for a, b, _, o in clashes[:5]]

    def assert_eval_draws_nothing(self):
        assert not [r for r in self.records if r["phase"] == "eval" and r["kind"] != "walk"]

    def offsets_of_step(self, s):
        return sorted(r["off"] for r in self.train_records() if r["step"] == s)

    def assert_checked(self):
        assert self.checked and all(self.checked), self.checked


def _gcn_problem(n=1200, e=8000, F=32, C=8, seed=0):
    ei = skewed_edges(n, e, seed)
    row, col, _ = og.to_sparse_adj_t(ei.numpy(), n)
    r, c = og.to_symmetric(row, col, n)
    adj = SparseTensor(row=torch.from_numpy(r).cuda(), col=torch.from_numpy(c).cuda(), sparse_sizes=(n, n), is_sorted=True)
    g = torch.Generator().manual_seed(seed + 9)
    x = torch.randn(n, F, generator=g).cuda()
    y = torch.randint(0, C, (n,), generator=g).cuda()
    t = (torch.randn(n, C, generator=g) * 2).cuda()
    idx = torch.randperm(n, generator=g)[: n // 2].sort().values.cuda()
    return adj, x, y, t, idx


@pytest.mark.parametrize("with_gcrd", [False, True], ids=["plain", "gcrd"])
@pytest.mark.parametrize("L", [2, 3])
@pytest.mark.parametrize("kind", ["gcn", "sage"])
def test_stream_audit_gcn_sage(monkeypatch, kind, L, with_gcrd):
    from efficient_gnns_b200.engine import GCNStudentTrainer
    from efficient_gnns_b200.engine_sage import SAGEStudentTrainer
    from efficient_gnns_b200.gcrd import GCRD
    adj, x, y, t, idx = _gcn_problem()
    dims = [32] + [64] * (L - 1) + [8]
    seed = 5
    head = GCRD(torch.randn(x.shape[0], 64, device="cuda"), idx, dims[-2], proj_dim=64, max_samples=256, seed=seed) \
        if with_gcrd else None
    tr = {"gcn": GCNStudentTrainer, "sage": SAGEStudentTrainer}[kind](adj, dims, dropout=0.5, lr=0.01, seed=seed, gcrd=head)
    rec = Recorder(monkeypatch)
    for _ in range(3):
        tr.train_step(x, y, idx, t)
    rec.phase = "eval"
    tr.forward(x, training=False)
    rec.assert_eval_draws_nothing()
    rec.assert_checked()
    for s in range(3):
        assert rec.offsets_of_step(s) == sorted(od.gcn_streams(L, s).values()), s
    samples = [r for r in rec.train_records() if r["kind"] == "sample"]
    if with_gcrd:
        assert len(samples) == 3 and all(r["off"] == od.SAMPLE_STREAM and r["seed"] == seed for r in samples)
        # the sampler adds the device step to SAMPLE_STREAM: its effective offsets stay far from the dropout streams
        expanded = [dict(r, off=od.gcrd_sample_stream(s)) for s, r in enumerate(samples)]
    else:
        assert not samples
        expanded = []
    rec.assert_disjoint([r for r in rec.train_records() if r["kind"] != "sample"] + expanded)


def _gat_graph():
    from pathlib import Path
    gold = torch.load(Path(__file__).resolve().parent / "golden" / "gat_model_arxiv.pt")
    n = gold["x"].shape[0]
    adj = SparseTensor(row=gold["row"].cuda(), col=gold["col"].cuda(), sparse_sizes=(n, n), is_sorted=True)
    return adj, gold, n


def test_stream_audit_gat(monkeypatch):
    from efficient_gnns_b200.engine_gat import GATTrainer
    adj, gold, n = _gat_graph()
    g = torch.Generator().manual_seed(2)
    x, y, idx = torch.randn(n, 32, generator=g).cuda(), gold["y"].cuda(), gold["train_idx"].cuda()
    L = 3
    tr = GATTrainer(adj, 32, 8, 10, L, 3, dropout=0.5, input_drop=0.1, edge_drop=0.25, lr=1e-2, seed=4)
    rec = Recorder(monkeypatch)
    for _ in range(3):
        tr.train_step(x, y, idx)
    rec.phase = "eval"
    tr.forward(x, training=False)
    rec.assert_disjoint()
    rec.assert_eval_draws_nothing()
    rec.assert_checked()
    for s in range(3):
        assert rec.offsets_of_step(s) == sorted(od.gat_streams(L, s).values()), s


@pytest.mark.parametrize("use_labels,iters", [(True, 0), (True, 1), (True, 2), (False, 0)])
def test_stream_audit_gat_teacher(monkeypatch, use_labels, iters):
    from pathlib import Path
    from efficient_gnns_b200.engine_gat_teacher import GATTeacherTrainer
    gold = torch.load(Path(__file__).resolve().parent / "golden" / "gat_teacher_arxiv.pt", weights_only=False)
    n = gold["x"].shape[0]
    adj = SparseTensor(row=gold["row"].long().cuda(), col=gold["col"].long().cuda(), sparse_sizes=(n, n), is_sorted=True)
    split = {"train": gold["train_idx"], "valid": gold["val_idx"], "test": gold["test_idx"]}
    L = gold["n_layers"]
    tr = GATTeacherTrainer(adj, gold["x"].cuda(), gold["y"].cuda(), split, n_classes=gold["n_classes"], use_labels=use_labels,
                           n_label_iters=iters, n_hidden=gold["n_hidden"], n_layers=L, n_heads=gold["n_heads"], dropout=0.75,
                           input_drop=0.25, edge_drop=0.3, seed=3)
    assert tr.step_mul == od.gat_teacher_step_streams(L, iters)
    rec = Recorder(monkeypatch)
    for _ in range(3):
        tr.train_step()
    rec.phase = "eval"
    tr.evaluate()
    rec.assert_disjoint()
    rec.assert_eval_draws_nothing()
    rec.assert_checked()
    for s in range(3):
        assert rec.offsets_of_step(s) == sorted(od.gat_teacher_streams(L, iters, s).values()), s
    assert sum(r["kind"] == "label_mask" for r in rec.train_records()) == 3


@pytest.mark.parametrize("ff", [1, 2, 3])
def test_stream_audit_sign(monkeypatch, ff):
    from efficient_gnns_b200.engine_sign import SIGNStudentTrainer
    g = torch.Generator().manual_seed(0)
    n, F, H, C = 600, 16, 3, 8
    feats = [torch.randn(n, F, generator=g).cuda() for _ in range(H)]
    y = torch.randint(0, C, (n,), generator=g).cuda()
    t = (torch.randn(n, C, generator=g) * 2).cuda()
    train_idx = torch.randperm(n, generator=g)[:300].cuda()
    tr = SIGNStudentTrainer(feats, C, hidden=32, ff_layer=ff, dropout=0.5, input_drop=0.1, batch_size=128, seed=2)
    assert tr.D == od.sign_step_streams(H, ff)
    rec = Recorder(monkeypatch)
    for s in range(3):
        tr.train_step(train_idx[s * 100:(s + 1) * 100 - s], y, t)          # ragged batches
    rec.phase = "eval"
    tr.predict()
    rec.assert_disjoint()
    rec.assert_eval_draws_nothing()
    rec.assert_checked()
    for s in range(3):
        assert rec.offsets_of_step(s) == sorted(od.sign_streams(H, ff, s).values()), s


@pytest.mark.parametrize("loader_seed", [1, 0], ids=["distinct-seeds", "same-seed"])
def test_stream_audit_rgcn_on_graphsaint(monkeypatch, loader_seed):
    """The R-GCN's own draws are disjoint.  The GraphSAINT walks draw at (loader seed, batch number) from block 0: with the
    loader's seed equal to the trainer's they share counters with the dropout streams, as DESIGN §4.3 documents."""
    from test_rgcn_train_gpu import small_mag, trainer
    data, x, rel = small_mag(0)
    L, seed = 2, 0
    tr = trainer(rel, L=L, p=0.5, seed=seed)
    rec = Recorder(monkeypatch)
    loader = sampling.GraphSAINTRandomWalkSampler(data, batch_size=150, walk_length=L, num_steps=3, seed=loader_seed)
    batches = list(loader)
    for b in batches:
        tr.train_step(b, x)
    rec.phase = "eval"
    tr.forward(batches[0], x, training=False)
    rec.assert_eval_draws_nothing()
    rec.assert_checked()
    own = [r for r in rec.train_records() if r["kind"] != "walk"]
    walks = [r for r in rec.train_records() if r["kind"] == "walk"]
    assert [r["off"] for r in walks] == [od.saint_walk_stream(0, 3, i) for i in range(3)]
    rec.assert_disjoint(own)
    for s in range(3):
        assert rec.offsets_of_step(s) == sorted(od.gcn_streams(L, s).values()), s
    clashes = od.disjoint([(r["seed"], r["off"], r["blocks"]) for r in own + walks])
    if loader_seed != seed:
        assert not clashes
    else:
        kinds = {(own + walks)[b]["kind"] for _, b, _, _ in clashes} | {(own + walks)[a]["kind"] for a, _, _, _ in clashes}
        assert clashes and kinds == {"mapped", "walk"}
