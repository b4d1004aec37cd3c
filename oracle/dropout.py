"""CPU restatement (numpy, test infrastructure only) of the dropout keep decisions and of the Philox stream layout of every
training engine.  Restated from the contract in efficient-gnns_b200/csrc/philox.cuh and DESIGN §4.3, not from the kernels.

A [rows, K] matrix is drawn in float4 units: flat float4 index g = row * (K / 4) + column / 4, component c = column % 4.

  * P16 path (p * 65536 an integer and p > 0, fp32 p): block g >> 1 of Philox4x32-10(seed, offset).  Even g reads words
    (x, y), odd g reads (z, w); each word gives two 16-bit uniforms, the low half first.  Keep iff u16 >= p * 65536.
  * 24-bit path (otherwise): block g, word c of it.  Keep iff (word >> 8) * 2^-24 >= p.

Every producer reduces to these two rules for a set of flat indices g at one effective offset
(offset + step * step_mul, read on the device by the step forms)."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from .sampling import philox4x32

U64 = 1 << 64
SAMPLE_STREAM = 1 << 62                     # the G-CRD / GSP row sampler's base offset (heads.py)


def f32(p: float) -> float:
    """p as the ABI passes it (an fp32 argument)."""
    return float(np.float32(p))


def p16_threshold(p: float) -> Optional[int]:
    """thr = p * 65536 if the 16-bit path applies to fp32 p, else None."""
    t = f32(p) * 65536.0
    return int(t) if f32(p) > 0.0 and t == int(t) else None


def sources(g: np.ndarray, p16: bool) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Which random bits decide component c of float4 g: (block [n], word [n, 4], half [n, 4]); half is -1 on the 24-bit
    path (the whole word)."""
    g = np.asarray(g, dtype=np.uint64)
    c = np.arange(4)
    if p16:
        odd = (g & np.uint64(1)).astype(np.int64)[:, None]
        return g >> np.uint64(1), 2 * odd + c[None, :] // 2, np.broadcast_to(c % 2, (len(g), 4)).copy()
    return g.copy(), np.broadcast_to(c, (len(g), 4)).copy(), np.full((len(g), 4), -1)


def keep_float4(g: np.ndarray, p: float, seed: int, offset: int, src=sources) -> np.ndarray:
    """bool [len(g), 4]: the keep decisions of float4s g at (seed, offset).  p = 0 keeps everything."""
    g = np.asarray(g, dtype=np.uint64)
    if f32(p) == 0.0:
        return np.ones((len(g), 4), dtype=bool)
    thr = p16_threshold(p)
    block, word, half = src(g, thr is not None)
    uniq, inv = np.unique(block, return_inverse=True)
    r = philox4x32(seed % U64, offset % U64, uniq)[inv.reshape(-1)]             # [n, 4] uint32
    w = np.take_along_axis(r, word, axis=1).astype(np.uint64)
    if thr is not None:
        u16 = np.where(half == 1, w >> np.uint64(16), w & np.uint64(0xFFFF))
        return u16 >= thr
    return (w >> np.uint64(8)).astype(np.float64) * 2.0 ** -24 >= f32(p)


def expected_keep_rate(p: float) -> float:
    """The exact probability of a keep: 1 - thr / 65536 on P16, 1 - ceil(p * 2^24) / 2^24 on the 24-bit path."""
    thr = p16_threshold(p)
    if thr is not None:
        return 1.0 - thr / 65536.0
    return 1.0 - np.ceil(f32(p) * 2.0 ** 24) / 2.0 ** 24


def audit_word_use(g: np.ndarray, p16: bool, src=sources) -> bool:
    """True iff over the float4s g every random unit (a 16-bit half on P16, a 32-bit word otherwise) of every block
    decides at most one element."""
    block, word, half = src(np.asarray(g, dtype=np.uint64), p16)
    key = np.stack([np.repeat(block, 4).astype(np.uint64), word.reshape(-1).astype(np.uint64),
                    (half.reshape(-1) + 1).astype(np.uint64)], axis=1)
    return len(np.unique(key, axis=0)) == len(key)


# ------------------------------------------------------------------------------------------------------ derived layouts
def mask(n_rows: int, K: int, p: float, seed: int, offset: int, row_offset: int = 0) -> np.ndarray:
    """bool [n_rows, K] of b200gnn_dropout_mask_u8 / affine_relu_dropout(row_offset) / dropout_mask_step (at its effective
    offset): rows row_offset … of a K-wide matrix."""
    nv = K // 4
    g = np.uint64(row_offset * nv) + np.arange(n_rows * nv, dtype=np.uint64)
    return keep_float4(g, p, seed, offset).reshape(n_rows, K)


def mask_mapped(gid: np.ndarray, K: int, K_global: int, col_offset: int, p: float, seed: int, offset: int) -> np.ndarray:
    """bool [len(gid), K] of affine_relu_dropout_mapped / _scatter: local row r is global row gid[r] of a K_global-wide
    matrix, local columns start at col_offset.  g = gid * (K_global / 4) + col_offset / 4 + cv."""
    gid = np.asarray(gid, dtype=np.uint64)
    g = (gid[:, None] * np.uint64(K_global // 4) + np.uint64(col_offset // 4)
         + np.arange(K // 4, dtype=np.uint64)[None, :]).reshape(-1)
    return keep_float4(g, p, seed, offset).reshape(len(gid), K)


def bits(n_layers: int, n_rows: int, K: int, p: float, seed: int, offset: int) -> np.ndarray:
    """uint32 [n_layers, n_rows, ceil(K / 32)] of b200gnn_dropout_bits_u32: layer l at offset + l, bit b of word w is
    column 32 w + b, zero past K."""
    words = (K + 31) // 32
    out = np.zeros((n_layers, n_rows, words), dtype=np.uint32)
    for l in range(n_layers):
        m = np.zeros((n_rows, 32 * words), dtype=np.uint64)
        m[:, :K] = mask(n_rows, K, p, seed, offset + l)
        out[l] = (m.reshape(n_rows, words, 32) << np.arange(32, dtype=np.uint64)).sum(axis=2).astype(np.uint32)
    return out


def sign_hops(n_hops: int, B: int, F: int, p: float, seed: int, offset: int) -> np.ndarray:
    """bool [n_hops, B, F] of b200gnn_sign_gather_f32's input dropout: hop h is the [B, F] mask at offset + h."""
    return np.stack([mask(B, F, p, seed, offset + h) for h in range(n_hops)])


def label_drop(n_train: int, p: float, seed: int, offset: int) -> np.ndarray:
    """bool [n_train] of label_inputs' drop_decision (rand < mask_rate): training position j is component j % 4 of float4
    j / 4, dropped where the mask does not keep it."""
    nv = (n_train + 3) // 4
    return ~keep_float4(np.arange(nv, dtype=np.uint64), p, seed, offset).reshape(-1)[:n_train]


def blocks_of(g: np.ndarray, p: float) -> np.ndarray:
    """The Philox blocks the float4s g read."""
    g = np.asarray(g, dtype=np.uint64)
    return np.unique(g >> np.uint64(1)) if p16_threshold(p) is not None else np.unique(g)


# ------------------------------------------------------------------------------------------------------ stream layouts
# Each function returns {stream name: effective Philox offset} of one training step.  A trainer's streams all use the
# trainer's seed; the layouts must give every (step, stream) its own offset.
def gcn_streams(L: int, step: int) -> Dict[str, int]:
    """GCN / GraphSAGE students and the R-GCN: hidden layer l at l + step * L."""
    return {f"dropout{l}": l + step * L for l in range(L - 1)}


def gcrd_sample_stream(step: int) -> int:
    """The G-CRD / GSP row sampler: SAMPLE_STREAM + step."""
    return SAMPLE_STREAM + step


def gat_streams(L: int, step: int, n_fwd: int = 1, step_streams: Optional[int] = None) -> Dict[str, int]:
    """GATTrainer: training forward f of step s draws hidden layer l at l, the input at L - 1 and edge layer l at L + l,
    each plus f * 2L + s * step_streams (default 2L)."""
    mul = 2 * L if step_streams is None else step_streams
    out = {}
    for f in range(n_fwd):
        b = f * 2 * L + step * mul
        out.update({f"f{f}.dropout{l}": b + l for l in range(L - 1)})
        out[f"f{f}.input"] = b + L - 1
        out.update({f"f{f}.edge{l}": b + L + l for l in range(L)})
    return out


def gat_teacher_step_streams(L: int, n_label_iters: int) -> int:
    """GATTeacherTrainer: (n_label_iters + 1) training forwards of 2L streams, then the label mask."""
    return (n_label_iters + 1) * 2 * L + 1


def gat_teacher_streams(L: int, n_label_iters: int, step: int) -> Dict[str, int]:
    n_fwd = n_label_iters + 1
    mul = gat_teacher_step_streams(L, n_label_iters)
    out = gat_streams(L, step, n_fwd, mul)
    out["label_mask"] = n_fwd * 2 * L + step * mul
    return out


def sign_step_streams(H: int, ff: int) -> int:
    """SIGNStudentTrainer: D = H + (H + 1)(ff - 1) + 1 offsets per step."""
    return H + (H + 1) * (ff - 1) + 1


def sign_streams(H: int, ff: int, step: int) -> Dict[str, int]:
    """hop h's input dropout at h, hidden layer j at H + j, the concatenation at H + (H + 1)(ff - 1); plus step * D."""
    D = sign_step_streams(H, ff)
    out = {f"hop{h}": h + step * D for h in range(H)}
    out.update({f"hidden{j}": H + j + step * D for j in range((H + 1) * (ff - 1))})
    out["cat"] = H + (H + 1) * (ff - 1) + step * D
    return out


def saint_walk_stream(epoch: int, num_steps: int, i: int) -> int:
    """GraphSAINTRandomWalkSampler: batch i of epoch e walks at (loader seed, e * num_steps + i)."""
    return epoch * num_steps + i


def disjoint(records: List[Tuple[int, int, np.ndarray]]) -> List[Tuple[int, int, int, int]]:
    """records: (seed, effective offset, Philox blocks).  Returns (record a, record b, seed, offset) for every pair of
    records that share a block at the same (seed, offset); empty when every draw has counters of its own."""
    groups: Dict[Tuple[int, int], List[int]] = {}
    for i, (s, o, _) in enumerate(records):
        groups.setdefault((s % U64, o % U64), []).append(i)
    clashes = []
    for (s, o), ids in groups.items():
        for a in range(len(ids)):
            for b in range(a + 1, len(ids)):
                if np.intersect1d(records[ids[a]][2], records[ids[b]][2]).size:
                    clashes.append((ids[a], ids[b], s, o))
    return clashes
