// Row-segmented CSR SpMM for sm_90a:  Y[i,:] = reduce_e val[e] * X[col[e],:]
//
// Replaces torch_sparse spmm_sum/spmm_mean as reached from the reference's
// GCNConv / SAGEConv / SparseTensor.matmul call sites (arxiv_pyg/gnn.py:47,52,
// 79,84; mag_pyg/gnn.py:162) and their backward (same kernel on the CSC view).
//
// Design (HBM/L2-bound gather, no tensor cores):
//   * one warp per CHUNK of consecutive destination rows holding ~chunk_nnz
//     non-zeros (plan built once per graph), so warps are load-balanced on
//     power-law graphs; within a row 32 (col,val) pairs are fetched with one
//     coalesced load and broadcast by warp shuffle; each neighbour's feature
//     row is gathered with 128-bit read-only loads, U*CH of them in flight per
//     lane (8 x 16 B) so a warp keeps 4 KB of gather traffic outstanding;
//   * narrow rows (K/4 < 32 vectors) fold several neighbours across the warp
//     ("groups") and combine with shuffles, so K=40 keeps 30/32 lanes busy;
//   * hub rows (degree > hub_threshold) are skipped here and split into
//     fixed-length segments, one CTA each, reduced in a fixed order by a
//     finalize kernel: no atomics anywhere, run-to-run deterministic;
//   * epilogue fuses mean division, bias, and per-CTA partial column
//     sum / sum-of-squares for the BatchNorm that follows the conv.
#include <cuda.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace b200gnn {

constexpr int SPMM_THREADS = 256;
constexpr int SPMM_WARPS = SPMM_THREADS / 32;
constexpr int SPMM_MAX_SLAB_FLOATS = 512;  // 32 lanes * CH(<=4) * W(<=4)

struct SpmmParams {
  const int32_t* rowptr;
  const int32_t* col;
  const float* val;
  const float* X;
  float* Y;
  const float* bias;
  float* stat_partial;
  const int32_t* chunk_rowptr;
  const int32_t* hub_rows;
  const int32_t* hub_segptr;
  float* hub_ws;
  int64_t ldx, ldy;  // in floats
  int32_t n_rows, K, nvec;
  int32_t hub_threshold, seg_len, n_hub, n_seg, n_chunks;
  int32_t mean, stream_store, main_grid;
  int32_t n_slabs, l2_hint;   // bulk kernel: column slabs (slab-major grid), evict_last policy on the gathers
  // Fused C->R layout exchange of the multi-GPU engine (hybrid.py): output row i of this [n_rows, K] product belongs to the
  // rank q with yoff[q] <= i < yoff[q+1] and is stored to Yp[q] + (i - yoff[q]) * ldyp + ycol (float index): the aggregation's
  // epilogue writes straight into the consumers' R-layout buffers (peer mappings).  n_yp = 0: off (plain Y / ldy).
  float* Yp[16];
  int32_t yoff[17];
  int32_t n_yp, ycol;
  int64_t ldyp;
};

// address of output row `row` (float4 units) for the kernels that support the fused C->R scatter
__device__ __forceinline__ float4* y_row_v4(const SpmmParams& p, int row) {
  if (p.n_yp == 0) return reinterpret_cast<float4*>(p.Y) + (size_t)row * (size_t)(p.ldy / 4);
  int q = 0;
#pragma unroll 1
  while (q + 1 < p.n_yp && row >= p.yoff[q + 1]) ++q;
  return reinterpret_cast<float4*>(p.Yp[q] + (size_t)(row - p.yoff[q]) * (size_t)p.ldyp + p.ycol);
}

struct LaneMap {
  int lpr, groups, g, l;
  bool active;
};

__device__ __forceinline__ LaneMap make_lane_map(int nvec, int lane) {
  LaneMap m;
  if (nvec >= 32) {
    m.lpr = 32; m.groups = 1; m.g = 0; m.l = lane; m.active = true;
  } else {
    m.lpr = nvec; m.groups = 32 / nvec; m.g = lane / nvec; m.l = lane - m.g * nvec;
    m.active = m.g < m.groups;
  }
  return m;
}

// Accumulate edges [beg,end) of one row into per-lane partials for one column slab.
template <typename V, int CH, bool HAS_VAL>
__device__ __forceinline__ void walk_edges(const int32_t* __restrict__ col, const float* __restrict__ val,
                                           const V* __restrict__ Xv, size_t ldxv, int beg, int end,
                                           int lane, const LaneMap& m, int slab_voff, int nvec, V (&acc)[CH]) {
  constexpr int U = 8 / CH;
  bool cvalid[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) cvalid[j] = m.active && (slab_voff + m.l + 32 * j < nvec);

  for (int base = beg; base < end; base += 32) {
    const int e = base + lane;
    int c = 0;
    float v = HAS_VAL ? 0.f : 1.f;
    if (e < end) {
      c = __ldg(col + e);
      if (HAS_VAL) v = __ldg(val + e);
    }
    const int cnt = min(32, end - base);
    for (int t = 0; t < cnt; t += m.groups * U) {
      V xv[U][CH];
      float vv[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int idx = t + u * m.groups + m.g;
        const int cc = __shfl_sync(FULL_MASK, c, idx & 31);
        const float w = __shfl_sync(FULL_MASK, v, idx & 31);
        const bool ok = idx < cnt;
        vv[u] = ok ? w : 0.f;
        const V* p = Xv + (size_t)cc * ldxv + slab_voff + m.l;
#pragma unroll
        for (int j = 0; j < CH; ++j) {
          if (ok && cvalid[j]) xv[u][j] = vldg(p + 32 * j);
          else vzero(xv[u][j]);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < CH; ++j) vfma(acc[j], vv[u], xv[u][j]);
    }
  }
}

template <typename V>
__device__ __forceinline__ void group_reduce(V& a, const LaneMap& m) {
  for (int gg = 1; gg < m.groups; ++gg) {
    V o = vshfl_down(a, gg * m.lpr);
    if (m.g == 0) vadd(a, o);
  }
}

template <typename V>
__device__ __forceinline__ V load_bias(const float* bias, int voff);
template <> __device__ __forceinline__ float load_bias<float>(const float* b, int voff) { return __ldg(b + voff); }
template <> __device__ __forceinline__ float2 load_bias<float2>(const float* b, int voff) {
  return make_float2(__ldg(b + 2 * voff), __ldg(b + 2 * voff + 1));
}
template <> __device__ __forceinline__ float4 load_bias<float4>(const float* b, int voff) {
  return make_float4(__ldg(b + 4 * voff), __ldg(b + 4 * voff + 1), __ldg(b + 4 * voff + 2), __ldg(b + 4 * voff + 3));
}

__device__ __forceinline__ void smem_accum(float* s, float* q, int voff, const float& a, const float& b) {
  s[voff] += a; q[voff] += b;
}
__device__ __forceinline__ void smem_accum(float* s, float* q, int voff, const float2& a, const float2& b) {
  s[2 * voff] += a.x; s[2 * voff + 1] += a.y; q[2 * voff] += b.x; q[2 * voff + 1] += b.y;
}
__device__ __forceinline__ void smem_accum(float* s, float* q, int voff, const float4& a, const float4& b) {
  s[4 * voff] += a.x; s[4 * voff + 1] += a.y; s[4 * voff + 2] += a.z; s[4 * voff + 3] += a.w;
  q[4 * voff] += b.x; q[4 * voff + 1] += b.y; q[4 * voff + 2] += b.z; q[4 * voff + 3] += b.w;
}
__device__ __forceinline__ void smem_add1(float* s, int voff, const float& a) { s[voff] += a; }
__device__ __forceinline__ void smem_add1(float* s, int voff, const float2& a) { s[2 * voff] += a.x; s[2 * voff + 1] += a.y; }
__device__ __forceinline__ void smem_add1(float* s, int voff, const float4& a) {
  s[4 * voff] += a.x; s[4 * voff + 1] += a.y; s[4 * voff + 2] += a.z; s[4 * voff + 3] += a.w;
}

// ---------------------------------------------------------------- main kernel
template <typename V, int CH, bool HAS_VAL, bool STATS>
__device__ __forceinline__ void spmm_chunk_cta(const SpmmParams& p, const int cta, float* s_stat) {
  constexpr int W = VecTraits<V>::W;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const LaneMap m = make_lane_map(p.nvec, lane);
  const int slab_vecs = 32 * CH;
  const int nslab = (p.nvec <= 32) ? 1 : (p.nvec + slab_vecs - 1) / slab_vecs;
  const V* Xv = reinterpret_cast<const V*>(p.X);
  V* Yv = reinterpret_cast<V*>(p.Y);
  const size_t ldxv = (size_t)(p.ldx / W), ldyv = (size_t)(p.ldy / W);
  constexpr bool do_stats = STATS;  // host guarantees nslab == 1 when set

  V ssum[CH], ssq[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) { vzero(ssum[j]); vzero(ssq[j]); }

  // one warp per chunk: a run of consecutive rows holding ~chunk_nnz non-zeros (plan from csr_chunk_plan),
  // so every warp has about the same amount of gather work whatever the degree distribution.
  const int chunk = cta * SPMM_WARPS + warp;
  const int row_lo = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk) : 0;
  const int row_hi = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk + 1) : 0;
  int end = row_lo < row_hi ? __ldg(p.rowptr + row_lo) : 0;
  for (int row = row_lo; row < row_hi; ++row) {
    const int beg = end;
    end = __ldg(p.rowptr + row + 1);
    const int deg = end - beg;
    if (deg > p.hub_threshold) continue;  // split path owns this row (incl. its statistics)
    for (int slab = 0; slab < nslab; ++slab) {
      const int slab_voff = slab * slab_vecs;
      V acc[CH];
#pragma unroll
      for (int j = 0; j < CH; ++j) vzero(acc[j]);
      walk_edges<V, CH, HAS_VAL>(p.col, p.val, Xv, ldxv, beg, end, lane, m, slab_voff, p.nvec, acc);
      if (m.groups > 1) group_reduce(acc[0], m);
      if (m.g == 0 && m.active) {
#pragma unroll
        for (int j = 0; j < CH; ++j) {
          const int voff = slab_voff + m.l + 32 * j;
          if (voff < p.nvec) {
            V y = acc[j];
            if (p.mean) vdiv(y, (float)max(deg, 1));
            if (p.bias) vadd(y, load_bias<V>(p.bias, voff));
            V* dst = Yv + (size_t)row * ldyv + voff;
            if (p.stream_store) vstcs(dst, y); else *dst = y;
            if (do_stats) vstat(ssum[j], ssq[j], y);
          }
        }
      }
    }
  }

  if (do_stats) {
    float* ss = s_stat;
    float* sq = s_stat + p.K;
    for (int i = threadIdx.x; i < 2 * p.K; i += SPMM_THREADS) s_stat[i] = 0.f;
    __syncthreads();
    for (int w = 0; w < SPMM_WARPS; ++w) {  // fixed order => deterministic
      if (warp == w && m.g == 0 && m.active) {
#pragma unroll
        for (int j = 0; j < CH; ++j) {
          const int voff = m.l + 32 * j;
          if (voff < p.nvec) smem_accum(ss, sq, voff, ssum[j], ssq[j]);
        }
      }
      __syncthreads();
    }
    float* out = p.stat_partial + (size_t)cta * 2 * p.K;
    for (int i = threadIdx.x; i < 2 * p.K; i += SPMM_THREADS) out[i] = s_stat[i];
  }
}

// ------------------------------------------------------- hub segment kernel
// One CTA per segment of a hub row: 8 warps take contiguous sub-ranges, then
// combine in warp order through shared memory; raw (un-normalised) partials go
// to the workspace.
template <typename V, int CH, bool HAS_VAL>
__device__ __forceinline__ void spmm_hub_seg_cta(const SpmmParams& p, const int seg, float* s_buf, const int slab_lo = 0,
                                                 const int slab_hi = 1 << 30) {
  constexpr int W = VecTraits<V>::W;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const LaneMap m = make_lane_map(p.nvec, lane);
  const int slab_vecs = 32 * CH;
  const int nslab = (p.nvec <= 32) ? 1 : (p.nvec + slab_vecs - 1) / slab_vecs;
  const V* Xv = reinterpret_cast<const V*>(p.X);
  const size_t ldxv = (size_t)(p.ldx / W);

  int lo = 0, hi = p.n_hub;  // largest h with hub_segptr[h] <= seg
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(p.hub_segptr + mid) <= seg) lo = mid; else hi = mid;
  }
  const int h = lo;
  const int row = __ldg(p.hub_rows + h);
  const int s = seg - __ldg(p.hub_segptr + h);
  const int rbeg = __ldg(p.rowptr + row), rend = __ldg(p.rowptr + row + 1);
  const int sbeg = rbeg + s * p.seg_len;
  const int send = min(rend, sbeg + p.seg_len);
  int per = (send - sbeg + SPMM_WARPS - 1) / SPMM_WARPS;
  per = (per + 31) / 32 * 32;
  const int wbeg = min(send, sbeg + warp * per);
  const int wend = min(send, wbeg + per);

  float* ws = p.hub_ws + (size_t)seg * p.K;
  for (int slab = slab_lo; slab < min(nslab, slab_hi); ++slab) {
    const int slab_voff = slab * slab_vecs;
    V acc[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) vzero(acc[j]);
    walk_edges<V, CH, HAS_VAL>(p.col, p.val, Xv, ldxv, wbeg, wend, lane, m, slab_voff, p.nvec, acc);
    if (m.groups > 1) group_reduce(acc[0], m);

    for (int i = threadIdx.x; i < SPMM_MAX_SLAB_FLOATS; i += SPMM_THREADS) s_buf[i] = 0.f;
    __syncthreads();
    for (int w = 0; w < SPMM_WARPS; ++w) {
      if (warp == w && m.g == 0 && m.active) {
#pragma unroll
        for (int j = 0; j < CH; ++j) {
          const int voff = slab_voff + m.l + 32 * j;
          if (voff < p.nvec) smem_add1(s_buf, m.l + 32 * j, acc[j]);
        }
      }
      __syncthreads();
    }
    const int slab_f0 = slab_voff * W;
    const int slab_fn = min(slab_vecs * W, p.K - slab_f0);
    for (int i = threadIdx.x; i < slab_fn; i += SPMM_THREADS) ws[slab_f0 + i] = s_buf[i];
    __syncthreads();
  }
}

// One launch: the first n_seg CTAs take the hub segments (the longest work items start first), the rest take
// chunks of ordinary rows.
template <typename V, int CH, bool HAS_VAL, bool STATS>
__global__ void __launch_bounds__(SPMM_THREADS, 3) spmm_rows_kernel(const SpmmParams p) {
  __shared__ float s_mem[2 * SPMM_MAX_SLAB_FLOATS];
  if ((int)blockIdx.x < p.n_seg) spmm_hub_seg_cta<V, CH, HAS_VAL>(p, (int)blockIdx.x, s_mem);
  else spmm_chunk_cta<V, CH, HAS_VAL, STATS>(p, (int)blockIdx.x - p.n_seg, s_mem);
}


// ------------------------------------------------------------------ pipelined chunk kernel (K = 128*CH floats)
// Same chunk/row ownership as spmm_chunk_cta, but the neighbour rows of a whole run of consecutive rows are
// streamed through a per-warp shared-memory ring with cp.async (LDGSTS.128, L1 bypass): each lane copies the
// 16-byte slices it will later consume itself, so no cross-lane synchronisation is needed, the copies cost no
// registers, and the pipeline keeps PIPE_BYTES of gather traffic per warp in flight ACROSS row boundaries
// (the register-staged loop drains at every row end, which is what limits it on graphs of mean degree ~15).
constexpr int PIPE_BYTES = 8192;                 // ring bytes per warp
constexpr int PIPE_SMEM = SPMM_WARPS * PIPE_BYTES;

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int CH, bool HAS_VAL, bool STATS>
__device__ __forceinline__ void spmm_chunk_cta_pipe(const SpmmParams& p, const int cta, float* s_stat, float4* ring_all) {
  constexpr int D = PIPE_BYTES / (CH * 512);     // ring depth in neighbour rows (CH=2 -> 8, CH=1 -> 16)
  constexpr int G = D >= 8 ? 4 : 2, NG = D / G;   // cp.async group = G edges; NG groups in flight
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4* ring = ring_all + (size_t)warp * (PIPE_BYTES / 16);   // slot s: ring[s*CH*32 + j*32 + lane]
  const float4* Xv = reinterpret_cast<const float4*>(p.X);
  float4* Yv = reinterpret_cast<float4*>(p.Y);
  const size_t ldxv = (size_t)(p.ldx / 4), ldyv = (size_t)(p.ldy / 4);

  float4 ssum[CH], ssq[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) { vzero(ssum[j]); vzero(ssq[j]); }

  const int chunk = cta * SPMM_WARPS + warp;
  const int row_lo = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk) : 0;
  const int row_hi = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk + 1) : 0;

  auto flush = [&](int row, int deg, float4 (&acc)[CH]) {
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      const int voff = lane + 32 * j;
      float4 y = acc[j];
      if (p.mean) vdiv(y, (float)max(deg, 1));
      if (p.bias) vadd(y, load_bias<float4>(p.bias, voff));
      float4* dst = Yv + (size_t)row * ldyv + voff;
      if (p.stream_store) vstcs(dst, y); else *dst = y;
      if (STATS) vstat(ssum[j], ssq[j], y);
      vzero(acc[j]);
    }
  };

  int r = row_lo;
  while (r < row_hi) {
    // ---- a run [r, run_end) of consecutive non-hub rows; hub rows belong to the split path
    int e_lo = __ldg(p.rowptr + r);
    {
      const int e_next = __ldg(p.rowptr + r + 1);
      if (e_next - e_lo > p.hub_threshold) { ++r; continue; }
    }
    int run_end = r + 1, e_hi = __ldg(p.rowptr + r + 1);
    while (run_end < row_hi) {
      const int nx = __ldg(p.rowptr + run_end + 1);
      if (nx - e_hi > p.hub_threshold) break;
      e_hi = nx; ++run_end;
    }
    const int n = e_hi - e_lo;

    // row ends of the run, 32 at a time in registers
    int rbase = r;
    int rp = (rbase + lane < run_end) ? __ldg(p.rowptr + rbase + lane + 1) : e_hi;
    auto row_end_of = [&](int row) {
      if (row - rbase >= 32) {            // warp-uniform
        rbase = row;
        rp = (rbase + lane < run_end) ? __ldg(p.rowptr + rbase + lane + 1) : e_hi;
      }
      return __shfl_sync(FULL_MASK, rp, row - rbase);
    };

    float4 acc[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) vzero(acc[j]);
    int row_beg = e_lo;                    // first edge of row r
    int rend = row_end_of(r);
    while (r < run_end && rend == row_beg) {   // leading empty rows
      flush(r, 0, acc);
      ++r;
      if (r < run_end) rend = row_end_of(r);
    }
    if (n == 0) continue;

    // Two cursors over the run's edges, each with a 32-edge register window: the issue side reads `col` (cI), the consume
    // side reads `val` (vA); both advance in groups of G edges, so window reloads and ring slots are decided per group and
    // the slot index is a compile-time constant inside the unrolled body.  One cp.async group per G edges, NG groups
    // (= D neighbour rows) in flight per warp.
    int cI = 0;
    float vA = 1.f;
    auto issue_group = [&](int jg, int slot0) {      // edges jg..jg+G-1 (relative to e_lo) -> slots slot0..slot0+G-1
      if ((jg & 31) == 0) { const int e = e_lo + jg + lane; cI = e < e_hi ? __ldg(p.col + e) : 0; }
#pragma unroll
      for (int u = 0; u < G; ++u) {
        if (jg + u < n) {                            // warp-uniform
          const int cc = __shfl_sync(FULL_MASK, cI, (jg + u) & 31);
          const float4* src = Xv + (size_t)cc * ldxv + lane;
          float4* dst = ring + (slot0 + u) * (CH * 32) + lane;
#pragma unroll
          for (int jj = 0; jj < CH; ++jj) cp_async16(dst + 32 * jj, src + 32 * jj);
        }
      }
      cp_async_commit();                             // always commit: keeps the group count uniform
    };
    auto boundary = [&]() {                          // the current row is complete: store it (+ empty rows that follow)
      do {
        flush(r, rend - row_beg, acc);
        row_beg = rend;
        ++r;
        if (r < run_end) rend = row_end_of(r);
      } while (r < run_end && rend == row_beg);
    };
    auto consume_group = [&](int j0, int slot0) {    // j0 < n
      if (HAS_VAL && (j0 & 31) == 0) { const int e = e_lo + j0 + lane; vA = e < e_hi ? __ldg(p.val + e) : 0.f; }
      const float4* sbase = ring + slot0 * (CH * 32) + lane;
      const int cnt = min(G, n - j0);
      int done = 0;
      while (done < cnt) {                           // pieces of the group that lie in one row (all warp-uniform)
        const int room = rend - (e_lo + j0 + done);  // >= 1: edges left in the current row
        const int take = min(cnt - done, room);
        if (take == G) {                             // common case: the whole group inside one row
#pragma unroll
          for (int u = 0; u < G; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
#pragma unroll
            for (int jj = 0; jj < CH; ++jj) vfma(acc[jj], w, sbase[u * (CH * 32) + 32 * jj]);
          }
        } else {
#pragma unroll 1
          for (int u = done; u < done + take; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
#pragma unroll
            for (int jj = 0; jj < CH; ++jj) vfma(acc[jj], w, sbase[u * (CH * 32) + 32 * jj]);
          }
        }
        done += take;
        if (take == room) boundary();
      }
    };
#pragma unroll
    for (int g = 0; g < NG; ++g) issue_group(g * G, g * G);
#pragma unroll 1
    for (int j = 0, s0 = 0; j < n; j += G, s0 = (s0 + G) & (D - 1)) {
      cp_async_wait<NG - 1>();                       // the oldest group (edges j ..) has landed; groups retire in order
      consume_group(j, s0);
      issue_group(j + D, s0);                        // refill the slots just consumed (their loads fed the FMAs above)
    }
    cp_async_wait<0>();
  }

  if (STATS) {
    float* ss = s_stat;
    float* sq = s_stat + p.K;
    for (int i = threadIdx.x; i < 2 * p.K; i += SPMM_THREADS) s_stat[i] = 0.f;
    __syncthreads();
    for (int w = 0; w < SPMM_WARPS; ++w) {
      if (warp == w) {
#pragma unroll
        for (int j = 0; j < CH; ++j) smem_accum(ss, sq, lane + 32 * j, ssum[j], ssq[j]);
      }
      __syncthreads();
    }
    float* out = p.stat_partial + (size_t)cta * 2 * p.K;
    for (int i = threadIdx.x; i < 2 * p.K; i += SPMM_THREADS) out[i] = s_stat[i];
  }
}

template <int CH, bool HAS_VAL, bool STATS>
__global__ void __launch_bounds__(SPMM_THREADS, 3) spmm_rows_pipe_kernel(const SpmmParams p) {
  __shared__ float s_mem[2 * SPMM_MAX_SLAB_FLOATS];
  extern __shared__ float4 s_ring[];
  if ((int)blockIdx.x < p.n_seg) spmm_hub_seg_cta<float4, CH, HAS_VAL>(p, (int)blockIdx.x, s_mem);
  else spmm_chunk_cta_pipe<CH, HAS_VAL, STATS>(p, (int)blockIdx.x - p.n_seg, s_mem, s_ring);
}


// ------------------------------------------------------------------ bulk-copy (TMA) chunk kernel, column-slab tiled
// TMA bulk-copy data path for wide rows (K a multiple of 128 floats).  Same chunk / run / row-boundary ownership as the
// cp.async kernel above, but every neighbour row (slab) is ONE cp.async.bulk (SASS UBLKCP) of 512*CH bytes issued by the
// lane that holds its column index, completing on an mbarrier per group of G ring slots: no per-lane copy instructions,
// no address arithmetic on 32 lanes, and the ring keeps BULK_RING bytes per warp in flight across row boundaries.
// K is tiled into column slabs of 128*CH floats and the grid is slab-major (all chunks of slab 0, then slab 1, ...), so
// the [N, slab] operand the resident CTAs gather from is 1/n_slabs of X, which keeps more of it L2-resident (ARXIV-shape
// K=256: 87 MB per 128-float slab instead of 173 MB, against a 50 MB L2); (col,val) are re-read per slab (8 B per edge).
constexpr int BULK_RING = 8192;                  // ring bytes per warp
constexpr int BULK_MAX_GROUPS = 8;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_g2s_hint(void* dst, const void* src, uint32_t bytes, uint64_t* bar, uint64_t pol) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::
                   "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)), "l"(pol)
               : "memory");
}

template <int CH, int G, bool HAS_VAL, bool STATS>
__device__ __forceinline__ void spmm_chunk_cta_bulk(const SpmmParams& p, const int cta, const int slab, float* s_stat,
                                                    float4* ring_all, uint64_t* bars_all) {
  constexpr int SLOT_V = CH * 32;                 // float4 per ring slot (one neighbour row of the slab)
  constexpr int SLOT_B = SLOT_V * 16;
  constexpr int D = BULK_RING / SLOT_B;           // ring depth in neighbour rows
  constexpr int NG = D / G;                       // barrier groups in flight
  static_assert(NG >= 2 && NG <= BULK_MAX_GROUPS && (32 % G) == 0 && D <= 32, "ring geometry");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4* ring = ring_all + (size_t)warp * (BULK_RING / 16);
  uint64_t* bars = bars_all + warp * BULK_MAX_GROUPS;
  if (lane < NG) mbar_init(bars + lane, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  uint64_t pol = 0;
  if (p.l2_hint) asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));

  const int slab_voff = slab * SLOT_V;
  const float4* Xv = reinterpret_cast<const float4*>(p.X) + slab_voff;
  float4* Yv = reinterpret_cast<float4*>(p.Y) + slab_voff;
  const size_t ldxv = (size_t)(p.ldx / 4), ldyv = (size_t)(p.ldy / 4);

  float4 ssum[CH], ssq[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) { vzero(ssum[j]); vzero(ssq[j]); }
  float4 bias4[CH];
#pragma unroll
  for (int j = 0; j < CH; ++j) {
    vzero(bias4[j]);
    if (p.bias) bias4[j] = load_bias<float4>(p.bias, slab_voff + lane + 32 * j);
  }

  const int chunk = cta * SPMM_WARPS + warp;
  const int row_lo = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk) : 0;
  const int row_hi = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk + 1) : 0;

  auto flush = [&](int row, int deg, float4 (&acc)[CH]) {
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      float4 y = acc[j];
      if (p.mean) vdiv(y, (float)max(deg, 1));
      vadd(y, bias4[j]);
      float4* dst = (p.n_yp ? y_row_v4(p, row) + slab_voff : Yv + (size_t)row * ldyv) + lane + 32 * j;
      if (p.stream_store) vstcs(dst, y); else *dst = y;
      if (STATS) vstat(ssum[j], ssq[j], y);
      vzero(acc[j]);
    }
  };

  uint32_t phases = 0;                           // bit b = parity the next wait on barrier b expects
  int r = row_lo;
  while (r < row_hi) {
    // ---- a run [r, run_end) of consecutive non-hub rows; hub rows belong to the split path
    int e_lo = __ldg(p.rowptr + r);
    {
      const int e_next = __ldg(p.rowptr + r + 1);
      if (e_next - e_lo > p.hub_threshold) { ++r; continue; }
    }
    int run_end = r + 1, e_hi = __ldg(p.rowptr + r + 1);
    while (run_end < row_hi) {
      const int nx = __ldg(p.rowptr + run_end + 1);
      if (nx - e_hi > p.hub_threshold) break;
      e_hi = nx; ++run_end;
    }
    const int n = e_hi - e_lo;

    int rbase = r;                                // row ends of the run, 32 at a time in registers
    int rp = (rbase + lane < run_end) ? __ldg(p.rowptr + rbase + lane + 1) : e_hi;
    auto row_end_of = [&](int row) {
      if (row - rbase >= 32) {                    // warp-uniform
        rbase = row;
        rp = (rbase + lane < run_end) ? __ldg(p.rowptr + rbase + lane + 1) : e_hi;
      }
      return __shfl_sync(FULL_MASK, rp, row - rbase);
    };

    float4 acc[CH];
#pragma unroll
    for (int j = 0; j < CH; ++j) vzero(acc[j]);
    int row_beg = e_lo;
    int rend = row_end_of(r);
    while (r < run_end && rend == row_beg) {      // leading empty rows
      flush(r, 0, acc);
      ++r;
      if (r < run_end) rend = row_end_of(r);
    }
    if (n == 0) continue;

    // Issue side: a 32-edge register window of column indices (cI); the lane that holds edge j's column issues its copy.
    int cI = 0;
    float vA = 1.f;
    auto issue_group = [&](int jg, int slot0, int b) {    // edges jg..jg+G-1 (relative to e_lo) -> slots slot0.., barrier b
      if (jg >= n) return;                                 // warp-uniform
      if ((jg & 31) == 0) { const int e = e_lo + jg + lane; cI = e < e_hi ? __ldg(p.col + e) : 0; }
      const int cnt = min(G, n - jg);
      const int u = lane - (jg & 31);
      if (lane == 0) mbar_expect_tx(bars + b, (uint32_t)(cnt * SLOT_B));
      if (u >= 0 && u < cnt) {
        const float4* src = Xv + (size_t)cI * ldxv;
        float4* dst = ring + (slot0 + u) * SLOT_V;
        if (p.l2_hint) bulk_g2s_hint(dst, src, SLOT_B, bars + b, pol);
        else bulk_g2s(dst, src, SLOT_B, bars + b);
      }
    };
    auto boundary = [&]() {                          // the current row is complete: store it (+ empty rows that follow)
      do {
        flush(r, rend - row_beg, acc);
        row_beg = rend;
        ++r;
        if (r < run_end) rend = row_end_of(r);
      } while (r < run_end && rend == row_beg);
    };
    auto consume_group = [&](int j0, int slot0) {    // j0 < n
      if (HAS_VAL && (j0 & 31) == 0) { const int e = e_lo + j0 + lane; vA = e < e_hi ? __ldg(p.val + e) : 0.f; }
      const float4* sbase = ring + slot0 * SLOT_V + lane;
      const int cnt = min(G, n - j0);
      int done = 0;
      while (done < cnt) {                           // pieces of the group that lie in one row (all warp-uniform)
        const int room = rend - (e_lo + j0 + done);  // >= 1: edges left in the current row
        const int take = min(cnt - done, room);
        if (take == G) {                             // common case: the whole group inside one row
#pragma unroll
          for (int u = 0; u < G; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
#pragma unroll
            for (int jj = 0; jj < CH; ++jj) vfma(acc[jj], w, sbase[u * SLOT_V + 32 * jj]);
          }
        } else {
#pragma unroll 1
          for (int u = done; u < done + take; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
#pragma unroll
            for (int jj = 0; jj < CH; ++jj) vfma(acc[jj], w, sbase[u * SLOT_V + 32 * jj]);
          }
        }
        done += take;
        if (take == room) boundary();
      }
    };
#pragma unroll
    for (int g = 0; g < NG; ++g) issue_group(g * G, g * G, g);
    int b = 0;
#pragma unroll 1
    for (int j = 0, s0 = 0; j < n; j += G) {
      mbar_wait(bars + b, (phases >> b) & 1u);     // this group's rows have landed (complete_tx of all its copies)
      phases ^= 1u << b;
      consume_group(j, s0);
      __syncwarp();                                // every lane has read the slots before they are refilled
      issue_group(j + D, s0, b);
      s0 = (s0 + G) & (D - 1);
      b = (b + 1 == NG) ? 0 : b + 1;
    }
  }

  if (STATS) {
    constexpr int SW = SLOT_V * 4;                 // slab width in floats
    float* ss = s_stat;
    float* sq = s_stat + SW;
    for (int i = threadIdx.x; i < 2 * SW; i += SPMM_THREADS) s_stat[i] = 0.f;
    __syncthreads();
    for (int w = 0; w < SPMM_WARPS; ++w) {          // fixed order => deterministic
      if (warp == w) {
#pragma unroll
        for (int j = 0; j < CH; ++j) smem_accum(ss, sq, lane + 32 * j, ssum[j], ssq[j]);
      }
      __syncthreads();
    }
    float* out = p.stat_partial + (size_t)cta * 2 * p.K + slab * SW;
    for (int i = threadIdx.x; i < SW; i += SPMM_THREADS) { out[i] = ss[i]; out[p.K + i] = sq[i]; }
  }
}

constexpr int BULK_SMEM = SPMM_WARPS * BULK_RING + SPMM_WARPS * BULK_MAX_GROUPS * 8;

template <int CH, int G, bool HAS_VAL, bool STATS>
__global__ void __launch_bounds__(SPMM_THREADS, 3) spmm_rows_bulk_kernel(const SpmmParams p) {
  __shared__ float s_mem[2 * SPMM_MAX_SLAB_FLOATS];
  extern __shared__ __align__(128) unsigned char s_dyn[];
  const int per_slab = p.main_grid + p.n_seg;
  const int slab = (int)blockIdx.x / per_slab;
  const int b = (int)blockIdx.x - slab * per_slab;
  if (b < p.n_seg) spmm_hub_seg_cta<float4, CH, HAS_VAL>(p, b, s_mem, slab, slab + 1);
  else spmm_chunk_cta_bulk<CH, G, HAS_VAL, STATS>(p, b - p.n_seg, slab, s_mem, reinterpret_cast<float4*>(s_dyn),
                                                  reinterpret_cast<uint64_t*>(s_dyn + SPMM_WARPS * BULK_RING));
}


// ------------------------------------------------------------------ lane-copy column-slab kernel (K = 128 or 256, X beyond L2)
// When X is larger than L2, the bulk kernel's 128- or 256-float slabs (87 / 173 MB at ARXIV shape) still come mostly from
// DRAM.  This kernel tiles K into narrow slabs of SW floats (SLAB_SW = 64), so the [N, SW] operand of one slab (43 MB at
// N = 169,343) mostly stays in L2 while the resident CTAs gather from it; DRAM then carries X about once, Y once and
// (col, val) once per slab.  A narrow row is too small for one bulk copy each (the copy engine retires a roughly fixed
// number of copies per second), so the lanes issue the copies: every lane copies 16-byte slices with cp.async.cg into a
// per-warp ring, E = 32·4 / SW neighbour rows per warp instruction, SLAB_G rows per commit group, the ring keeping about
// 6 KB per warp in flight across row boundaries.  A slice is consumed by another lane than the one that copied it, so
// cp.async.wait_group is followed by __syncwarp() before the reads, and the reads by __syncwarp() before the refill.
// The slab gathers carry an evict_last L2 policy; (col, val) are loaded evict_first and Y is stored st.global.cs (when
// stream_store), so the index and output streams do not push the slab out of L2.
// Arithmetic: lane l owns floats [l·SW/32, (l+1)·SW/32) of the slab and forms acc = fmaf(w_e, x_e, acc) from zero in CSR
// edge order, then the bulk kernel's epilogue (/ max(deg, 1), + bias, store, statistics) and its warp-ordered statistics
// combine: every Y element and statistics slot equals spmm_rows_bulk_kernel's bit for bit.  Hub rows take
// spmm_hub_seg_cta over the full width in the CTAs that lead the grid, whose per-element order is the bulk path's too.
constexpr int SLAB_RING = 8192;                  // ring bytes per warp
constexpr int SLAB_G = 8;                        // neighbour rows per cp.async group
constexpr int SLAB_SMEM = SPMM_WARPS * SLAB_RING;

__device__ __forceinline__ void cp_async16_pol(void* smem_dst, const void* gsrc, uint64_t pol) {
  asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "l"(pol)
               : "memory");
}
__device__ __forceinline__ int32_t ldg_pol(const int32_t* p, uint64_t pol) {
  int32_t v;
  asm("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
}
__device__ __forceinline__ float ldg_pol(const float* p, uint64_t pol) {
  float v;
  asm("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(p), "l"(pol));
  return v;
}

template <int SW> struct SlabLane;               // a lane's share of one slab row
template <> struct SlabLane<32> { using V = float; };
template <> struct SlabLane<64> { using V = float2; };

template <int SW, bool HAS_VAL, bool STATS>
__device__ __forceinline__ void spmm_chunk_cta_slab(const SpmmParams& p, const int cta, const int slab, float* s_stat,
                                                    float* ring_all) {
  using V = typename SlabLane<SW>::V;
  constexpr int LPR = SW / 4;                     // lanes per neighbour row (16 B each)
  constexpr int E = 32 / LPR;                     // neighbour rows per warp-wide cp.async
  constexpr int D = SLAB_RING / (SW * 4);         // ring depth in neighbour rows
  constexpr int G = SLAB_G, NG = D / G;           // commit groups in the ring
  static_assert(G % E == 0 && 32 % G == 0 && NG >= 2 && (D & (D - 1)) == 0, "ring geometry");
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* ring = ring_all + (size_t)warp * (SLAB_RING / 4);   // slot s: ring[s*SW .. s*SW + SW)
  uint64_t pol_keep, pol_stream;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol_keep));
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol_stream));

  const int f0 = slab * SW;
  const float* Xs = p.X + f0 + (lane % LPR) * 4;  // this lane's 16-byte slice of a neighbour's slab row
  float* ring_dst = ring + (lane / LPR) * SW + (lane % LPR) * 4;
  const int vlane = slab * 32 + lane;             // this lane's V index within a row of Y / bias

  V ssum, ssq, bias_l;
  vzero(ssum); vzero(ssq); vzero(bias_l);
  if (p.bias) bias_l = load_bias<V>(p.bias, vlane);

  const int chunk = cta * SPMM_WARPS + warp;
  const int row_lo = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk) : 0;
  const int row_hi = chunk < p.n_chunks ? __ldg(p.chunk_rowptr + chunk + 1) : 0;

  auto flush = [&](int row, int deg, V& acc) {
    V y = acc;
    if (p.mean) vdiv(y, (float)max(deg, 1));
    vadd(y, bias_l);
    V* dst = reinterpret_cast<V*>(p.Y + (size_t)row * p.ldy) + vlane;
    if (p.stream_store) vstcs(dst, y); else *dst = y;
    if (STATS) vstat(ssum, ssq, y);
    vzero(acc);
  };

  int next_r = row_lo, next_e = row_lo < row_hi ? __ldg(p.rowptr + row_lo) : 0;
  for (int r = row_lo, e_r = next_e; r < row_hi; r = next_r, e_r = next_e) {
    // ---- a run [r, run_end) of consecutive non-hub rows, ended by a hub row (which belongs to the split path) or by the
    // chunk's end.  A chunk is a few rows and this kernel walks every chunk once per slab, so the run is found 32 rows at a
    // time (one load and a ballot over the degrees) rather than with one dependent rowptr load per row.
    const int e_lo = e_r;
    int run_end = r, e_hi = e_r, rp_first = 0;
    for (;;) {
      const int rr = run_end + lane;
      const int rp1 = rr < row_hi ? __ldg(p.rowptr + rr + 1) : 0;
      if (run_end == r) rp_first = rp1;           // rowptr[r + lane + 1]: the run's first 32 row ends
      int rp0 = __shfl_up_sync(FULL_MASK, rp1, 1);
      if (lane == 0) rp0 = e_hi;
      const unsigned stop = __ballot_sync(FULL_MASK, rr >= row_hi || rp1 - rp0 > p.hub_threshold);
      const int k = stop ? __ffs(stop) - 1 : 31;
      const int end_before = __shfl_sync(FULL_MASK, rp1, (k + 31) & 31);   // rowptr[run_end + k] when k > 0
      next_e = __shfl_sync(FULL_MASK, rp1, k);                            // rowptr[run_end + k + 1]
      if (stop) {
        if (k > 0) e_hi = end_before;
        run_end += k;
        break;
      }
      e_hi = next_e;
      run_end += 32;
    }
    next_r = run_end + 1;                         // past the hub row that ends the run (or past row_hi)
    if (run_end == r) continue;                   // row r is a hub row
    const int n = e_hi - e_lo;

    // Edge windows of 32 (col, val), each loaded one window ahead of its use so that the load latency hides behind the
    // previous window's gathers; the first two are loaded here, before the run's first copies and empty rows.
    auto col_win = [&](int jw) { const int e = e_lo + jw + lane; return e < e_hi ? ldg_pol(p.col + e, pol_stream) : 0; };
    auto val_win = [&](int jw) { const int e = e_lo + jw + lane; return e < e_hi ? ldg_pol(p.val + e, pol_stream) : 0.f; };
    int cI = col_win(0), cN = col_win(32);
    float vA = 1.f, vN = 1.f;
    if (HAS_VAL) { vA = val_win(0); vN = val_win(32); }

    int rbase = r;                                // row ends of the run, 32 at a time in registers
    int rp = (rbase + lane < run_end) ? rp_first : e_hi;
    auto row_end_of = [&](int row) {
      if (row - rbase >= 32) {                    // warp-uniform
        rbase = row;
        rp = (rbase + lane < run_end) ? __ldg(p.rowptr + rbase + lane + 1) : e_hi;
      }
      return __shfl_sync(FULL_MASK, rp, row - rbase);
    };

    V acc;
    vzero(acc);
    int row_beg = e_lo;
    int rend = row_end_of(r);
    while (r < run_end && rend == row_beg) {      // leading empty rows
      flush(r, 0, acc);
      ++r;
      if (r < run_end) rend = row_end_of(r);
    }
    if (n == 0) continue;

    // Issue side: the column window (cI); edge jg + u is copied by lanes [u%E·LPR, u%E·LPR + LPR) of warp instruction u/E.
    // Consume side: the value window (vA).  Both advance in groups of G edges; one commit per group (empty past the run's
    // end, so the group count stays uniform), NG groups in the ring.
    auto issue_group = [&](int jg, int slot0) {   // edges jg..jg+G-1 (relative to e_lo) -> slots slot0..slot0+G-1
      if (jg < n) {                               // warp-uniform
        if (jg > 0 && (jg & 31) == 0) { cI = cN; cN = col_win(jg + 32); }
#pragma unroll
        for (int i = 0; i < G / E; ++i) {
          const int u = i * E + lane / LPR;
          const int cc = __shfl_sync(FULL_MASK, cI, (jg + u) & 31);
          if (jg + u < n) cp_async16_pol(ring_dst + (slot0 + i * E) * SW, Xs + (size_t)cc * p.ldx, pol_keep);
        }
      }
      cp_async_commit();
    };
    auto boundary = [&]() {                       // the current row is complete: store it (+ empty rows that follow)
      do {
        flush(r, rend - row_beg, acc);
        row_beg = rend;
        ++r;
        if (r < run_end) rend = row_end_of(r);
      } while (r < run_end && rend == row_beg);
    };
    auto consume_group = [&](int j0, int slot0) {  // j0 < n
      if (HAS_VAL && j0 > 0 && (j0 & 31) == 0) { vA = vN; vN = val_win(j0 + 32); }
      const V* sbase = reinterpret_cast<const V*>(ring + slot0 * SW) + lane;
      const int cnt = min(G, n - j0);
      int done = 0;
      while (done < cnt) {                        // pieces of the group that lie in one row (all warp-uniform)
        const int room = rend - (e_lo + j0 + done);   // >= 1: edges left in the current row
        const int take = min(cnt - done, room);
        if (take == G) {                          // common case: the whole group inside one row
#pragma unroll
          for (int u = 0; u < G; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
            vfma(acc, w, sbase[u * 32]);
          }
        } else {
#pragma unroll 1
          for (int u = done; u < done + take; ++u) {
            const float w = HAS_VAL ? __shfl_sync(FULL_MASK, vA, (j0 + u) & 31) : 1.f;
            vfma(acc, w, sbase[u * 32]);
          }
        }
        done += take;
        if (take == room) boundary();
      }
    };
#pragma unroll
    for (int g = 0; g < NG; ++g) issue_group(g * G, g * G);
#pragma unroll 1
    for (int j = 0, s0 = 0; j < n; j += G, s0 = (s0 + G) & (D - 1)) {
      cp_async_wait<NG - 1>();                    // this thread's copies of the oldest group have landed
      __syncwarp();                               // ... and every other lane's
      consume_group(j, s0);
      __syncwarp();                               // every lane has read the slots before they are refilled
      issue_group(j + D, s0);
    }
    cp_async_wait<0>();
  }

  if (STATS) {
    float* ss = s_stat;
    float* sq = s_stat + SW;
    for (int i = threadIdx.x; i < 2 * SW; i += SPMM_THREADS) s_stat[i] = 0.f;
    __syncthreads();
    for (int w = 0; w < SPMM_WARPS; ++w) {          // fixed order => deterministic, the bulk kernel's order
      if (warp == w) smem_accum(ss, sq, lane, ssum, ssq);
      __syncthreads();
    }
    float* out = p.stat_partial + (size_t)cta * 2 * p.K + f0;
    for (int i = threadIdx.x; i < SW; i += SPMM_THREADS) { out[i] = ss[i]; out[p.K + i] = sq[i]; }
  }
}

// Grid: the n_seg hub-segment CTAs (full width), then n_slabs slabs of main_grid chunk CTAs each, slab-major.
template <int SW, bool HAS_VAL, bool STATS>
__global__ void __launch_bounds__(SPMM_THREADS, 3) spmm_rows_slab_kernel(const SpmmParams p) {
  __shared__ float s_mem[2 * SPMM_MAX_SLAB_FLOATS];
  extern __shared__ __align__(128) unsigned char s_dyn[];
  const int b = (int)blockIdx.x;
  if (b < p.n_seg) {   // CH = 1: 128-float passes; each element's order does not depend on CH (and CH = 2 would spill)
    spmm_hub_seg_cta<float4, 1, HAS_VAL>(p, b, s_mem);
    return;
  }
  const int slab = (b - p.n_seg) / p.main_grid;
  spmm_chunk_cta_slab<SW, HAS_VAL, STATS>(p, b - p.n_seg - slab * p.main_grid, slab, s_mem, reinterpret_cast<float*>(s_dyn));
}


// ------------------------------------------------------------------ narrow rows (K <= 64 floats: e.g. the 40 logits)
// A 160-byte row needs only 10 lanes.  Instead of folding several NEIGHBOURS of one row across the warp (which drains
// at every row end and needs cross-group shuffles), each group of lanes takes its OWN ROW of the chunk: 3 rows
// (K=40) advance concurrently per warp, each with 4 independent 128-bit gathers in flight, no shuffles at all.
template <bool HAS_VAL, int U>
__device__ __forceinline__ void spmm_chunk_cta_narrow(const SpmmParams& p, const int cta) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int lpr = p.nvec, groups = 32 / lpr;
  const int g = lane / lpr, l = lane - g * lpr;
  const bool active = g < groups;
  const float4* Xv = reinterpret_cast<const float4*>(p.X);
  float4* Yv = reinterpret_cast<float4*>(p.Y);
  const size_t ldxv = (size_t)(p.ldx / 4), ldyv = (size_t)(p.ldy / 4);
  const int chunk = cta * SPMM_WARPS + warp;
  if (chunk >= p.n_chunks || !active) return;
  const int row_lo = __ldg(p.chunk_rowptr + chunk), row_hi = __ldg(p.chunk_rowptr + chunk + 1);
  float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
  if (p.bias) bias4 = load_bias<float4>(p.bias, l);
  for (int row = row_lo + g; row < row_hi; row += groups) {
    const int beg = __ldg(p.rowptr + row), end = __ldg(p.rowptr + row + 1);
    const int deg = end - beg;
    if (deg > p.hub_threshold) continue;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int e = beg;
    if (e + U <= end) {                              // software-pipelined: the next batch's (col,val) load overlaps this batch's gathers
      int c[U]; float w[U];
#pragma unroll
      for (int u = 0; u < U; ++u) { c[u] = __ldg(p.col + e + u); w[u] = HAS_VAL ? __ldg(p.val + e + u) : 1.f; }
      for (; e + U <= end; e += U) {
        float4 x[U];
#pragma unroll
        for (int u = 0; u < U; ++u) x[u] = vldg(Xv + (size_t)c[u] * ldxv + l);
        float wc[U];
#pragma unroll
        for (int u = 0; u < U; ++u) wc[u] = w[u];
        if (e + 2 * U <= end) {
#pragma unroll
          for (int u = 0; u < U; ++u) { c[u] = __ldg(p.col + e + U + u); w[u] = HAS_VAL ? __ldg(p.val + e + U + u) : 1.f; }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) vfma(acc, wc[u], x[u]);
      }
    }
    if (U > 4 && e + 4 <= end) {                     // a half batch before the scalar tail
      int c[4]; float w[4]; float4 x[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) { c[u] = __ldg(p.col + e + u); w[u] = HAS_VAL ? __ldg(p.val + e + u) : 1.f; }
#pragma unroll
      for (int u = 0; u < 4; ++u) x[u] = vldg(Xv + (size_t)c[u] * ldxv + l);
#pragma unroll
      for (int u = 0; u < 4; ++u) vfma(acc, w[u], x[u]);
      e += 4;
    }
    for (; e < end; ++e) {
      const int c = __ldg(p.col + e);
      const float w = HAS_VAL ? __ldg(p.val + e) : 1.f;
      vfma(acc, w, vldg(Xv + (size_t)c * ldxv + l));
    }
    if (p.mean) vdiv(acc, (float)max(deg, 1));
    if (p.bias) vadd(acc, bias4);
    if (p.n_yp) y_row_v4(p, row)[l] = acc; else Yv[(size_t)row * ldyv + l] = acc;
  }
}

template <bool HAS_VAL, int U>
__global__ void __launch_bounds__(SPMM_THREADS, 3) spmm_rows_narrow_kernel(const SpmmParams p) {
  __shared__ float s_mem[SPMM_MAX_SLAB_FLOATS];
  if ((int)blockIdx.x < p.n_seg) spmm_hub_seg_cta<float4, 1, HAS_VAL>(p, (int)blockIdx.x, s_mem);
  else spmm_chunk_cta_narrow<HAS_VAL, U>(p, (int)blockIdx.x - p.n_seg);
}

// Sum a hub row's segment partials in segment order, apply the epilogue.
__global__ void __launch_bounds__(256) spmm_hub_finalize_kernel(const SpmmParams p) {
  __shared__ float4 sh[256];
  const int h = blockIdx.x;
  const int row = __ldg(p.hub_rows + h);
  const int s0 = __ldg(p.hub_segptr + h), s1 = __ldg(p.hub_segptr + h + 1);
  const int deg = __ldg(p.rowptr + row + 1) - __ldg(p.rowptr + row);
  float* stat = p.stat_partial ? p.stat_partial + (size_t)(p.main_grid + h) * 2 * p.K : nullptr;
  const int nvec = p.K >> 2;
  const auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if ((p.K & 3) == 0 && nvec <= 256 && (p.ldy & 3) == 0 && al16(p.Y) && al16(p.hub_ws) && (!stat || al16(stat))) {
    // segment-parallel: G groups of nvec lanes, group g adds segments s0+g, s0+g+G, ...; groups combined in order
    const int G = min(256 / nvec, 16);
    const int v = threadIdx.x % nvec, g = threadIdx.x / nvec;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g < G)
      for (int s = s0 + g; s < s1; s += G) {
        const float4 x = *reinterpret_cast<const float4*>(p.hub_ws + (size_t)s * p.K + 4 * v);
        acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
      }
    sh[threadIdx.x] = acc;
    __syncthreads();
    if (g != 0) return;
    for (int j = 1; j < G; ++j) {
      const float4 x = sh[j * nvec + v];
      acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
    }
    if (p.mean) { const float d = (float)max(deg, 1); acc.x /= d; acc.y /= d; acc.z /= d; acc.w /= d; }
    if (p.bias) {
      acc.x += __ldg(p.bias + 4 * v); acc.y += __ldg(p.bias + 4 * v + 1);
      acc.z += __ldg(p.bias + 4 * v + 2); acc.w += __ldg(p.bias + 4 * v + 3);
    }
    if (p.n_yp) y_row_v4(p, row)[v] = acc; else *reinterpret_cast<float4*>(p.Y + (size_t)row * p.ldy + 4 * v) = acc;
    if (stat) {
      *reinterpret_cast<float4*>(stat + 4 * v) = acc;
      *reinterpret_cast<float4*>(stat + p.K + 4 * v) = make_float4(acc.x * acc.x, acc.y * acc.y, acc.z * acc.z, acc.w * acc.w);
    }
    return;
  }
  // scalar path (K % 4 != 0, K > 1024 or a misaligned operand); in scatter mode the row goes to its rank's buffer
  float* yrow = p.n_yp ? reinterpret_cast<float*>(y_row_v4(p, row)) : p.Y + (size_t)row * p.ldy;
  for (int k = threadIdx.x; k < p.K; k += blockDim.x) {
    float acc = 0.f;
    for (int s = s0; s < s1; ++s) acc += p.hub_ws[(size_t)s * p.K + k];
    if (p.mean) acc /= (float)max(deg, 1);
    if (p.bias) acc += __ldg(p.bias + k);
    yrow[k] = acc;
    if (stat) { stat[k] = acc; stat[p.K + k] = acc * acc; }
  }
}

// Column sum / sum-of-squares of a dense [n_rows,K] matrix into `slots`
// deterministic partials (used when the producer could not fuse them).
__global__ void __launch_bounds__(256) col_stats_kernel(const float* __restrict__ Y, int64_t ldy, int64_t n_rows,
                                                        int K, float* __restrict__ partial, int slots) {
  const int slot = blockIdx.x;
  const int64_t per = (n_rows + slots - 1) / slots;
  const int64_t r0 = (int64_t)slot * per, r1 = min(n_rows, r0 + per);
  float* out = partial + (size_t)slot * 2 * K;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    float s = 0.f, q = 0.f;
    for (int64_t r = r0; r < r1; ++r) {
      const float y = Y[(size_t)r * ldy + k];
      s += y; q = fmaf(y, y, q);
    }
    out[k] = s; out[K + k] = q;
  }
}

template <typename V, int CH>
static int launch_spmm(const SpmmParams& p, cudaStream_t st) {
  int rc;
  const bool stats = p.stat_partial != nullptr;
  const int grid = p.main_grid + p.n_seg;
  if (p.val) {
    if (stats) spmm_rows_kernel<V, CH, true, true><<<grid, SPMM_THREADS, 0, st>>>(p);
    else spmm_rows_kernel<V, CH, true, false><<<grid, SPMM_THREADS, 0, st>>>(p);
  } else {
    if (stats) spmm_rows_kernel<V, CH, false, true><<<grid, SPMM_THREADS, 0, st>>>(p);
    else spmm_rows_kernel<V, CH, false, false><<<grid, SPMM_THREADS, 0, st>>>(p);
  }
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    spmm_hub_finalize_kernel<<<p.n_hub, 256, 0, st>>>(p);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

template <int CH>
static int launch_spmm_pipe(const SpmmParams& p, cudaStream_t st) {
  int rc;
  const bool stats = p.stat_partial != nullptr;
  const int grid = p.main_grid + p.n_seg;
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_done_dev[64] = {};
  if (dev >= 0 && dev < 64 && !attr_done_dev[dev]) {
    cudaFuncSetAttribute(spmm_rows_pipe_kernel<CH, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PIPE_SMEM);
    cudaFuncSetAttribute(spmm_rows_pipe_kernel<CH, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PIPE_SMEM);
    cudaFuncSetAttribute(spmm_rows_pipe_kernel<CH, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, PIPE_SMEM);
    cudaFuncSetAttribute(spmm_rows_pipe_kernel<CH, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, PIPE_SMEM);
    attr_done_dev[dev] = true;
  }
  if (p.val) {
    if (stats) spmm_rows_pipe_kernel<CH, true, true><<<grid, SPMM_THREADS, PIPE_SMEM, st>>>(p);
    else spmm_rows_pipe_kernel<CH, true, false><<<grid, SPMM_THREADS, PIPE_SMEM, st>>>(p);
  } else {
    if (stats) spmm_rows_pipe_kernel<CH, false, true><<<grid, SPMM_THREADS, PIPE_SMEM, st>>>(p);
    else spmm_rows_pipe_kernel<CH, false, false><<<grid, SPMM_THREADS, PIPE_SMEM, st>>>(p);
  }
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    spmm_hub_finalize_kernel<<<p.n_hub, 256, 0, st>>>(p);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

constexpr int BULK_SMEM_2CTA = 112 * 1024;       // dynamic smem request that leaves room for only 2 CTAs per SM

template <int CH, int G>
static int launch_spmm_bulk(const SpmmParams& p, cudaStream_t st, bool two_ctas) {
  int rc;
  const bool stats = p.stat_partial != nullptr;
  const int grid = (p.main_grid + p.n_seg) * p.n_slabs;
  const int smem = two_ctas ? BULK_SMEM_2CTA : BULK_SMEM;
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_done[64] = {};                  // per device (cudaFuncSetAttribute is per device); idempotent if raced
  if (dev >= 0 && dev < 64 && !attr_done[dev]) {
    cudaFuncSetAttribute(spmm_rows_bulk_kernel<CH, G, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BULK_SMEM_2CTA);
    cudaFuncSetAttribute(spmm_rows_bulk_kernel<CH, G, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BULK_SMEM_2CTA);
    cudaFuncSetAttribute(spmm_rows_bulk_kernel<CH, G, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BULK_SMEM_2CTA);
    cudaFuncSetAttribute(spmm_rows_bulk_kernel<CH, G, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BULK_SMEM_2CTA);
    attr_done[dev] = true;
  }
  if (p.val) {
    if (stats) spmm_rows_bulk_kernel<CH, G, true, true><<<grid, SPMM_THREADS, smem, st>>>(p);
    else spmm_rows_bulk_kernel<CH, G, true, false><<<grid, SPMM_THREADS, smem, st>>>(p);
  } else {
    if (stats) spmm_rows_bulk_kernel<CH, G, false, true><<<grid, SPMM_THREADS, smem, st>>>(p);
    else spmm_rows_bulk_kernel<CH, G, false, false><<<grid, SPMM_THREADS, smem, st>>>(p);
  }
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    spmm_hub_finalize_kernel<<<p.n_hub, 256, 0, st>>>(p);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

template <int SW>
static int launch_spmm_slab(const SpmmParams& p, cudaStream_t st) {
  int rc;
  const bool stats = p.stat_partial != nullptr;
  const int grid = p.n_seg + p.main_grid * p.n_slabs;
  int dev = 0;
  cudaGetDevice(&dev);
  static bool attr_done[64] = {};                  // per device (cudaFuncSetAttribute is per device); idempotent if raced
  if (dev >= 0 && dev < 64 && !attr_done[dev]) {
    cudaFuncSetAttribute(spmm_rows_slab_kernel<SW, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SLAB_SMEM);
    cudaFuncSetAttribute(spmm_rows_slab_kernel<SW, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SLAB_SMEM);
    cudaFuncSetAttribute(spmm_rows_slab_kernel<SW, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SLAB_SMEM);
    cudaFuncSetAttribute(spmm_rows_slab_kernel<SW, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SLAB_SMEM);
    attr_done[dev] = true;
  }
  if (p.val) {
    if (stats) spmm_rows_slab_kernel<SW, true, true><<<grid, SPMM_THREADS, SLAB_SMEM, st>>>(p);
    else spmm_rows_slab_kernel<SW, true, false><<<grid, SPMM_THREADS, SLAB_SMEM, st>>>(p);
  } else {
    if (stats) spmm_rows_slab_kernel<SW, false, true><<<grid, SPMM_THREADS, SLAB_SMEM, st>>>(p);
    else spmm_rows_slab_kernel<SW, false, false><<<grid, SPMM_THREADS, SLAB_SMEM, st>>>(p);
  }
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    spmm_hub_finalize_kernel<<<p.n_hub, 256, 0, st>>>(p);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

template <typename V>
static int dispatch_ch(const SpmmParams& p, cudaStream_t st) {
  if (p.nvec <= 32) return launch_spmm<V, 1>(p, st);
  if (p.nvec <= 64) return launch_spmm<V, 2>(p, st);
  return launch_spmm<V, 4>(p, st);
}

// ------------------------------------------------------------ hub plan kernels
__global__ void __launch_bounds__(1024) hub_count_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows,
                                                         int32_t thr, int32_t seg_len, int32_t* __restrict__ out) {
  __shared__ int s_cnt[2];
  if (threadIdx.x < 2) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  int nh = 0, ns = 0;
  for (int64_t r = threadIdx.x; r < n_rows; r += blockDim.x) {
    const int deg = rowptr[r + 1] - rowptr[r];
    if (deg > thr) { nh += 1; ns += (deg + seg_len - 1) / seg_len; }
  }
  atomicAdd(&s_cnt[0], nh);
  atomicAdd(&s_cnt[1], ns);
  __syncthreads();
  if (threadIdx.x < 2) out[threadIdx.x] = s_cnt[threadIdx.x];
}

// Ordered compaction of hub rows (ascending row id) with their segment offsets.
__global__ void __launch_bounds__(1024) hub_fill_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows,
                                                        int32_t thr, int32_t seg_len, int32_t* __restrict__ hub_rows,
                                                        int32_t* __restrict__ hub_segptr, int64_t n_hub) {
  __shared__ int s_wflag[32], s_wseg[32];
  __shared__ int s_base[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_base[0] = 0; s_base[1] = 0; }
  __syncthreads();
  for (int64_t r0 = 0; r0 < n_rows; r0 += blockDim.x) {
    const int64_t r = r0 + threadIdx.x;
    int flag = 0, segs = 0;
    if (r < n_rows) {
      const int deg = rowptr[r + 1] - rowptr[r];
      if (deg > thr) { flag = 1; segs = (deg + seg_len - 1) / seg_len; }
    }
    int f = flag, s = segs;  // inclusive warp scans
    for (int d = 1; d < 32; d <<= 1) {
      const int of = __shfl_up_sync(FULL_MASK, f, d), os = __shfl_up_sync(FULL_MASK, s, d);
      if (lane >= d) { f += of; s += os; }
    }
    if (lane == 31) { s_wflag[warp] = f; s_wseg[warp] = s; }
    __syncthreads();
    if (warp == 0) {
      int wf = s_wflag[lane], wsg = s_wseg[lane];
      int xf = wf, xs = wsg;
      for (int d = 1; d < 32; d <<= 1) {
        const int of = __shfl_up_sync(FULL_MASK, xf, d), os = __shfl_up_sync(FULL_MASK, xs, d);
        if (lane >= d) { xf += of; xs += os; }
      }
      s_wflag[lane] = xf - wf;  // exclusive warp offsets
      s_wseg[lane] = xs - wsg;
    }
    __syncthreads();
    const int pos = s_base[0] + s_wflag[warp] + f - flag;
    const int soff = s_base[1] + s_wseg[warp] + s - segs;
    if (flag && pos < n_hub) { hub_rows[pos] = (int32_t)r; hub_segptr[pos] = soff; }
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) {
      s_base[0] = pos + flag;
      s_base[1] = soff + segs;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) hub_segptr[n_hub] = s_base[1];
}

// chunk c starts at the first row r with key(r) = rowptr[r] + r*row_cost >= c*chunk_nnz  (key is strictly
// increasing, so empty rows are spread over chunks too); chunk_rowptr[n_chunks] = n_rows.
__global__ void __launch_bounds__(256) chunk_plan_kernel(const int32_t* __restrict__ rowptr, int64_t n_rows,
                                                         int32_t chunk_nnz, int32_t row_cost,
                                                         int32_t* __restrict__ chunk_rowptr, int64_t n_chunks) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c > n_chunks) return;
  if (c == n_chunks) { chunk_rowptr[c] = (int32_t)n_rows; return; }
  const int64_t target = c * (int64_t)chunk_nnz;
  int64_t lo = 0, hi = n_rows;  // smallest r in [0,n_rows] with key(r) >= target
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const int64_t key = (int64_t)rowptr[mid] + mid * (int64_t)row_cost;
    if (key >= target) hi = mid; else lo = mid + 1;
  }
  chunk_rowptr[c] = (int32_t)lo;
}

}  // namespace b200gnn

using namespace b200gnn;

// see the variant word in b200gnn_spmm_csr_f32
static int g_spmm_variant = 0;

struct ScatterArgs { int n; float* ptr[16]; int32_t off[17]; int64_t ld, col; };
static thread_local ScatterArgs g_scatter = {0, {}, {}, 0, 0};

// Slab width (floats) the bulk kernel uses when left to choose: the widest slab the ring supports.  The copy engine
// retires a roughly fixed number of row copies per second whatever their size (tools/bulk_probe.cu), so narrower slabs
// pay more in per-copy cost than their L2 residency wins back.
static int bulk_auto_slab(int64_t K, int64_t n_src) {
  (void)n_src;
  return (K % 256 == 0) ? 256 : 128;
}
// The lane-copy slab kernel takes K = 128 / 256 when X is larger than SLAB_L2_BUDGET bytes and the choice is automatic.
// tools/l2_probe.cu (H100 SXM, BENCH.md): random 256-byte row gathers reach 7.3 TB/s from tables up to 40 MB, 6.7 at
// 48 MB, 5.7 at 64 MB; below 40 MB the bulk kernel's full-width rows are L2 hits already.  Slab width 64 floats: 32-float
// slabs (22 MB per slab at ARXIV shape) hit L2 more often but double the per-slab walk of every chunk, and measured
// slower than the bulk kernel at both widths.
constexpr int64_t SLAB_L2_BUDGET = (int64_t)40 << 20;
constexpr int SLAB_SW = 64;
extern "C" void b200gnn_spmm_set_variant(int v) { g_spmm_variant = v; }

extern "C" int64_t b200gnn_csr_chunk_count(int64_t n_rows, int64_t nnz, int32_t chunk_nnz, int32_t row_cost) {
  if (n_rows < 0 || nnz < 0 || chunk_nnz <= 0 || row_cost <= 0) return B200GNN_ERR_BAD_ARG;
  const int64_t total = nnz + n_rows * (int64_t)row_cost;
  return total == 0 ? 0 : (total + chunk_nnz - 1) / chunk_nnz;
}

extern "C" int b200gnn_csr_chunk_plan(const int32_t* rowptr, int64_t n_rows, int64_t nnz, int32_t chunk_nnz,
                                      int32_t row_cost, int32_t* chunk_rowptr, void* stream) {
  const int64_t n_chunks = b200gnn_csr_chunk_count(n_rows, nnz, chunk_nnz, row_cost);
  if (n_chunks < 0 || !rowptr || !chunk_rowptr) return B200GNN_ERR_BAD_ARG;
  chunk_plan_kernel<<<(int)((n_chunks + 1 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(rowptr, n_rows, chunk_nnz,
                                                                                        row_cost, chunk_rowptr, n_chunks);
  return check_launch();
}

extern "C" int b200gnn_csr_hub_count(const int32_t* rowptr, int64_t n_rows, int32_t hub_threshold, int32_t seg_len,
                                     int32_t* counts_out, void* stream) {
  if (!rowptr || !counts_out || n_rows < 0 || hub_threshold < 0 || seg_len <= 0) return B200GNN_ERR_BAD_ARG;
  hub_count_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(rowptr, n_rows, hub_threshold, seg_len, counts_out);
  return check_launch();
}

extern "C" int b200gnn_csr_hub_fill(const int32_t* rowptr, int64_t n_rows, int32_t hub_threshold, int32_t seg_len,
                                    int32_t* hub_rows, int32_t* hub_segptr, int64_t n_hub, void* stream) {
  if (!rowptr || !hub_segptr || n_rows < 0 || n_hub < 0 || hub_threshold < 0 || seg_len <= 0) return B200GNN_ERR_BAD_ARG;
  if (n_hub > 0 && !hub_rows) return B200GNN_ERR_BAD_ARG;
  hub_fill_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(rowptr, n_rows, hub_threshold, seg_len, hub_rows, hub_segptr, n_hub);
  return check_launch();
}

extern "C" int64_t b200gnn_spmm_stat_slots(int64_t n_chunks, int64_t n_hub) {
  return (n_chunks + SPMM_WARPS - 1) / SPMM_WARPS + n_hub;
}

extern "C" int b200gnn_spmm_csr_f32(const int32_t* rowptr, const int32_t* col, const float* val, const float* X,
                                    int64_t ldx, float* Y, int64_t ldy, int64_t n_rows, int64_t n_src, int64_t K,
                                    int reduce, const float* bias, float* stat_partial,
                                    const int32_t* chunk_rowptr, int64_t n_chunks, int32_t hub_threshold,
                                    int32_t seg_len, const int32_t* hub_rows, const int32_t* hub_segptr,
                                    int64_t n_hub, int64_t n_seg, float* hub_workspace, void* stream) {
  if (n_rows < 0 || n_src < 0 || K <= 0 || n_rows >= INT32_MAX || n_src >= INT32_MAX || K > (1 << 20))
    return B200GNN_ERR_BAD_ARG;
  if (reduce != B200GNN_REDUCE_SUM && reduce != B200GNN_REDUCE_MEAN) return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  if (!rowptr || !Y || ldy < K || !chunk_rowptr || n_chunks <= 0 || n_chunks >= INT32_MAX) return B200GNN_ERR_BAD_ARG;
  if (n_src > 0 && (!X || ldx < K)) return B200GNN_ERR_BAD_ARG;  // col may be NULL when nnz == 0
  if (n_hub < 0 || n_seg < 0 || hub_threshold < 0) return B200GNN_ERR_BAD_ARG;
  if (n_hub > 0 && (!hub_rows || !hub_segptr || !hub_workspace || seg_len <= 0 || n_seg < n_hub))
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;

  SpmmParams p;
  p.rowptr = rowptr; p.col = col; p.val = val; p.X = X; p.Y = Y; p.bias = bias;
  p.stat_partial = stat_partial;
  p.chunk_rowptr = chunk_rowptr; p.n_chunks = (int32_t)n_chunks;
  p.hub_rows = hub_rows; p.hub_segptr = hub_segptr; p.hub_ws = hub_workspace;
  p.ldx = ldx; p.ldy = ldy;
  p.n_rows = (int32_t)n_rows; p.K = (int32_t)K;
  p.hub_threshold = hub_threshold; p.seg_len = seg_len; p.n_hub = (int32_t)n_hub;
  p.n_seg = n_hub > 0 ? (int32_t)n_seg : 0;
  p.mean = reduce == B200GNN_REDUCE_MEAN;
  p.stream_store = (n_rows * K * 4 > (int64_t)64 << 20) ? 1 : 0;
  p.main_grid = (int32_t)((n_chunks + SPMM_WARPS - 1) / SPMM_WARPS);

  // widest vector type the layout allows
  int W = 1;
  if (K % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && aligned_to(X, 16) && aligned_to(Y, 16)) W = 4;
  else if (K % 2 == 0 && ldx % 2 == 0 && ldy % 2 == 0 && aligned_to(X, 8) && aligned_to(Y, 8)) W = 2;
  p.nvec = (int32_t)(K / W);
  p.n_slabs = 1; p.l2_hint = 0;
  p.n_yp = 0; p.ycol = 0; p.ldyp = 0;
  if (g_scatter.n > 0) {            // set by b200gnn_spmm_csr_scatter_f32 around this call (same thread)
    if (W != 4 || K % 4 || g_scatter.ld % 4 || g_scatter.col % 4) return B200GNN_ERR_UNSUPPORTED;
    // only the bulk-copy kernels (automatic choice or families 3-7) and the narrow kernel store through y_row_v4
    const int sfam = g_spmm_variant & 15;
    const bool to_bulk = K % 128 == 0 && K <= 4096 && (sfam == 0 || (sfam >= 3 && sfam <= 7));
    const bool to_narrow = p.nvec <= 16 && !stat_partial && sfam != 1 && sfam != 2;
    if (!to_bulk && !to_narrow) return B200GNN_ERR_UNSUPPORTED;
    p.n_yp = g_scatter.n; p.ycol = (int32_t)g_scatter.col; p.ldyp = g_scatter.ld;
    for (int q = 0; q < g_scatter.n; ++q) { p.Yp[q] = g_scatter.ptr[q]; p.yoff[q] = g_scatter.off[q]; }
    p.yoff[g_scatter.n] = g_scatter.off[g_scatter.n];
  }

  // Variant word (b200gnn_spmm_set_variant; tuning and A/B tests): low nibble = kernel family
  //   0 automatic, 1 register-staged, 2 cp.async ring (round-1 kernel), 3 bulk-copy ring, one slab of min(K,256) floats
  //   per pass, 4 bulk-copy ring with 128-float slabs, 5 bulk-copy ring with 256-float slabs, 6 / 7 bulk-copy ring
  //   with 128-float slabs and 8 / 4 edges per barrier group;
  //   +16 = evict_last L2 policy on the gathers, +32 = the other barrier-group size, +64 = 2 CTAs per SM.
  // Automatic choice only: X beyond the L2 budget at the widths the bulk kernel serves -> the lane-copy slab kernel,
  // which reproduces the bulk kernel's results bit for bit.
  if (g_spmm_variant == 0 && W == 4 && p.n_yp == 0 && (K == 128 || K == 256) && n_src * K * 4 > SLAB_L2_BUDGET) {
    p.n_slabs = (int32_t)(K / SLAB_SW);
    return launch_spmm_slab<SLAB_SW>(p, st);
  }

  const int fam = g_spmm_variant & 15;
  const bool alt_g = (g_spmm_variant & 32) != 0;
  int bulk_sw = 0;                                  // slab width in floats (0 = not the bulk kernel)
  if (W == 4 && K % 128 == 0 && K <= 4096) {
    if (fam == 3) bulk_sw = (K % 256 == 0) ? 256 : 128;
    else if (fam == 4) bulk_sw = 128;
    else if (fam == 5) bulk_sw = (K % 256 == 0) ? 256 : 128;
    else if (fam == 6 || fam == 7) bulk_sw = 128;
    else if (fam == 0) bulk_sw = bulk_auto_slab(K, n_src);
  }
  int rc;
  float* fused_stats = stat_partial;
  bool single_slab = true;
  if (bulk_sw) {
    p.n_slabs = (int32_t)(K / bulk_sw);
    p.l2_hint = (g_spmm_variant & 16) ? 1 : 0;
    if (fam == 6) return launch_spmm_bulk<1, 8>(p, st, false);
    if (fam == 7) return launch_spmm_bulk<1, 4>(p, st, false);
    const bool two = (g_spmm_variant & 64) != 0;    // +64: two CTAs per SM instead of three
    if (bulk_sw == 128) rc = alt_g ? launch_spmm_bulk<1, 2>(p, st, two) : launch_spmm_bulk<1, 4>(p, st, two);
    else rc = alt_g ? launch_spmm_bulk<2, 2>(p, st, two) : launch_spmm_bulk<2, 4>(p, st, two);
    return rc;                                      // statistics are fused per slab
  }

  const int ch = p.nvec <= 32 ? 1 : (p.nvec <= 64 ? 2 : 4);
  single_slab = p.nvec <= 32 * ch;
  if (!single_slab) p.stat_partial = nullptr;  // stats by a separate pass below

  const bool pipe_ok = (W == 4) && fam == 2 && (p.nvec == 32 || p.nvec == 64 || p.nvec == 128);
  const bool narrow_ok = (W == 4) && p.nvec <= 16 && !p.stat_partial && fam != 1;
  if (narrow_ok) {
    rc = B200GNN_OK;
    const int grid = p.main_grid + p.n_seg;
    const bool deep = (g_spmm_variant & 128) != 0;   // +128: 8 gathers in flight per lane group instead of 4 (A/B)
    if (p.val) { if (deep) spmm_rows_narrow_kernel<true, 8><<<grid, SPMM_THREADS, 0, st>>>(p); else spmm_rows_narrow_kernel<true, 4><<<grid, SPMM_THREADS, 0, st>>>(p); }
    else { if (deep) spmm_rows_narrow_kernel<false, 8><<<grid, SPMM_THREADS, 0, st>>>(p); else spmm_rows_narrow_kernel<false, 4><<<grid, SPMM_THREADS, 0, st>>>(p); }
    if ((rc = check_launch())) return rc;
    if (p.n_hub > 0) {
      spmm_hub_finalize_kernel<<<p.n_hub, 256, 0, st>>>(p);
      if ((rc = check_launch())) return rc;
    }
  }
  else if (pipe_ok && p.nvec == 32) rc = launch_spmm_pipe<1>(p, st);
  else if (pipe_ok && p.nvec == 64) rc = launch_spmm_pipe<2>(p, st);
  else if (pipe_ok && p.nvec == 128) rc = launch_spmm_pipe<4>(p, st);
  else if (W == 4) rc = dispatch_ch<float4>(p, st);
  else if (W == 2) rc = dispatch_ch<float2>(p, st);
  else rc = dispatch_ch<float>(p, st);
  if (rc) return rc;

  if (fused_stats && !single_slab) {
    const int slots = (int)b200gnn_spmm_stat_slots(n_chunks, n_hub);
    col_stats_kernel<<<slots, 256, 0, st>>>(Y, ldy, n_rows, (int)K, fused_stats, slots);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

// The same product with the C->R layout exchange of the multi-GPU engine fused into the epilogue: output row i goes to
// Y_ptrs[q][(i - row_off[q]) * ldy_dst + col_dst ...] for the rank q that owns it (row_off: world+1 ascending offsets, HOST
// array; Y_ptrs: HOST array of `world` device pointers, peer-mapped R-layout buffers).  Supported where the TMA kernels
// (K % 128 == 0) or the narrow kernel (K <= 64, no statistics) run; Y itself is not written.
extern "C" int b200gnn_spmm_csr_scatter_f32(const int32_t* rowptr, const int32_t* col, const float* val, const float* X,
                                            int64_t ldx, float* const* Y_ptrs, const int32_t* row_off, int32_t world,
                                            int64_t ldy_dst, int64_t col_dst, int64_t n_rows, int64_t n_src, int64_t K, int reduce,
                                            const float* bias, const int32_t* chunk_rowptr, int64_t n_chunks,
                                            int32_t hub_threshold, int32_t seg_len, const int32_t* hub_rows,
                                            const int32_t* hub_segptr, int64_t n_hub, int64_t n_seg, float* hub_workspace,
                                            void* stream) {
  if (!Y_ptrs || !row_off || world <= 0 || world > 16 || ldy_dst < K || col_dst < 0 || row_off[0] != 0 || row_off[world] != n_rows)
    return B200GNN_ERR_BAD_ARG;
  g_scatter.n = world; g_scatter.ld = ldy_dst; g_scatter.col = col_dst;
  for (int q = 0; q < world; ++q) {
    if (!Y_ptrs[q] || !aligned_to(Y_ptrs[q], 16) || row_off[q + 1] < row_off[q]) { g_scatter.n = 0; return B200GNN_ERR_BAD_ARG; }
    g_scatter.ptr[q] = Y_ptrs[q]; g_scatter.off[q] = row_off[q];
  }
  g_scatter.off[world] = row_off[world];
  // Y: any aligned non-null pointer passes the checks of the plain entry point; it is never dereferenced in scatter mode
  const int rc = b200gnn_spmm_csr_f32(rowptr, col, val, X, ldx, Y_ptrs[0], K, n_rows, n_src, K, reduce, bias, nullptr, chunk_rowptr,
                                      n_chunks, hub_threshold, seg_len, hub_rows, hub_segptr, n_hub, n_seg, hub_workspace, stream);
  g_scatter.n = 0;
  return rc;
}
