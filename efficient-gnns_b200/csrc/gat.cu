// Graph-attention aggregation (config 4): per-destination edge softmax + multi-head weighted neighbour sum.
//   DGL GATConv.forward  arxiv_dgl/models.py:196-217 : e = leaky_relu(el[src] + er[dst]); a = edge_softmax(e);
//                                                      out[dst,h,:] = sum_e a[e,h] * ft[src,h,:]
//   PyG GATConv (ppi_pyg/gnn.py:27-31) is the same computation with softmax_eps = 1e-16.
// CSR rows = destinations, col = sources, heads H, head width D (K = H*D floats per row).
// Forward : gat_edge_softmax (a[nnz,H]) + gat_aggregate (also used for d ft on the transposed graph through `eidx`).
// Backward: gat_bwd_rows (per destination: d a = <ft[src], d out[dst]> per head, softmax + leaky-relu backward,
//           d er, d pre[nnz,H]) + gat_segment_sum (d el over the transposed graph).
// Work split.  Row-wide kernels (aggregate, bwd_rows): one warp per chunk of rows (the SpMM chunk plan); lanes own
// vectors lane+32j of the K-float row and U edges are loaded before they are consumed, so U*NJ independent row
// gathers are in flight per warp.  Rows above hub_threshold are split into seg_len-edge segments (the SpMM hub plan):
// one CTA per segment, scheduled as the first CTAs of the same launch, 8 warps striding over groups of U edges and
// combining in warp order through shared memory into a per-segment partial; a small finalize kernel adds a hub
// row's segments in order (and, in the backward, runs the softmax pass once S is complete).  Scalar kernels (edge softmax,
// segment sum): lanes stride over a row's edges and carry all H heads at once; rows above GAT_CTA_DEG are taken
// by the whole CTA.  No atomics anywhere: every sum has a fixed order.
#include "common.cuh"

namespace b200gnn {

constexpr int GAT_THREADS = 256, GAT_WARPS = 8, GAT_MAXH = 16, GAT_MAXJ = 12;
constexpr int GAT_CTA_DEG = 512;

__device__ __forceinline__ float gsum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}
__device__ __forceinline__ float gmax(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, d));
  return v;
}
__device__ __forceinline__ float lrelu(float x, float slope) { return x > 0.f ? x : x * slope; }
__device__ __forceinline__ float vdot(const float& a, const float& b) { return a * b; }
__device__ __forceinline__ float vdot(const float2& a, const float2& b) { return fmaf(a.x, b.x, a.y * b.y); }
__device__ __forceinline__ float vdot(const float4& a, const float4& b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}

// per-head reduction over the group that owns a row: a warp (shuffles) or the 8-warp CTA (shuffles + shared memory,
// combined in warp order).  Every thread of the group gets the result.
template <bool CTA, bool MAX>
__device__ __forceinline__ void reduce_heads(float (&v)[GAT_MAXH], int H, float (*s_red)[GAT_MAXH], int lane, int warp) {
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h)
    if (h < H) v[h] = MAX ? gmax(v[h]) : gsum(v[h]);
  if (CTA) {
    if (lane == 0) {
#pragma unroll
      for (int h = 0; h < GAT_MAXH; ++h)
        if (h < H) s_red[warp][h] = v[h];
    }
    __syncthreads();
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < H) {
        float t = s_red[0][h];
        for (int w = 1; w < GAT_WARPS; ++w) t = MAX ? fmaxf(t, s_red[w][h]) : t + s_red[w][h];
        v[h] = t;
      }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- edge softmax: a[e,h]
struct GatSoftmax {
  const int32_t* rowptr; const int32_t* col; const float* el; const float* er; float* a;
  const uint8_t* keep;   // [nnz] or NULL: edges with keep == 0 are dropped (a = 0, excluded from the softmax) — edge_drop
  int64_t n_rows; int32_t H; float slope, eps;
};

template <bool CTA>
__device__ __forceinline__ void softmax_row(const GatSoftmax& p, int64_t i, int b, int e, int tid, int nt,
                                            float (*s_red)[GAT_MAXH], int lane, int warp) {
  float r[GAT_MAXH], m[GAT_MAXH], s[GAT_MAXH];
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) {
    r[h] = (p.er && h < p.H) ? __ldg(p.er + (size_t)i * p.H + h) : 0.f;
    m[h] = -INFINITY;
    s[h] = 0.f;
  }
  for (int k = b + tid; k < e; k += nt) {
    if (p.keep && !p.keep[k]) continue;
    const float* x = p.el + (size_t)__ldg(p.col + k) * p.H;
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) m[h] = fmaxf(m[h], lrelu(__ldg(x + h) + r[h], p.slope));
  }
  reduce_heads<CTA, true>(m, p.H, s_red, lane, warp);
  for (int k = b + tid; k < e; k += nt) {
    if (p.keep && !p.keep[k]) continue;
    const float* x = p.el + (size_t)__ldg(p.col + k) * p.H;
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) s[h] += expf(lrelu(__ldg(x + h) + r[h], p.slope) - m[h]);
  }
  reduce_heads<CTA, false>(s, p.H, s_red, lane, warp);
  for (int k = b + tid; k < e; k += nt) {
    const bool kept = !p.keep || p.keep[k];
    const float* x = p.el + (size_t)__ldg(p.col + k) * p.H;
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) p.a[(size_t)k * p.H + h] = kept ? expf(lrelu(__ldg(x + h) + r[h], p.slope) - m[h]) / (s[h] + p.eps) : 0.f;
  }
}

__global__ void __launch_bounds__(GAT_THREADS) gat_edge_softmax_kernel(const GatSoftmax p) {
  __shared__ float s_red[GAT_WARPS][GAT_MAXH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t r0 = (int64_t)blockIdx.x * GAT_WARPS; r0 < p.n_rows; r0 += (int64_t)gridDim.x * GAT_WARPS) {
    const int64_t i = r0 + warp;
    if (i < p.n_rows) {
      const int b = __ldg(p.rowptr + i), e = __ldg(p.rowptr + i + 1);
      if (e > b && e - b <= GAT_CTA_DEG) softmax_row<false>(p, i, b, e, lane, 32, s_red, lane, warp);
    }
    for (int w = 0; w < GAT_WARPS; ++w) {          // same decision in every thread of the CTA
      const int64_t r = r0 + w;
      if (r >= p.n_rows) break;
      const int b = __ldg(p.rowptr + r), e = __ldg(p.rowptr + r + 1);
      if (e - b > GAT_CTA_DEG) softmax_row<true>(p, r, b, e, threadIdx.x, GAT_THREADS, s_red, lane, warp);
    }
  }
}

// ---------------------------------------------------------------- out[j,h] = sum_k vals[eidx[k], h]   (d el)
struct GatSegSum {
  const int32_t* rowptr; const int32_t* eidx; const float* vals; float* out;
  int64_t n_rows; int32_t H;
};

template <bool CTA>
__device__ __forceinline__ void segsum_row(const GatSegSum& p, int64_t j, int b, int e, int tid, int nt,
                                           float (*s_red)[GAT_MAXH], int lane, int warp) {
  float s[GAT_MAXH];
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) s[h] = 0.f;
  for (int k = b + tid; k < e; k += nt) {
    const float* x = p.vals + (size_t)(p.eidx ? __ldg(p.eidx + k) : k) * p.H;
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) s[h] += __ldg(x + h);
  }
  reduce_heads<CTA, false>(s, p.H, s_red, lane, warp);
  if (tid == 0) {
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) p.out[(size_t)j * p.H + h] = s[h];
  }
}

__global__ void __launch_bounds__(GAT_THREADS) gat_segment_sum_kernel(const GatSegSum p) {
  __shared__ float s_red[GAT_WARPS][GAT_MAXH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t r0 = (int64_t)blockIdx.x * GAT_WARPS; r0 < p.n_rows; r0 += (int64_t)gridDim.x * GAT_WARPS) {
    const int64_t j = r0 + warp;
    if (j < p.n_rows) {
      const int b = __ldg(p.rowptr + j), e = __ldg(p.rowptr + j + 1);
      if (e - b <= GAT_CTA_DEG) segsum_row<false>(p, j, b, e, lane, 32, s_red, lane, warp);
    }
    for (int w = 0; w < GAT_WARPS; ++w) {
      const int64_t r = r0 + w;
      if (r >= p.n_rows) break;
      const int b = __ldg(p.rowptr + r), e = __ldg(p.rowptr + r + 1);
      if (e - b > GAT_CTA_DEG) segsum_row<true>(p, r, b, e, threadIdx.x, GAT_THREADS, s_red, lane, warp);
    }
  }
}

// ---------------------------------------------------------------- aggregate
struct GatAgg {
  const int32_t* rowptr; const int32_t* col; const int32_t* eidx;   // eidx: position of edge k in a[] (NULL: k)
  const int32_t* chunk_rowptr; const int32_t* hub_rows; const int32_t* hub_segptr;
  const float* a; const float* ft; float* out; float* ws;   // ws: [n_seg, K] hub-segment partials
  int64_t ldf, ldo;
  int32_t n_chunks, n_hub, n_seg, seg_len, hub_threshold, H, D, K;
};

// segment s of the hub plan -> (hub index, edge range)
__device__ __forceinline__ void hub_segment(const int32_t* rowptr, const int32_t* hub_rows, const int32_t* hub_segptr,
                                            int n_hub, int seg_len, int s, int& r, int& b, int& e) {
  int lo = 0, hi = n_hub;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(hub_segptr + mid) <= s) lo = mid; else hi = mid;
  }
  r = __ldg(hub_rows + lo);
  b = __ldg(rowptr + r) + (s - __ldg(hub_segptr + lo)) * seg_len;
  e = min(__ldg(rowptr + r + 1), b + seg_len);
}

// lane handles vectors v = lane + 32*j (j < NJ) of width W; head of vector v = (v*W)/D.  The group's warps take
// groups of U consecutive edges: warp `first` of `stride` warps starts at beg + first*U.
// SS: the coefficient of edge k is a[k,h] * src_scale[col[k]] (the fused layer's out_deg^-1/2, or 1 when the vector is absent).
template <typename V, int NJ, int U, bool SS = false>
__device__ __forceinline__ void agg_edges(const GatAgg& p, int beg, int end, int first, int stride, int lane, int nvec,
                                          const int (&head)[NJ], V (&acc)[NJ], const float* src_scale = nullptr) {
  constexpr int W = VecTraits<V>::W;
  const V* F = reinterpret_cast<const V*>(p.ft);
  const size_t ldv = (size_t)(p.ldf / W);
  for (int k0 = beg + first * U; k0 < end; k0 += stride * U) {
    V x[U][NJ];
    float w[U][NJ];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int kk = k0 + u;
      if (kk < end) {
        const int c = __ldg(p.col + kk);
        const V* row = F + (size_t)c * ldv + lane;
        const float* ak = p.a + (size_t)(p.eidx ? __ldg(p.eidx + kk) : kk) * p.H;
        float ss = 1.f;
        if (SS) ss = src_scale ? __ldg(src_scale + c) : 1.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if (lane + 32 * j < nvec) { x[u][j] = vldg(row + 32 * j); w[u][j] = SS ? __ldg(ak + head[j]) * ss : __ldg(ak + head[j]); }
          else { vzero(x[u][j]); w[u][j] = 0.f; }
        }
      } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) { vzero(x[u][j]); w[u][j] = 0.f; }
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int j = 0; j < NJ; ++j) vfma(acc[j], w[u][j], x[u][j]);
  }
}

template <typename V, int NJ, int U>
__global__ void __launch_bounds__(GAT_THREADS) gat_aggregate_kernel(const GatAgg p) {
  constexpr int W = VecTraits<V>::W;
  extern __shared__ float s_row[];   // K floats (hub-segment CTAs)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = p.K / W;
  int head[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) head[j] = ((lane + 32 * j) * W) / p.D;
  if ((int)blockIdx.x < p.n_seg) {     // hub segment: warps stride over groups of U edges, combined in warp order
    int r, b, e;
    hub_segment(p.rowptr, p.hub_rows, p.hub_segptr, p.n_hub, p.seg_len, blockIdx.x, r, b, e);
    V acc[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) vzero(acc[j]);
    agg_edges<V, NJ, U>(p, b, e, warp, GAT_WARPS, lane, nvec, head, acc);
    for (int i = threadIdx.x; i < p.K; i += GAT_THREADS) s_row[i] = 0.f;
    __syncthreads();
    V* sv = reinterpret_cast<V*>(s_row);
    for (int w = 0; w < GAT_WARPS; ++w) {
      if (warp == w) {
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (lane + 32 * j < nvec) { V t = sv[lane + 32 * j]; vadd(t, acc[j]); sv[lane + 32 * j] = t; }
      }
      __syncthreads();
    }
    for (int i = threadIdx.x; i < p.K; i += GAT_THREADS) p.ws[(size_t)blockIdx.x * p.K + i] = s_row[i];
    return;
  }
  V* O = reinterpret_cast<V*>(p.out);
  const size_t ldov = (size_t)(p.ldo / W);
  const int chunk = (blockIdx.x - p.n_seg) * GAT_WARPS + warp;
  if (chunk >= p.n_chunks) return;
  const int r0 = __ldg(p.chunk_rowptr + chunk), r1 = __ldg(p.chunk_rowptr + chunk + 1);
  for (int r = r0; r < r1; ++r) {
    const int b = __ldg(p.rowptr + r), e = __ldg(p.rowptr + r + 1);
    if (e - b > p.hub_threshold) continue;
    V acc[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) vzero(acc[j]);
    agg_edges<V, NJ, U>(p, b, e, 0, 1, lane, nvec, head, acc);
#pragma unroll
    for (int j = 0; j < NJ; ++j)
      if (lane + 32 * j < nvec) O[(size_t)r * ldov + lane + 32 * j] = acc[j];
  }
}

// out[hub row] = its segments' partials added in segment order
__global__ void __launch_bounds__(GAT_THREADS) gat_hub_finalize_kernel(const int32_t* __restrict__ hub_rows,
                                                                       const int32_t* __restrict__ hub_segptr,
                                                                       const float* __restrict__ ws, float* __restrict__ out,
                                                                       int64_t ldo, int K) {
  const int r = __ldg(hub_rows + blockIdx.x);
  const int q0 = __ldg(hub_segptr + blockIdx.x), q1 = __ldg(hub_segptr + blockIdx.x + 1);
  for (int i = threadIdx.x; i < K; i += GAT_THREADS) {
    float t = 0.f;
    for (int q = q0; q < q1; ++q) t += ws[(size_t)q * K + i];
    out[(size_t)r * ldo + i] = t;
  }
}

// ---------------------------------------------------------------- backward, per destination row
struct GatBwd {
  const int32_t* rowptr; const int32_t* col; const float* a; const float* ft; const float* dout;
  const float* el; const float* er;
  const float* scale;   // [nnz,H] or NULL: attention dropout, the aggregation used a*scale (scale = keep/(1-p)); d a = d(a*scale)*scale
  float* dpre;   // [nnz,H]  out: d loss / d (el[src]+er[dst])
  float* der;    // [n_rows,H] out (may be NULL when there is no er)
  const int32_t* chunk_rowptr; const int32_t* hub_rows; const int32_t* hub_segptr;
  float* ws;     // [n_seg, H] hub-segment partials of S
  int64_t ldf, ldd, n_rows;
  int32_t n_chunks, n_hub, n_seg, seg_len, hub_threshold;
  int32_t H, D, K;
  float slope;
};

// phase 1 over a group's share of the row's edges: d a[k,h] = <ft[src,h,:], dout[i,h,:]> staged in dpre, and the
// group-local S[h] += a[k,h] * d a[k,h] (same value on every lane).  Per-head sums over the lanes: SEG = false
// reduces one head at a time over the whole warp (H * 5 shuffles per edge; right for few wide heads, e.g. the
// teacher's 3 x 250); SEG = true needs D/W a power of two <= 32, so a head is an aligned group of lph lanes of one
// vector index j, and a segmented xor-reduction costs NJ * log2(lph) shuffles (many narrow heads).
template <typename V, int NJ, int U, bool SEG>
__device__ __forceinline__ void bwd_edges(const GatBwd& p, int beg, int end, int first, int stride, int lane, int nvec,
                                          const V (&g)[NJ], const int (&head)[NJ], float (&S)[GAT_MAXH]) {
  constexpr int W = VecTraits<V>::W;
  const V* F = reinterpret_cast<const V*>(p.ft);
  const size_t ldv = (size_t)(p.ldf / W);
  const int lph = p.D / W;
  float Sj[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) Sj[j] = 0.f;
  for (int k0 = beg + first * U; k0 < end; k0 += stride * U) {
    V x[U][NJ];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int kk = k0 + u;
      if (kk < end) {
        const V* row = F + (size_t)__ldg(p.col + kk) * ldv + lane;
#pragma unroll
        for (int j = 0; j < NJ; ++j) {
          if (lane + 32 * j < nvec) x[u][j] = vldg(row + 32 * j);
          else vzero(x[u][j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < NJ; ++j) vzero(x[u][j]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int kk = k0 + u;
      if (kk < end) {
        float d[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) d[j] = vdot(x[u][j], g[j]);
        if (SEG) {
#pragma unroll
          for (int j = 0; j < NJ; ++j) {
#pragma unroll
            for (int o = 1; o < 32; o <<= 1)
              if (o < lph) d[j] += __shfl_xor_sync(FULL_MASK, d[j], o);
            if (lane + 32 * j < nvec) {
              const size_t o = (size_t)kk * p.H + head[j];
              const float da = p.scale ? d[j] * __ldg(p.scale + o) : d[j];
              if ((lane & (lph - 1)) == 0) p.dpre[o] = da;
              Sj[j] = fmaf(__ldg(p.a + o), da, Sj[j]);
            }
          }
        } else {
#pragma unroll
          for (int h = 0; h < GAT_MAXH; ++h)
            if (h < p.H) {
              float part = 0.f;
#pragma unroll
              for (int j = 0; j < NJ; ++j) part += (head[j] == h) ? d[j] : 0.f;
              const size_t o = (size_t)kk * p.H + h;
              const float da = p.scale ? gsum(part) * __ldg(p.scale + o) : gsum(part);
              if (lane == 0) p.dpre[o] = da;
              S[h] = fmaf(__ldg(p.a + o), da, S[h]);
            }
        }
      }
    }
  }
  if (SEG) {   // head h lives in vector index v = h*lph: lane v%32 of j = v/32 holds its S
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) {
        const int v = h * lph;
        float val = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) val = (j == (v >> 5)) ? Sj[j] : val;
        S[h] = __shfl_sync(FULL_MASK, val, v & 31);
      }
  }
}

// phase 2: d e = a (d a - S);  d pre = d e * leaky'(pre);  dr[h] = this thread's share of d er[i,h]
__device__ __forceinline__ void bwd_phase2(const GatBwd& p, int64_t i, int b, int e, int tid, int nt,
                                           const float (&S)[GAT_MAXH], float (&dr)[GAT_MAXH]) {
  float r[GAT_MAXH];
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) {
    r[h] = (p.er && h < p.H) ? __ldg(p.er + (size_t)i * p.H + h) : 0.f;
    dr[h] = 0.f;
  }
  for (int k = b + tid; k < e; k += nt) {
    const float* x = p.el + (size_t)__ldg(p.col + k) * p.H;
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) {
        const size_t o = (size_t)k * p.H + h;
        const float de = p.a[o] * (p.dpre[o] - S[h]);
        const float dp = (__ldg(x + h) + r[h]) > 0.f ? de : de * p.slope;
        p.dpre[o] = dp;
        dr[h] += dp;
      }
  }
}

template <typename V, int NJ, int U, bool SEG>
__global__ void __launch_bounds__(GAT_THREADS) gat_bwd_rows_kernel(const GatBwd p) {
  constexpr int W = VecTraits<V>::W;
  __shared__ float s_S[GAT_WARPS][GAT_MAXH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = p.K / W;
  const V* G = reinterpret_cast<const V*>(p.dout);
  const size_t lddv = (size_t)(p.ldd / W);
  int head[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) head[j] = ((lane + 32 * j) * W) / p.D;
  V g[NJ];
  float S[GAT_MAXH], dr[GAT_MAXH];
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) S[h] = 0.f;
  if ((int)blockIdx.x < p.n_seg) {     // hub segment: phase 1 only, partial S to the workspace
    int i, b, e;
    hub_segment(p.rowptr, p.hub_rows, p.hub_segptr, p.n_hub, p.seg_len, blockIdx.x, i, b, e);
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (lane + 32 * j < nvec) g[j] = vldg(G + (size_t)i * lddv + lane + 32 * j);
      else vzero(g[j]);
    }
    bwd_edges<V, NJ, U, SEG>(p, b, e, warp, GAT_WARPS, lane, nvec, g, head, S);
    if (lane == 0) {
#pragma unroll
      for (int h = 0; h < GAT_MAXH; ++h)
        if (h < p.H) s_S[warp][h] = S[h];
    }
    __syncthreads();
    if (threadIdx.x < p.H) {
      float t = 0.f;
      for (int w = 0; w < GAT_WARPS; ++w) t += s_S[w][threadIdx.x];
      p.ws[(size_t)blockIdx.x * p.H + threadIdx.x] = t;
    }
    return;
  }
  const int chunk = (blockIdx.x - p.n_seg) * GAT_WARPS + warp;
  if (chunk >= p.n_chunks) return;
  const int r0 = __ldg(p.chunk_rowptr + chunk), r1 = __ldg(p.chunk_rowptr + chunk + 1);
  for (int i = r0; i < r1; ++i) {
    const int b = __ldg(p.rowptr + i), e = __ldg(p.rowptr + i + 1);
    if (e - b > p.hub_threshold) continue;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      if (lane + 32 * j < nvec) g[j] = vldg(G + (size_t)i * lddv + lane + 32 * j);
      else vzero(g[j]);
    }
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h) S[h] = 0.f;
    bwd_edges<V, NJ, U, SEG>(p, b, e, 0, 1, lane, nvec, g, head, S);
    __syncwarp();                                   // lane 0's staged d a is read by every lane below
    bwd_phase2(p, i, b, e, lane, 32, S, dr);
    if (p.der) {
#pragma unroll
      for (int h = 0; h < GAT_MAXH; ++h)
        if (h < p.H) { const float t = gsum(dr[h]); if (lane == 0) p.der[(size_t)i * p.H + h] = t; }
    }
  }
}

// hub rows, after their segments: S = sum of the segment partials (segment order), then phase 2 over the whole row
__global__ void __launch_bounds__(GAT_THREADS) gat_bwd_hub_finalize_kernel(const GatBwd p) {
  __shared__ float s_S[GAT_WARPS][GAT_MAXH];
  __shared__ float s_tot[GAT_MAXH];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t i = __ldg(p.hub_rows + blockIdx.x);
  const int b = __ldg(p.rowptr + i), e = __ldg(p.rowptr + i + 1);
  if (threadIdx.x < p.H) {
    float t = 0.f;
    for (int q = __ldg(p.hub_segptr + blockIdx.x); q < __ldg(p.hub_segptr + blockIdx.x + 1); ++q)
      t += p.ws[(size_t)q * p.H + threadIdx.x];
    s_tot[threadIdx.x] = t;
  }
  __syncthreads();
  float S[GAT_MAXH], dr[GAT_MAXH];
#pragma unroll
  for (int h = 0; h < GAT_MAXH; ++h) S[h] = h < p.H ? s_tot[h] : 0.f;
  bwd_phase2(p, i, b, e, threadIdx.x, GAT_THREADS, S, dr);
  if (p.der) {
#pragma unroll
    for (int h = 0; h < GAT_MAXH; ++h)
      if (h < p.H) { const float t = gsum(dr[h]); if (lane == 0) s_S[warp][h] = t; }
    __syncthreads();
    if (threadIdx.x < p.H) {
      float t = 0.f;
      for (int w = 0; w < GAT_WARPS; ++w) t += s_S[w][threadIdx.x];
      p.der[(size_t)i * p.H + threadIdx.x] = t;
    }
  }
}

// ---------------------------------------------------------------- aggregate with the layer's epilogue
// The fused GAT layer (engine_gat.py): out[i,:] = row_scale[i] * sum_k a[k,h] src_scale[col[k]] ft[col[k],h,:] + res[i,:] + bias,
// and per CTA the (sum, sum of squares) of its output rows in the [slots][2][K] layout b200gnn_bn_finalize_f32 reads.
// Same decomposition and summation order as gat_aggregate_kernel: with every epilogue operand absent the output is its
// output bit for bit (a * 1.f is a).
struct GatEpi {
  const float* src_scale; const float* row_scale; const float* res; const float* bias; float* stat;
  float* act;                    // ELU instantiations only: elu(out) is also stored here, row pitch lda
  int64_t ldr, lda; int32_t n_main;   // n_main: CTAs of the chunk part of the launch = first hub slot
};

template <typename V>
__device__ __forceinline__ V epi_row(const GatEpi& q, V y, int64_t r, int v) {
  constexpr int W = VecTraits<V>::W;
  if (q.row_scale) { V z; vzero(z); vfma(z, __ldg(q.row_scale + r), y); y = z; }
  if (q.res) vadd(y, vldg(reinterpret_cast<const V*>(q.res + (size_t)r * q.ldr) + v));
  if (q.bias) vadd(y, vldg(reinterpret_cast<const V*>(q.bias) + v));
  (void)W;
  return y;
}

// F.elu with alpha 1 as torch computes it: z > 0 ? z : expm1(z)
__device__ __forceinline__ float elu1(float z) { return z > 0.f ? z : expm1f(z); }
__device__ __forceinline__ float velu(float z) { return elu1(z); }
__device__ __forceinline__ float2 velu(float2 z) { return make_float2(elu1(z.x), elu1(z.y)); }
__device__ __forceinline__ float4 velu(float4 z) { return make_float4(elu1(z.x), elu1(z.y), elu1(z.z), elu1(z.w)); }

template <typename V, int NJ, int U, bool ELU = false>
__global__ void __launch_bounds__(GAT_THREADS) gat_aggregate_epi_kernel(const GatAgg p, const GatEpi q) {
  constexpr int W = VecTraits<V>::W;
  extern __shared__ float s_row[];   // K floats (hub-segment CTAs), 2K floats (statistics of the chunk CTAs)
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nvec = p.K / W;
  int head[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) head[j] = ((lane + 32 * j) * W) / p.D;
  if ((int)blockIdx.x < p.n_seg) {
    int r, b, e;
    hub_segment(p.rowptr, p.hub_rows, p.hub_segptr, p.n_hub, p.seg_len, blockIdx.x, r, b, e);
    V acc[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) vzero(acc[j]);
    agg_edges<V, NJ, U, true>(p, b, e, warp, GAT_WARPS, lane, nvec, head, acc, q.src_scale);
    for (int i = threadIdx.x; i < p.K; i += GAT_THREADS) s_row[i] = 0.f;
    __syncthreads();
    V* sv = reinterpret_cast<V*>(s_row);
    for (int w = 0; w < GAT_WARPS; ++w) {
      if (warp == w) {
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (lane + 32 * j < nvec) { V t = sv[lane + 32 * j]; vadd(t, acc[j]); sv[lane + 32 * j] = t; }
      }
      __syncthreads();
    }
    for (int i = threadIdx.x; i < p.K; i += GAT_THREADS) p.ws[(size_t)blockIdx.x * p.K + i] = s_row[i];
    return;
  }
  V* O = reinterpret_cast<V*>(p.out);
  const size_t ldov = (size_t)(p.ldo / W);
  const int cta = blockIdx.x - p.n_seg;
  const int chunk = cta * GAT_WARPS + warp;
  V ssum[NJ], ssq[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) { vzero(ssum[j]); vzero(ssq[j]); }
  if (chunk < p.n_chunks) {
    const int r0 = __ldg(p.chunk_rowptr + chunk), r1 = __ldg(p.chunk_rowptr + chunk + 1);
    for (int r = r0; r < r1; ++r) {
      const int b = __ldg(p.rowptr + r), e = __ldg(p.rowptr + r + 1);
      if (e - b > p.hub_threshold) continue;
      V acc[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) vzero(acc[j]);
      agg_edges<V, NJ, U, true>(p, b, e, 0, 1, lane, nvec, head, acc, q.src_scale);
#pragma unroll
      for (int j = 0; j < NJ; ++j)
        if (lane + 32 * j < nvec) {
          const V y = epi_row<V>(q, acc[j], r, lane + 32 * j);
          O[(size_t)r * ldov + lane + 32 * j] = y;
          if (ELU) reinterpret_cast<V*>(q.act)[(size_t)r * (size_t)(q.lda / W) + lane + 32 * j] = velu(y);
          if (q.stat) vstat(ssum[j], ssq[j], y);
        }
    }
  }
  if (q.stat) {     // the CTA's warps combine in warp order; every slot is written on every launch
    for (int i = threadIdx.x; i < 2 * p.K; i += GAT_THREADS) s_row[i] = 0.f;
    __syncthreads();
    V* ss = reinterpret_cast<V*>(s_row);
    V* sq = reinterpret_cast<V*>(s_row + p.K);
    for (int w = 0; w < GAT_WARPS; ++w) {
      if (warp == w) {
#pragma unroll
        for (int j = 0; j < NJ; ++j)
          if (lane + 32 * j < nvec) {
            V t = ss[lane + 32 * j]; vadd(t, ssum[j]); ss[lane + 32 * j] = t;
            V u = sq[lane + 32 * j]; vadd(u, ssq[j]); sq[lane + 32 * j] = u;
          }
      }
      __syncthreads();
    }
    float* out = q.stat + (size_t)cta * 2 * p.K;
    for (int i = threadIdx.x; i < 2 * p.K; i += GAT_THREADS) out[i] = s_row[i];
  }
}

template <bool ELU = false>
__global__ void __launch_bounds__(GAT_THREADS) gat_hub_finalize_epi_kernel(const int32_t* __restrict__ hub_rows,
                                                                           const int32_t* __restrict__ hub_segptr,
                                                                           const float* __restrict__ ws, float* __restrict__ out,
                                                                           int64_t ldo, int K, const GatEpi q) {
  const int r = __ldg(hub_rows + blockIdx.x);
  const int q0 = __ldg(hub_segptr + blockIdx.x), q1 = __ldg(hub_segptr + blockIdx.x + 1);
  float* stat = q.stat ? q.stat + (size_t)(q.n_main + blockIdx.x) * 2 * K : nullptr;
  for (int i = threadIdx.x; i < K; i += GAT_THREADS) {
    float t = 0.f;
    for (int s = q0; s < q1; ++s) t += ws[(size_t)s * K + i];
    t = epi_row<float>(q, t, r, i);
    out[(size_t)r * ldo + i] = t;
    if (ELU) q.act[(size_t)r * q.lda + i] = elu1(t);
    if (stat) { stat[i] = t; stat[K + i] = t * t; }
  }
}

// ---------------------------------------------------------------- attention scores
// el[n,h] = src_scale[n] * <ft[n,h,:], attn_l[h,:]>,  er[n,h] = <ft[n,h,:], attn_r[h,:]>   (one warp per node; lanes
// stride over the head and combine by the xor butterfly: one fixed order)
struct GatScores {
  const float* ft; const float* attn_l; const float* attn_r; const float* src_scale; float* el; float* er;
  int64_t ldf, n_rows; int32_t H, D;
};

__global__ void __launch_bounds__(GAT_THREADS) gat_scores_kernel(const GatScores p) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t n = (int64_t)blockIdx.x * GAT_WARPS + warp; n < p.n_rows; n += (int64_t)gridDim.x * GAT_WARPS) {
    const float* row = p.ft + (size_t)n * p.ldf;
    const float sc = p.src_scale ? __ldg(p.src_scale + n) : 1.f;
    for (int h = 0; h < p.H; ++h) {
      float sl = 0.f, sr = 0.f;
      for (int d = lane; d < p.D; d += 32) {
        const float f = __ldg(row + h * p.D + d);
        sl = fmaf(f, __ldg(p.attn_l + h * p.D + d), sl);
        if (p.attn_r) sr = fmaf(f, __ldg(p.attn_r + h * p.D + d), sr);
      }
      sl = gsum(sl);
      if (p.attn_r) sr = gsum(sr);
      if (lane == 0) {
        p.el[(size_t)n * p.H + h] = p.src_scale ? sl * sc : sl;
        if (p.attn_r) p.er[(size_t)n * p.H + h] = sr;
      }
    }
  }
}

// backward: dft[n,h,:] += del[n,h] src_scale[n] attn_l[h,:] + der[n,h] attn_r[h,:] in place, and per CTA (a contiguous
// block of rows, added in row order) the partial sums of d attn_l / d attn_r; a second kernel adds the slots in order.
constexpr int GAT_SB_MAXJ = 6;   // columns per thread: K <= 1536
struct GatScoresBwd {
  const float* ft; const float* attn_l; const float* attn_r; const float* src_scale; const float* del; const float* der;
  float* dft; float* partial;   // [slots][2][K]
  int64_t ldf, ldd, n_rows; int32_t H, D, K, rows_per_cta;
};

__global__ void __launch_bounds__(GAT_THREADS) gat_scores_bwd_kernel(const GatScoresBwd p) {
  float al[GAT_SB_MAXJ], ar[GAT_SB_MAXJ], accl[GAT_SB_MAXJ], accr[GAT_SB_MAXJ];
  int hd[GAT_SB_MAXJ];
#pragma unroll
  for (int j = 0; j < GAT_SB_MAXJ; ++j) {
    const int k = threadIdx.x + GAT_THREADS * j;
    hd[j] = k < p.K ? k / p.D : 0;
    al[j] = k < p.K ? __ldg(p.attn_l + k) : 0.f;
    ar[j] = (k < p.K && p.attn_r) ? __ldg(p.attn_r + k) : 0.f;
    accl[j] = accr[j] = 0.f;
  }
  const int64_t r0 = (int64_t)blockIdx.x * p.rows_per_cta;
  const int64_t r1 = r0 + p.rows_per_cta < p.n_rows ? r0 + p.rows_per_cta : p.n_rows;
  for (int64_t n = r0; n < r1; ++n) {
    const float sc = p.src_scale ? __ldg(p.src_scale + n) : 1.f;
#pragma unroll
    for (int j = 0; j < GAT_SB_MAXJ; ++j) {
      const int k = threadIdx.x + GAT_THREADS * j;
      if (k < p.K) {
        const float gl = __ldg(p.del + (size_t)n * p.H + hd[j]) * sc;
        const float f = __ldg(p.ft + (size_t)n * p.ldf + k);
        float g = fmaf(gl, al[j], p.dft[(size_t)n * p.ldd + k]);
        accl[j] = fmaf(gl, f, accl[j]);
        if (p.attn_r) {
          const float gr = __ldg(p.der + (size_t)n * p.H + hd[j]);
          g = fmaf(gr, ar[j], g);
          accr[j] = fmaf(gr, f, accr[j]);
        }
        p.dft[(size_t)n * p.ldd + k] = g;
      }
    }
  }
  float* out = p.partial + (size_t)blockIdx.x * 2 * p.K;
#pragma unroll
  for (int j = 0; j < GAT_SB_MAXJ; ++j) {
    const int k = threadIdx.x + GAT_THREADS * j;
    if (k < p.K) { out[k] = accl[j]; out[p.K + k] = accr[j]; }
  }
}

__global__ void __launch_bounds__(GAT_THREADS) gat_scores_bwd_finalize_kernel(const float* __restrict__ partial, int slots, int K,
                                                                              float* __restrict__ d_attn_l,
                                                                              float* __restrict__ d_attn_r) {
  const int i = blockIdx.x * GAT_THREADS + threadIdx.x;
  if (i >= 2 * K) return;
  float* dst = i < K ? d_attn_l + i : (d_attn_r ? d_attn_r + (i - K) : nullptr);
  if (!dst) return;
  float t = 0.f;
  for (int s = 0; s < slots; ++s) t += partial[(size_t)s * 2 * K + i];
  *dst = t;
}

static inline int rows_grid(int64_t n) {
  int64_t g = (n + GAT_WARPS - 1) / GAT_WARPS;
  if (g > 132 * 16) g = 132 * 16;
  return (int)(g < 1 ? 1 : g);
}

template <typename V, int NJ, int U>
static int launch_agg_nj(const GatAgg& p, cudaStream_t st) {
  int rc;
  const int grid = p.n_seg + (p.n_chunks + GAT_WARPS - 1) / GAT_WARPS;
  gat_aggregate_kernel<V, NJ, U><<<grid, GAT_THREADS, p.n_seg > 0 ? p.K * sizeof(float) : 0, st>>>(p);
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    gat_hub_finalize_kernel<<<p.n_hub, GAT_THREADS, 0, st>>>(p.hub_rows, p.hub_segptr, p.ws, p.out, p.ldo, p.K);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}

template <typename V, int NJ, int U, bool ELU>
static int launch_agg_epi_nj(const GatAgg& p, const GatEpi& q0, cudaStream_t st) {
  int rc;
  GatEpi q = q0;
  q.n_main = (p.n_chunks + GAT_WARPS - 1) / GAT_WARPS;
  const int grid = p.n_seg + q.n_main;
  const size_t smem = (q.stat ? 2 * p.K : (p.n_seg > 0 ? p.K : 0)) * sizeof(float);
  gat_aggregate_epi_kernel<V, NJ, U, ELU><<<grid, GAT_THREADS, smem, st>>>(p, q);
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    gat_hub_finalize_epi_kernel<ELU><<<p.n_hub, GAT_THREADS, 0, st>>>(p.hub_rows, p.hub_segptr, p.ws, p.out, p.ldo, p.K, q);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}
template <typename V, bool ELU = false>
static int launch_agg_epi(const GatAgg& p, const GatEpi& q, cudaStream_t st) {   // the (NJ, U) choice of launch_agg
  constexpr int W = VecTraits<V>::W;
  const int nj = (p.K / W + 31) / 32;
  if constexpr (W == 4) {
    if (nj <= 1) return launch_agg_epi_nj<V, 1, 8, ELU>(p, q, st);
    if (nj <= 2) return launch_agg_epi_nj<V, 2, 4, ELU>(p, q, st);
  }
  if (nj <= 4) return launch_agg_epi_nj<V, 4, 2, ELU>(p, q, st);
  if constexpr (W == 4) {
    if (nj <= 8) return launch_agg_epi_nj<V, 8, 1, ELU>(p, q, st);
  }
  return launch_agg_epi_nj<V, GAT_MAXJ, 1, ELU>(p, q, st);
}

template <typename V, int NJ, int U, bool SEG>
static int launch_bwd_seg(const GatBwd& p, cudaStream_t st) {
  int rc;
  const int grid = p.n_seg + (p.n_chunks + GAT_WARPS - 1) / GAT_WARPS;
  gat_bwd_rows_kernel<V, NJ, U, SEG><<<grid, GAT_THREADS, 0, st>>>(p);
  if ((rc = check_launch())) return rc;
  if (p.n_hub > 0) {
    gat_bwd_hub_finalize_kernel<<<p.n_hub, GAT_THREADS, 0, st>>>(p);
    if ((rc = check_launch())) return rc;
  }
  return B200GNN_OK;
}
template <typename V, int NJ, int U>
static int launch_bwd_nj(const GatBwd& p, cudaStream_t st) {
  constexpr int W = VecTraits<V>::W;
  if constexpr (W == 4) {   // segmented reduction when it is cheaper than H whole-warp sums
    const int lph = p.D / W, nj = (p.K / W + 31) / 32;
    int lg = 0;
    while ((1 << lg) < lph) ++lg;
    if (lph <= 32 && (lph & (lph - 1)) == 0 && nj * lg < p.H * 5) return launch_bwd_seg<V, NJ, U, true>(p, st);
  }
  return launch_bwd_seg<V, NJ, U, false>(p, st);
}

// vectors per lane -> (NJ, U): keep about 8 row vectors in flight per lane; the narrow vector types only get the
// two widest shapes (they are the odd-width fallbacks)
template <typename V>
static int launch_agg(const GatAgg& p, cudaStream_t st) {
  constexpr int W = VecTraits<V>::W;
  const int nj = (p.K / W + 31) / 32;
  if constexpr (W == 4) {
    if (nj <= 1) return launch_agg_nj<V, 1, 8>(p, st);
    if (nj <= 2) return launch_agg_nj<V, 2, 4>(p, st);
  }
  if (nj <= 4) return launch_agg_nj<V, 4, 2>(p, st);
  if constexpr (W == 4) {
    if (nj <= 8) return launch_agg_nj<V, 8, 1>(p, st);
  }
  return launch_agg_nj<V, GAT_MAXJ, 1>(p, st);
}
template <typename V>
static int launch_bwd(const GatBwd& p, cudaStream_t st) {
  constexpr int W = VecTraits<V>::W;
  const int nj = (p.K / W + 31) / 32;
  if constexpr (W == 4) {
    if (nj <= 1) return launch_bwd_nj<V, 1, 8>(p, st);
    if (nj <= 2) return launch_bwd_nj<V, 2, 4>(p, st);
  }
  if (nj <= 4) return launch_bwd_nj<V, 4, 2>(p, st);
  if constexpr (W == 4) {
    if (nj <= 8) return launch_bwd_nj<V, 8, 1>(p, st);
  }
  return launch_bwd_nj<V, GAT_MAXJ, 1>(p, st);
}

}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_gat_edge_softmax_f32(const int32_t* rowptr, const int32_t* col, const float* el, const float* er,
                                            int64_t n_rows, int64_t H, float negative_slope, float softmax_eps, float* a,
                                            const uint8_t* edge_keep, void* stream) {
  if (!rowptr || !el || !a || n_rows < 0 || H <= 0 || H > GAT_MAXH) return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  GatSoftmax p;
  p.rowptr = rowptr; p.col = col; p.el = el; p.er = er; p.a = a; p.keep = edge_keep; p.n_rows = n_rows; p.H = (int32_t)H;
  p.slope = negative_slope; p.eps = softmax_eps;
  gat_edge_softmax_kernel<<<rows_grid(n_rows), GAT_THREADS, 0, (cudaStream_t)stream>>>(p);
  return check_launch();
}

extern "C" int b200gnn_gat_aggregate_f32(const int32_t* rowptr, const int32_t* col, const int32_t* eidx, const float* a,
                                         const float* ft, int64_t ldf, float* out, int64_t ldo, int64_t n_rows, int64_t H,
                                         int64_t D, const int32_t* chunk_rowptr, int64_t n_chunks, int32_t hub_threshold,
                                         int32_t seg_len, const int32_t* hub_rows, const int32_t* hub_segptr, int64_t n_hub,
                                         int64_t n_seg, float* hub_workspace, void* stream) {
  const int64_t K = H * D;
  if (!rowptr || !a || !ft || !out || n_rows < 0 || H <= 0 || D <= 0 || H > GAT_MAXH || ldf < K || ldo < K || !chunk_rowptr ||
      n_chunks < 0 || n_hub < 0 || n_seg < n_hub ||
      (n_hub > 0 && (!hub_rows || !hub_segptr || !hub_workspace || seg_len <= 0)))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0 || n_chunks == 0) return B200GNN_OK;
  GatAgg p;
  p.rowptr = rowptr; p.col = col; p.eidx = eidx; p.chunk_rowptr = chunk_rowptr; p.hub_rows = hub_rows;
  p.hub_segptr = hub_segptr; p.ws = hub_workspace;
  p.a = a; p.ft = ft; p.out = out; p.ldf = ldf; p.ldo = ldo;
  p.n_chunks = (int32_t)n_chunks; p.n_hub = (int32_t)n_hub; p.n_seg = (int32_t)(n_hub > 0 ? n_seg : 0); p.seg_len = seg_len;
  p.hub_threshold = hub_threshold;
  p.H = (int32_t)H; p.D = (int32_t)D; p.K = (int32_t)K;
  cudaStream_t st = (cudaStream_t)stream;
  // a vector must not straddle two heads: D % W == 0
  if (D % 4 == 0 && ldf % 4 == 0 && ldo % 4 == 0 && aligned_to(ft, 16) && aligned_to(out, 16) && K <= 4 * 32 * GAT_MAXJ)
    return launch_agg<float4>(p, st);
  if (D % 2 == 0 && ldf % 2 == 0 && ldo % 2 == 0 && aligned_to(ft, 8) && aligned_to(out, 8) && K <= 2 * 32 * GAT_MAXJ)
    return launch_agg<float2>(p, st);
  if (K <= 32 * GAT_MAXJ) return launch_agg<float>(p, st);
  return B200GNN_ERR_UNSUPPORTED;
}

extern "C" int b200gnn_gat_bwd_rows_f32(const int32_t* rowptr, const int32_t* col, const float* a, const float* ft, int64_t ldf,
                                        const float* dout, int64_t ldd, const float* el, const float* er, int64_t n_rows,
                                        int64_t H, int64_t D, float negative_slope, float* dpre, float* der,
                                        const int32_t* chunk_rowptr, int64_t n_chunks, int32_t hub_threshold,
                                        int32_t seg_len, const int32_t* hub_rows, const int32_t* hub_segptr, int64_t n_hub,
                                        int64_t n_seg, float* hub_workspace, const float* attn_scale, void* stream) {
  const int64_t K = H * D;
  if (!rowptr || !a || !ft || !dout || !el || !dpre || n_rows < 0 || H <= 0 || D <= 0 || H > GAT_MAXH || ldf < K || ldd < K ||
      !chunk_rowptr || n_chunks < 0 || n_hub < 0 || n_seg < n_hub ||
      (n_hub > 0 && (!hub_rows || !hub_segptr || !hub_workspace || seg_len <= 0)))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0 || n_chunks == 0) return B200GNN_OK;
  GatBwd p;
  p.rowptr = rowptr; p.col = col; p.a = a; p.ft = ft; p.dout = dout; p.el = el; p.er = er; p.dpre = dpre; p.der = der;
  p.scale = attn_scale;
  p.chunk_rowptr = chunk_rowptr; p.hub_rows = hub_rows; p.hub_segptr = hub_segptr; p.ws = hub_workspace;
  p.ldf = ldf; p.ldd = ldd; p.n_rows = n_rows; p.n_chunks = (int32_t)n_chunks; p.n_hub = (int32_t)n_hub;
  p.n_seg = (int32_t)(n_hub > 0 ? n_seg : 0); p.seg_len = seg_len;
  p.hub_threshold = hub_threshold; p.H = (int32_t)H; p.D = (int32_t)D; p.K = (int32_t)K; p.slope = negative_slope;
  cudaStream_t st = (cudaStream_t)stream;
  if (D % 4 == 0 && ldf % 4 == 0 && ldd % 4 == 0 && aligned_to(ft, 16) && aligned_to(dout, 16) && K <= 4 * 32 * GAT_MAXJ)
    return launch_bwd<float4>(p, st);
  if (D % 2 == 0 && ldf % 2 == 0 && ldd % 2 == 0 && aligned_to(ft, 8) && aligned_to(dout, 8) && K <= 2 * 32 * GAT_MAXJ)
    return launch_bwd<float2>(p, st);
  if (K <= 32 * GAT_MAXJ) return launch_bwd<float>(p, st);
  return B200GNN_ERR_UNSUPPORTED;
}

extern "C" int b200gnn_segment_sum_heads_f32(const int32_t* rowptr, const int32_t* eidx, const float* vals, int64_t n_rows,
                                             int64_t H, float* out, void* stream) {
  if (!rowptr || !vals || !out || n_rows < 0 || H <= 0 || H > GAT_MAXH) return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  GatSegSum p;
  p.rowptr = rowptr; p.eidx = eidx; p.vals = vals; p.out = out; p.n_rows = n_rows; p.H = (int32_t)H;
  gat_segment_sum_kernel<<<rows_grid(n_rows), GAT_THREADS, 0, (cudaStream_t)stream>>>(p);
  return check_launch();
}

// ---- the fused GAT layer (engine_gat.py)
extern "C" int64_t b200gnn_gat_stat_slots(int64_t n_chunks, int64_t n_hub) {
  if (n_chunks < 0 || n_hub < 0) return B200GNN_ERR_BAD_ARG;
  return (n_chunks + GAT_WARPS - 1) / GAT_WARPS + n_hub;
}

extern "C" int b200gnn_gat_aggregate_epi_f32(const int32_t* rowptr, const int32_t* col, const int32_t* eidx, const float* a,
                                             const float* ft, int64_t ldf, float* out, int64_t ldo, int64_t n_rows, int64_t H,
                                             int64_t D, const float* src_scale, const float* row_scale, const float* res,
                                             int64_t ldr, const float* bias, float* stat_partial, int64_t stat_slots,
                                             const int32_t* chunk_rowptr, int64_t n_chunks, int32_t hub_threshold,
                                             int32_t seg_len, const int32_t* hub_rows, const int32_t* hub_segptr, int64_t n_hub,
                                             int64_t n_seg, float* hub_workspace, void* stream) {
  const int64_t K = H * D;
  if (!rowptr || !a || !ft || !out || n_rows < 0 || H <= 0 || D <= 0 || H > GAT_MAXH || ldf < K || ldo < K || !chunk_rowptr ||
      n_chunks < 0 || n_hub < 0 || n_seg < n_hub || (res && ldr < K) ||
      (stat_partial && stat_slots < b200gnn_gat_stat_slots(n_chunks, n_hub)) ||
      (n_hub > 0 && (!hub_rows || !hub_segptr || !hub_workspace || seg_len <= 0)))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0 || n_chunks == 0) return B200GNN_OK;
  GatAgg p;
  p.rowptr = rowptr; p.col = col; p.eidx = eidx; p.chunk_rowptr = chunk_rowptr; p.hub_rows = hub_rows;
  p.hub_segptr = hub_segptr; p.ws = hub_workspace;
  p.a = a; p.ft = ft; p.out = out; p.ldf = ldf; p.ldo = ldo;
  p.n_chunks = (int32_t)n_chunks; p.n_hub = (int32_t)n_hub; p.n_seg = (int32_t)(n_hub > 0 ? n_seg : 0); p.seg_len = seg_len;
  p.hub_threshold = hub_threshold;
  p.H = (int32_t)H; p.D = (int32_t)D; p.K = (int32_t)K;
  GatEpi q;
  q.src_scale = src_scale; q.row_scale = row_scale; q.res = res; q.bias = bias; q.stat = stat_partial; q.ldr = res ? ldr : 0;
  q.act = nullptr; q.lda = 0; q.n_main = 0;
  cudaStream_t st = (cudaStream_t)stream;
  const bool r4 = !res || (ldr % 4 == 0 && aligned_to(res, 16)), r2 = !res || (ldr % 2 == 0 && aligned_to(res, 8));
  const bool b4 = !bias || aligned_to(bias, 16), b2 = !bias || aligned_to(bias, 8);
  if (D % 4 == 0 && ldf % 4 == 0 && ldo % 4 == 0 && aligned_to(ft, 16) && aligned_to(out, 16) && r4 && b4 && K <= 4 * 32 * GAT_MAXJ)
    return launch_agg_epi<float4>(p, q, st);
  if (D % 2 == 0 && ldf % 2 == 0 && ldo % 2 == 0 && aligned_to(ft, 8) && aligned_to(out, 8) && r2 && b2 && K <= 2 * 32 * GAT_MAXJ)
    return launch_agg_epi<float2>(p, q, st);
  if (K <= 32 * GAT_MAXJ) return launch_agg_epi<float>(p, q, st);
  return B200GNN_ERR_UNSUPPORTED;
}

extern "C" int b200gnn_gat_scores_f32(const float* ft, int64_t ldf, const float* attn_l, const float* attn_r,
                                      const float* src_scale, int64_t n_rows, int64_t H, int64_t D, float* el, float* er,
                                      void* stream) {
  if (!ft || !attn_l || !el || (attn_r && !er) || n_rows < 0 || H <= 0 || D <= 0 || H > GAT_MAXH || ldf < H * D)
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  GatScores p;
  p.ft = ft; p.attn_l = attn_l; p.attn_r = attn_r; p.src_scale = src_scale; p.el = el; p.er = er; p.ldf = ldf; p.n_rows = n_rows;
  p.H = (int32_t)H; p.D = (int32_t)D;
  gat_scores_kernel<<<rows_grid(n_rows), GAT_THREADS, 0, (cudaStream_t)stream>>>(p);
  return check_launch();
}

// slots of the [slots][2][H*D] partial buffer of b200gnn_gat_scores_bwd_f32
extern "C" int64_t b200gnn_gat_scores_slots(int64_t n_rows) {
  if (n_rows < 0) return B200GNN_ERR_BAD_ARG;
  const int64_t s = (n_rows + 63) / 64;
  return s < 1 ? 1 : (s > 132 * 4 ? 132 * 4 : s);
}

extern "C" int b200gnn_gat_scores_bwd_f32(const float* ft, int64_t ldf, const float* attn_l, const float* attn_r,
                                          const float* src_scale, const float* d_el, const float* d_er, int64_t n_rows,
                                          int64_t H, int64_t D, float* dft, int64_t ldd, float* d_attn_l, float* d_attn_r,
                                          float* partial, int64_t slots, void* stream) {
  const int64_t K = H * D;
  if (!ft || !attn_l || !d_el || !dft || !d_attn_l || !partial || (attn_r && (!d_er || !d_attn_r)) || n_rows <= 0 || H <= 0 ||
      D <= 0 || H > GAT_MAXH || ldf < K || ldd < K || slots < b200gnn_gat_scores_slots(n_rows))
    return B200GNN_ERR_BAD_ARG;
  if (K > GAT_THREADS * GAT_SB_MAXJ) return B200GNN_ERR_UNSUPPORTED;
  const int64_t used = b200gnn_gat_scores_slots(n_rows);
  GatScoresBwd p;
  p.ft = ft; p.attn_l = attn_l; p.attn_r = attn_r; p.src_scale = src_scale; p.del = d_el; p.der = d_er; p.dft = dft;
  p.partial = partial; p.ldf = ldf; p.ldd = ldd; p.n_rows = n_rows; p.H = (int32_t)H; p.D = (int32_t)D; p.K = (int32_t)K;
  p.rows_per_cta = (int32_t)((n_rows + used - 1) / used);
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  gat_scores_bwd_kernel<<<(int)used, GAT_THREADS, 0, st>>>(p);
  if ((rc = check_launch())) return rc;
  gat_scores_bwd_finalize_kernel<<<(int)((2 * K + GAT_THREADS - 1) / GAT_THREADS), GAT_THREADS, 0, st>>>(
      partial, (int)used, (int)K, d_attn_l, attn_r ? d_attn_r : nullptr);
  return check_launch();
}

// ---- the PyG GAT layers of the PPI models (engine_ppi.py): x = elu(GATConv(x) + Linear(x)) and the head-mean logits layer
namespace b200gnn {

// dZ = dA * (Z > 0 ? 1 : exp(Z)): torch's elu_backward (alpha 1, on the input), every operand with its own row pitch
template <typename V>
__global__ void __launch_bounds__(256) elu_bwd_kernel(const float* __restrict__ dA, int64_t ldda, const float* __restrict__ Z,
                                                      int64_t ldz, float* __restrict__ dZ, int64_t lddz, int64_t n_rows, int kv) {
  constexpr int W = VecTraits<V>::W;
  for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_rows * kv; i += (int64_t)gridDim.x * 256) {
    const int64_t r = i / kv;
    const int v = (int)(i - r * kv);
    const V g = vldg(reinterpret_cast<const V*>(dA + (size_t)r * ldda) + v);
    const V z = vldg(reinterpret_cast<const V*>(Z + (size_t)r * ldz) + v);
    const float* gs = reinterpret_cast<const float*>(&g);
    const float* zs = reinterpret_cast<const float*>(&z);
    V o;
    float* os = reinterpret_cast<float*>(&o);
#pragma unroll
    for (int w = 0; w < W; ++w) os[w] = zs[w] > 0.f ? gs[w] : gs[w] * expf(zs[w]);
    reinterpret_cast<V*>(dZ + (size_t)r * lddz)[v] = o;
  }
}

// Logits layer with concat=False (ppi_pyg/gnn.py:31,61 + the Linear skip) and its BCE / logit-KD loss (criterion.py:8-19).
// One warp per row, lanes over the columns; per CTA the (classification, distillation) sums in fp64, warps added in order.
constexpr int PPI_TAIL_MAX_SLOTS = 132 * 4;
struct PpiTail {
  const float* agg; const float* res; const float* b_conv; const float* b_lin; const float* y; const float* t;
  float* logits; float* d_agg; float* d_res; double* partial;
  int64_t lda, ldr, ldy, ldt, ldl, ldga, ldgr, n_rows;
  int32_t H, Dp, C;
  float w_cls, w_kd;            // d loss / d z = w_cls (sigmoid(z) - y) + w_kd (sigmoid(z) - sigmoid(t))
};

__global__ void __launch_bounds__(256) ppi_tail_kernel(const PpiTail p) {
  __shared__ double s_red[8][2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double acc_c = 0.0, acc_k = 0.0;
  const float hf = (float)p.H;
  for (int64_t r = (int64_t)blockIdx.x * 8 + warp; r < p.n_rows; r += (int64_t)gridDim.x * 8) {
    const float* ag = p.agg + (size_t)r * p.lda;
    for (int c = lane; c < p.Dp; c += 32) {
      if (c >= p.C) {                                      // padded columns of the gradients stay zero
        if (p.y) {
          for (int h = 0; h < p.H; ++h) p.d_agg[(size_t)r * p.ldga + h * p.Dp + c] = 0.f;
          p.d_res[(size_t)r * p.ldgr + c] = 0.f;
        }
        continue;
      }
      float s = __ldg(ag + c);
      for (int h = 1; h < p.H; ++h) s += __ldg(ag + h * p.Dp + c);
      const float z = (s / hf + __ldg(p.b_conv + c)) + (__ldg(p.res + (size_t)r * p.ldr + c) + __ldg(p.b_lin + c));
      p.logits[(size_t)r * p.ldl + c] = z;
      if (!p.y) continue;
      const float yv = __ldg(p.y + (size_t)r * p.ldy + c);
      const float sp = log1pf(expf(-fabsf(z))), mz = fmaxf(z, 0.f);
      const float sig = 1.f / (1.f + expf(-z));
      acc_c += (double)(mz - z * yv + sp);
      float dz = p.w_cls * (sig - yv);
      if (p.t) {
        const float tv = 1.f / (1.f + expf(-__ldg(p.t + (size_t)r * p.ldt + c)));
        acc_k += (double)(mz - z * tv + sp);
        dz += p.w_kd * (sig - tv);
      }
      p.d_res[(size_t)r * p.ldgr + c] = dz;
      const float dh = dz / hf;                          // mean over heads: every head gets d z / H
      for (int h = 0; h < p.H; ++h) p.d_agg[(size_t)r * p.ldga + h * p.Dp + c] = dh;
    }
  }
  if (!p.y) return;
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    acc_c += __shfl_xor_sync(FULL_MASK, acc_c, d);
    acc_k += __shfl_xor_sync(FULL_MASK, acc_k, d);
  }
  if (lane == 0) { s_red[warp][0] = acc_c; s_red[warp][1] = acc_k; }
  __syncthreads();
  if (threadIdx.x < 2) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += s_red[w][threadIdx.x];
    p.partial[(size_t)blockIdx.x * 2 + threadIdx.x] = t;
  }
}

// loss_out = [alpha T^2 kd + (1 - alpha) cls, cls, kd] (KD) or [cls, cls, 0], the slots added in order
__global__ void ppi_tail_finalize_kernel(const double* __restrict__ partial, int slots, double inv_n, int kd, float alpha, float T,
                                         float* __restrict__ loss_out) {
  double c = 0.0, k = 0.0;
  for (int s = 0; s < slots; ++s) { c += partial[2 * s]; k += partial[2 * s + 1]; }
  const float cls = (float)(c * inv_n), dis = (float)(k * inv_n);
  loss_out[0] = kd ? dis * (alpha * T * T) + cls * (1.f - alpha) : cls;
  loss_out[1] = cls;
  loss_out[2] = kd ? dis : 0.f;
}

}  // namespace b200gnn

extern "C" int b200gnn_gat_aggregate_elu_f32(const int32_t* rowptr, const int32_t* col, const int32_t* eidx, const float* a,
                                             const float* ft, int64_t ldf, float* out, int64_t ldo, float* act, int64_t lda,
                                             int64_t n_rows, int64_t H, int64_t D, const float* res, int64_t ldr,
                                             const float* bias, const int32_t* chunk_rowptr, int64_t n_chunks,
                                             int32_t hub_threshold, int32_t seg_len, const int32_t* hub_rows,
                                             const int32_t* hub_segptr, int64_t n_hub, int64_t n_seg, float* hub_workspace,
                                             void* stream) {
  const int64_t K = H * D;
  if (!rowptr || !a || !ft || !out || !act || n_rows < 0 || H <= 0 || D <= 0 || H > GAT_MAXH || ldf < K || ldo < K || lda < K ||
      !chunk_rowptr || n_chunks < 0 || n_hub < 0 || n_seg < n_hub || (res && ldr < K) ||
      (n_hub > 0 && (!hub_rows || !hub_segptr || !hub_workspace || seg_len <= 0)))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0 || n_chunks == 0) return B200GNN_OK;
  GatAgg p;
  p.rowptr = rowptr; p.col = col; p.eidx = eidx; p.chunk_rowptr = chunk_rowptr; p.hub_rows = hub_rows;
  p.hub_segptr = hub_segptr; p.ws = hub_workspace;
  p.a = a; p.ft = ft; p.out = out; p.ldf = ldf; p.ldo = ldo;
  p.n_chunks = (int32_t)n_chunks; p.n_hub = (int32_t)n_hub; p.n_seg = (int32_t)(n_hub > 0 ? n_seg : 0); p.seg_len = seg_len;
  p.hub_threshold = hub_threshold;
  p.H = (int32_t)H; p.D = (int32_t)D; p.K = (int32_t)K;
  GatEpi q;
  q.src_scale = nullptr; q.row_scale = nullptr; q.res = res; q.bias = bias; q.stat = nullptr; q.ldr = res ? ldr : 0;
  q.act = act; q.lda = lda; q.n_main = 0;
  cudaStream_t st = (cudaStream_t)stream;
  // The vector width is chosen from the epi entry point's operands exactly as b200gnn_gat_aggregate_epi_f32 chooses it, so
  // both run the same (V, NJ, U) instantiation shape and Z is its output bit for bit.  act must then take that width too
  // (a narrower width would change U and with it the hub segments' summation order): otherwise the call is refused.
  const bool r4 = !res || (ldr % 4 == 0 && aligned_to(res, 16)), r2 = !res || (ldr % 2 == 0 && aligned_to(res, 8));
  const bool b4 = !bias || aligned_to(bias, 16), b2 = !bias || aligned_to(bias, 8);
  if (D % 4 == 0 && ldf % 4 == 0 && ldo % 4 == 0 && aligned_to(ft, 16) && aligned_to(out, 16) && r4 && b4 &&
      K <= 4 * 32 * GAT_MAXJ) {
    if (lda % 4 || !aligned_to(act, 16)) return B200GNN_ERR_BAD_ARG;
    return launch_agg_epi<float4, true>(p, q, st);
  }
  if (D % 2 == 0 && ldf % 2 == 0 && ldo % 2 == 0 && aligned_to(ft, 8) && aligned_to(out, 8) && r2 && b2 &&
      K <= 2 * 32 * GAT_MAXJ) {
    if (lda % 2 || !aligned_to(act, 8)) return B200GNN_ERR_BAD_ARG;
    return launch_agg_epi<float2, true>(p, q, st);
  }
  if (K <= 32 * GAT_MAXJ) return launch_agg_epi<float, true>(p, q, st);
  return B200GNN_ERR_UNSUPPORTED;
}

extern "C" int b200gnn_elu_bwd_f32(const float* dA, int64_t ldda, const float* Z, int64_t ldz, float* dZ, int64_t lddz,
                                   int64_t n_rows, int64_t K, void* stream) {
  if (!dA || !Z || !dZ || n_rows < 0 || K <= 0 || ldda < K || ldz < K || lddz < K) return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool v4 = K % 4 == 0 && ldda % 4 == 0 && ldz % 4 == 0 && lddz % 4 == 0 && aligned_to(dA, 16) && aligned_to(Z, 16) &&
                  aligned_to(dZ, 16);
  const int64_t kv = v4 ? K / 4 : K;
  int64_t grid = (n_rows * kv + 255) / 256;
  if (grid > 132 * 8) grid = 132 * 8;
  if (v4) elu_bwd_kernel<float4><<<(int)grid, 256, 0, st>>>(dA, ldda, Z, ldz, dZ, lddz, n_rows, (int)kv);
  else elu_bwd_kernel<float><<<(int)grid, 256, 0, st>>>(dA, ldda, Z, ldz, dZ, lddz, n_rows, (int)kv);
  return check_launch();
}

extern "C" int64_t b200gnn_ppi_tail_slots(int64_t n_rows) {
  if (n_rows < 0) return B200GNN_ERR_BAD_ARG;
  const int64_t s = (n_rows + 7) / 8;
  return s < 1 ? 1 : (s > PPI_TAIL_MAX_SLOTS ? PPI_TAIL_MAX_SLOTS : s);
}

extern "C" int b200gnn_ppi_logits_loss_f32(const float* agg, int64_t lda, const float* res, int64_t ldr, const float* b_conv,
                                           const float* b_lin, int64_t n_rows, int64_t H, int64_t Dp, int64_t C,
                                           float* logits, int64_t ldl, const float* labels, int64_t ldy,
                                           const float* teacher_logits, int64_t ldt, float alpha, float T, float* d_agg,
                                           int64_t ldga, float* d_res, int64_t ldgr, float* loss_out, double* partial,
                                           int64_t slots, void* stream) {
  if (!agg || !res || !b_conv || !b_lin || !logits || n_rows < 0 || H <= 0 || H > GAT_MAXH || C <= 0 || Dp < C ||
      lda < H * Dp || ldr < C || ldl < C)
    return B200GNN_ERR_BAD_ARG;
  if (labels && (ldy < C || !d_agg || !d_res || !loss_out || !partial || ldga < H * Dp || ldgr < Dp ||
                 slots < b200gnn_ppi_tail_slots(n_rows) || (teacher_logits && ldt < C) || n_rows == 0))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  PpiTail p;
  p.agg = agg; p.res = res; p.b_conv = b_conv; p.b_lin = b_lin; p.y = labels; p.t = labels ? teacher_logits : nullptr;
  p.logits = logits; p.d_agg = d_agg; p.d_res = d_res; p.partial = partial;
  p.lda = lda; p.ldr = ldr; p.ldy = ldy; p.ldt = ldt; p.ldl = ldl; p.ldga = ldga; p.ldgr = ldgr; p.n_rows = n_rows;
  p.H = (int32_t)H; p.Dp = (int32_t)Dp; p.C = (int32_t)C;
  const double n_el = (double)n_rows * (double)C;
  p.w_cls = (float)((p.t ? 1.0 - alpha : 1.0) / n_el);
  p.w_kd = p.t ? (float)((double)alpha * T * T / n_el) : 0.f;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)b200gnn_ppi_tail_slots(n_rows);
  int rc;
  ppi_tail_kernel<<<grid, 256, 0, st>>>(p);
  if ((rc = check_launch()) || !labels) return rc;
  ppi_tail_finalize_kernel<<<1, 1, 0, st>>>(partial, grid, 1.0 / n_el, p.t != nullptr, alpha, T, loss_out);
  return check_launch();
}
