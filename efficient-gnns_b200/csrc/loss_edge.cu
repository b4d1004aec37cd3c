// Local Structure Preserving loss (lpw_criterion, arxiv_pyg/criterion.py:95-126) as three passes over the edge list,
// sorted once by destination (the softmax group index, criterion.py:100-104):
//   1. edge_sim      : per edge  k(f[src], f[dst])  for k in {cosine, cosine^2, ||.||, exp(-||.||^2/2)} — the two feature
//                      rows are read in place (no [E,F] gathers materialised as the reference does: 4 x E x F floats);
//   2. lsp_segment   : per destination segment, PyG softmax statistics for student and teacher, the KL (or MSE) terms,
//                      and d loss / d sim_student for every edge;
//   3. edge_sim_bwd  : chain rule back to the student features (atomic row adds, like the reference's index backward).
#include "common.cuh"

namespace b200gnn {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, d));
  return v;
}

constexpr float COS_EPS = 1e-8f;   // F.cosine_similarity eps (each norm clamped separately, torch >= 1.12)

// kernel ids: 0 cosine, 1 poly (cosine^2), 2 l2, 3 rbf
__global__ void __launch_bounds__(256) edge_sim_kernel(const float* __restrict__ feat, int F, const int32_t* __restrict__ src,
                                                       const int32_t* __restrict__ dst, int64_t E, int kernel,
                                                       float* __restrict__ sim) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t e = warp; e < E; e += nwarps) {
    const float* a = feat + (size_t)src[e] * F;
    const float* b = feat + (size_t)dst[e] * F;
    float s;
    if (kernel <= 1) {
      float dot = 0.f, na = 0.f, nb = 0.f;
      for (int k = lane; k < F; k += 32) { const float x = __ldg(a + k), y = __ldg(b + k); dot = fmaf(x, y, dot); na = fmaf(x, x, na); nb = fmaf(y, y, nb); }
      dot = wsum(dot); na = wsum(na); nb = wsum(nb);
      const float c = dot / (fmaxf(sqrtf(na), COS_EPS) * fmaxf(sqrtf(nb), COS_EPS));
      s = kernel == 0 ? c : c * c;
    } else {
      float d2 = 0.f;
      for (int k = lane; k < F; k += 32) { const float d = __ldg(a + k) - __ldg(b + k); d2 = fmaf(d, d, d2); }
      d2 = wsum(d2);
      s = kernel == 2 ? sqrtf(d2) : expf(-0.5f * d2);
    }
    if (lane == 0) sim[e] = s;
  }
}

// One warp per destination segment [rowptr[i], rowptr[i+1]) of the dst-sorted edge arrays.
// criterion 0: kld  loss = (1/E) sum_e xlogy(pt,pt) - pt*log(ps) ; 1: mse  loss = (1/E) sum_e (ps-pt)^2
__global__ void __launch_bounds__(256) lsp_segment_kernel(const float* __restrict__ sim_s, const float* __restrict__ sim_t,
                                                          const int32_t* __restrict__ rowptr, int64_t n_seg, float inv_E,
                                                          int criterion, float* __restrict__ g, float* __restrict__ partial) {
  __shared__ float s_acc[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 8 + warp; i < n_seg; i += (int64_t)gridDim.x * 8) {
    const int b = rowptr[i], e = rowptr[i + 1];
    if (b == e) continue;
    float ms = -INFINITY, mt = -INFINITY;
    for (int k = b + lane; k < e; k += 32) { ms = fmaxf(ms, sim_s[k]); mt = fmaxf(mt, sim_t[k]); }
    ms = wmax(ms); mt = wmax(mt);
    float zs = 0.f, zt = 0.f;
    for (int k = b + lane; k < e; k += 32) { zs += expf(sim_s[k] - ms); zt += expf(sim_t[k] - mt); }
    zs = wsum(zs) + 1e-16f; zt = wsum(zt) + 1e-16f;           // PyG softmax: e / (sum + 1e-16)
    const float lzs = logf(zs), lzt = logf(zt);
    if (criterion == 0) {
      const float T = (zt - 1e-16f) / zt;                      // sum_e pt over the segment
      for (int k = b + lane; k < e; k += 32) {
        const float lps = (sim_s[k] - ms) - lzs, lpt = (sim_t[k] - mt) - lzt;
        const float ps = expf(lps), pt = expf(lpt);
        acc += pt > 0.f ? pt * (lpt - lps) : 0.f;
        g[k] = (ps * T - pt) * inv_E;
      }
    } else {
      float q = 0.f;
      for (int k = b + lane; k < e; k += 32) {
        const float ps = expf((sim_s[k] - ms) - lzs), pt = expf((sim_t[k] - mt) - lzt);
        q += (ps - pt) * ps;
      }
      q = wsum(q);
      for (int k = b + lane; k < e; k += 32) {
        const float ps = expf((sim_s[k] - ms) - lzs), pt = expf((sim_t[k] - mt) - lzt);
        const float d = ps - pt;
        acc = fmaf(d, d, acc);
        g[k] = 2.f * inv_E * ps * (d - q);
      }
    }
  }
  acc = wsum(acc);
  if (lane == 0) s_acc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_acc[w];
    partial[blockIdx.x] = t;
  }
}

__global__ void __launch_bounds__(256) edge_sim_bwd_kernel(const float* __restrict__ feat, int F, const int32_t* __restrict__ src,
                                                           const int32_t* __restrict__ dst, int64_t E, int kernel,
                                                           const float* __restrict__ sim, const float* __restrict__ g,
                                                           float* __restrict__ dfeat) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t e = warp; e < E; e += nwarps) {
    const int is = src[e], id = dst[e];
    const float* a = feat + (size_t)is * F;
    const float* b = feat + (size_t)id * F;
    float* da = dfeat + (size_t)is * F;
    float* db = dfeat + (size_t)id * F;
    float ge = g[e];
    if (kernel <= 1) {
      float dot = 0.f, na2 = 0.f, nb2 = 0.f;
      for (int k = lane; k < F; k += 32) { const float x = __ldg(a + k), y = __ldg(b + k); dot = fmaf(x, y, dot); na2 = fmaf(x, x, na2); nb2 = fmaf(y, y, nb2); }
      dot = wsum(dot); na2 = wsum(na2); nb2 = wsum(nb2);
      const float ra = sqrtf(na2), rb = sqrtf(nb2);
      const float na = fmaxf(ra, COS_EPS), nb = fmaxf(rb, COS_EPS);
      const float c = dot / (na * nb);
      if (kernel == 1) ge *= 2.f * c;
      const float cross = ge / (na * nb);
      const float sa = ra > COS_EPS ? ge * c / (na * na) : 0.f;   // clamped norm carries no gradient
      const float sb = rb > COS_EPS ? ge * c / (nb * nb) : 0.f;
      for (int k = lane; k < F; k += 32) {
        const float x = __ldg(a + k), y = __ldg(b + k);
        atomicAdd(da + k, cross * y - sa * x);
        atomicAdd(db + k, cross * x - sb * y);
      }
    } else {
      float coef;  // d sim / d a = coef * (a - b),  d sim / d b = -coef * (a - b)
      if (kernel == 2) { const float d = sim[e]; coef = d > 0.f ? ge / d : 0.f; }
      else coef = -ge * sim[e];
      for (int k = lane; k < F; k += 32) {
        const float v = coef * (__ldg(a + k) - __ldg(b + k));
        atomicAdd(da + k, v);
        atomicAdd(db + k, -v);
      }
    }
  }
}

// Deterministic backward (replaces the atomic row adds above on the autograd path).  The gradient of node i is
//     d f_i = sum_{e: dst=i} (w_e f[src_e] - sb_e f_i) + sum_{e: src=i} (w_e f[dst_e] - sa_e f_i)
// i.e. ONE sparse product  d F = C · F  with the (2E + n)-entry matrix C that holds w_e at (dst_e, src_e) and
// (src_e, dst_e) and  -(sum of the row's sa/sb)  on the diagonal.  The plan fixes C's CSR structure once per edge list
// (pos_dst / pos_src / diag_pos = where each edge and each diagonal sits); every backward fills the values with the two
// kernels below and runs the row-segmented SpMM (spmm.cu: fixed summation order, hub rows split) — bitwise repeatable.
__global__ void __launch_bounds__(256) lsp_edge_coef_kernel(const float* __restrict__ feat, int F, const int32_t* __restrict__ src,
                                                            const int32_t* __restrict__ dst, int64_t E, int kernel,
                                                            const float* __restrict__ sim, const float* __restrict__ g,
                                                            const int32_t* __restrict__ pos_dst, const int32_t* __restrict__ pos_src,
                                                            float* __restrict__ val, float* __restrict__ selfc) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t e = warp; e < E; e += nwarps) {
    float ge = g[e];
    float w, sa, sb;
    if (kernel <= 1) {
      const float* a = feat + (size_t)src[e] * F;
      const float* b = feat + (size_t)dst[e] * F;
      float dot = 0.f, na2 = 0.f, nb2 = 0.f;
      for (int k = lane; k < F; k += 32) { const float x = __ldg(a + k), y = __ldg(b + k); dot = fmaf(x, y, dot); na2 = fmaf(x, x, na2); nb2 = fmaf(y, y, nb2); }
      dot = wsum(dot); na2 = wsum(na2); nb2 = wsum(nb2);
      const float ra = sqrtf(na2), rb = sqrtf(nb2);
      const float na = fmaxf(ra, COS_EPS), nb = fmaxf(rb, COS_EPS);
      const float c = dot / (na * nb);
      if (kernel == 1) ge *= 2.f * c;
      w = ge / (na * nb);
      sa = ra > COS_EPS ? ge * c / (na * na) : 0.f;   // clamped norm carries no gradient
      sb = rb > COS_EPS ? ge * c / (nb * nb) : 0.f;
    } else {
      float coef;  // d sim / d a = coef * (a - b),  d sim / d b = -coef * (a - b)
      if (kernel == 2) { const float d = sim[e]; coef = d > 0.f ? ge / d : 0.f; }
      else coef = -ge * sim[e];
      w = -coef; sa = -coef; sb = -coef;
    }
    if (lane == 0) {
      const int pd = pos_dst[e], ps = pos_src[e];
      val[pd] = w; selfc[pd] = sb;
      val[ps] = w; selfc[ps] = sa;
    }
  }
}

// val[diag_pos[i]] = -(sum of selfc over row i's off-diagonal entries, in CSR order); selfc[diag] is ignored.
__global__ void __launch_bounds__(256) lsp_diag_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ diag_pos,
                                                       int64_t n, const float* __restrict__ selfc, float* __restrict__ val) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t i = warp; i < n; i += nwarps) {
    const int b = rowptr[i], e = rowptr[i + 1], dp = diag_pos[i];
    float acc = 0.f;
    for (int k = b + lane; k < e; k += 32) acc += (k == dp) ? 0.f : selfc[k];
    acc = wsum(acc);                                  // xor-butterfly: the same tree every run
    if (lane == 0) val[dp] = -acc;
  }
}

// The student side of the captured LSP step (criterion kld): edge_sim(student) -> lsp_segment -> lsp_edge_coef in one
// kernel, one warp per destination segment with lsp_segment_kernel's grid and warp-to-segment mapping, so every float it
// produces is the one the three kernels produce (same per-lane fmaf chains, same butterflies, same per-lane edge order).
//   pass 1: per edge, the whole warp forms k(f[src], f[dst]) as edge_sim_kernel does; the destination row (the same for the
//           whole segment) sits in registers, NC floats per lane (F <= 32 NC), and its squared norm is reduced once.
//           sim_s[e] and, for cosine / poly, c[e] and the unclamped source norm ra[e] go to memory.
//   pass 2 + 3: lane-per-edge, lsp_segment_kernel's statistics and KL terms, then g_e and lsp_edge_coef_kernel's w / sa / sb
//           from the pass-1 terms, without reading the features again.
template <int NC>
__global__ void __launch_bounds__(256, 4) lsp_student_kernel(const float* __restrict__ feat, int F, const int32_t* __restrict__ src,
                                                          const int32_t* __restrict__ dst, const int32_t* __restrict__ rowptr,
                                                          int64_t n_seg, const float* __restrict__ sim_t, int kernel,
                                                          float inv_E, const int32_t* __restrict__ pos_dst,
                                                          const int32_t* __restrict__ pos_src, float* sim_s, float* c_e,
                                                          float* ra_e, float* __restrict__ val, float* __restrict__ selfc,
                                                          float* __restrict__ partial) {
  __shared__ float s_acc[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * 8 + warp; i < n_seg; i += (int64_t)gridDim.x * 8) {
    const int b = rowptr[i], e = rowptr[i + 1];
    if (b == e) continue;
    // ---- pass 1
    const float* brow = feat + (size_t)dst[b] * F;
    float yr[NC];
#pragma unroll
    for (int j = 0; j < NC; ++j) yr[j] = lane + 32 * j < F ? __ldg(brow + lane + 32 * j) : 0.f;
    float rb = 0.f, nb = 0.f;
    if (kernel <= 1) {
      float nb2 = 0.f;
#pragma unroll
      for (int j = 0; j < NC; ++j)
        if (lane + 32 * j < F) nb2 = fmaf(yr[j], yr[j], nb2);
      rb = sqrtf(wsum(nb2));
      nb = fmaxf(rb, COS_EPS);
    }
    for (int k = b; k < e; ++k) {
      const float* a = feat + (size_t)src[k] * F;
      float s;
      if (kernel <= 1) {
        float dot = 0.f, na2 = 0.f;
#pragma unroll
        for (int j = 0; j < NC; ++j)
          if (lane + 32 * j < F) { const float x = __ldg(a + lane + 32 * j); dot = fmaf(x, yr[j], dot); na2 = fmaf(x, x, na2); }
        dot = wsum(dot); na2 = wsum(na2);
        const float ra = sqrtf(na2);
        const float c = dot / (fmaxf(ra, COS_EPS) * nb);
        s = kernel == 0 ? c : c * c;
        if (lane == 0) { c_e[k] = c; ra_e[k] = ra; }
      } else {
        float d2 = 0.f;
#pragma unroll
        for (int j = 0; j < NC; ++j)
          if (lane + 32 * j < F) { const float d = __ldg(a + lane + 32 * j) - yr[j]; d2 = fmaf(d, d, d2); }
        d2 = wsum(d2);
        s = kernel == 2 ? sqrtf(d2) : expf(-0.5f * d2);
      }
      if (lane == 0) sim_s[k] = s;
    }
    __syncwarp();                                   // lane 0's stores above are read by every lane below
    // ---- pass 2: lsp_segment_kernel, criterion 0
    float ms = -INFINITY, mt = -INFINITY;
    for (int k = b + lane; k < e; k += 32) { ms = fmaxf(ms, sim_s[k]); mt = fmaxf(mt, sim_t[k]); }
    ms = wmax(ms); mt = wmax(mt);
    float zs = 0.f, zt = 0.f;
    for (int k = b + lane; k < e; k += 32) { zs += expf(sim_s[k] - ms); zt += expf(sim_t[k] - mt); }
    zs = wsum(zs) + 1e-16f; zt = wsum(zt) + 1e-16f;
    const float lzs = logf(zs), lzt = logf(zt);
    const float T = (zt - 1e-16f) / zt;
    for (int k = b + lane; k < e; k += 32) {
      const float sk = sim_s[k];
      const float lps = (sk - ms) - lzs, lpt = (sim_t[k] - mt) - lzt;
      const float ps = expf(lps), pt = expf(lpt);
      acc += pt > 0.f ? pt * (lpt - lps) : 0.f;
      float ge = (ps * T - pt) * inv_E;
      // ---- pass 3: lsp_edge_coef_kernel from the pass-1 terms
      float w, sa, sb;
      if (kernel <= 1) {
        const float c = c_e[k], ra = ra_e[k];
        const float na = fmaxf(ra, COS_EPS);
        if (kernel == 1) ge *= 2.f * c;
        w = ge / (na * nb);
        sa = ra > COS_EPS ? ge * c / (na * na) : 0.f;   // clamped norm carries no gradient
        sb = rb > COS_EPS ? ge * c / (nb * nb) : 0.f;
      } else {
        float coef;
        if (kernel == 2) coef = sk > 0.f ? ge / sk : 0.f;
        else coef = -ge * sk;
        w = -coef; sa = -coef; sb = -coef;
      }
      const int pd = pos_dst[k], pq = pos_src[k];
      val[pd] = w; selfc[pd] = sb;
      val[pq] = w; selfc[pq] = sa;
    }
  }
  acc = wsum(acc);
  if (lane == 0) s_acc[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += s_acc[w];
    partial[blockIdx.x] = t;
  }
}

// dst[idx[i]] = src[i] * scale (a plain fp32 product), one warp per row; thread 0 of block 0 also forms
// loss_total[0] += loss_aux[0] * scale (fp32 product, then fp32 add) when loss_total is given.
template <bool VEC>
__global__ void __launch_bounds__(256) scatter_rows_scaled_kernel(const float* __restrict__ src, const int64_t* __restrict__ idx,
                                                                  int64_t n, int K, float scale, float* __restrict__ dst,
                                                                  int64_t ldd, const float* __restrict__ loss_aux,
                                                                  float* __restrict__ loss_total) {
  if (loss_total && blockIdx.x == 0 && threadIdx.x == 0) loss_total[0] = __fadd_rn(loss_total[0], __fmul_rn(loss_aux[0], scale));
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t i = warp; i < n; i += nwarps) {
    const float* s = src + (size_t)i * K;
    float* d = dst + (size_t)idx[i] * ldd;
    if (VEC) {
      for (int k = lane; k < K / 4; k += 32) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(s) + k);
        reinterpret_cast<float4*>(d)[k] = make_float4(__fmul_rn(v.x, scale), __fmul_rn(v.y, scale), __fmul_rn(v.z, scale),
                                                      __fmul_rn(v.w, scale));
      }
    } else {
      for (int k = lane; k < K; k += 32) d[k] = __fmul_rn(__ldg(s + k), scale);
    }
  }
}

static inline int edge_grid(int64_t items) {
  int64_t g = (items + 7) / 8;
  if (g > 132 * 16) g = 132 * 16;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_edge_sim_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst, int64_t E,
                                    int kernel, float* sim, void* stream) {
  if (!feat || !sim || F <= 0 || E < 0 || kernel < 0 || kernel > 3) return B200GNN_ERR_BAD_ARG;
  if (E == 0) return B200GNN_OK;
  if (!src || !dst) return B200GNN_ERR_BAD_ARG;
  edge_sim_kernel<<<edge_grid(E), 256, 0, (cudaStream_t)stream>>>(feat, (int)F, src, dst, E, kernel, sim);
  return check_launch();
}

extern "C" int64_t b200gnn_lsp_partials(int64_t n_seg) { return edge_grid(n_seg); }

extern "C" int b200gnn_lsp_segment_f32(const float* sim_s, const float* sim_t, const int32_t* rowptr, int64_t n_seg,
                                       int64_t E, int criterion, float* g, float* loss_out, float* partial, void* stream) {
  if (!sim_s || !sim_t || !rowptr || !g || !loss_out || !partial || n_seg <= 0 || E <= 0 || criterion < 0 || criterion > 1)
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = edge_grid(n_seg);
  int rc;
  lsp_segment_kernel<<<grid, 256, 0, st>>>(sim_s, sim_t, rowptr, n_seg, 1.f / (float)E, criterion, g, partial);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, grid, 1.0 / (double)E, loss_out);
  return check_launch();
}

extern "C" int b200gnn_edge_sim_bwd_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst, int64_t E,
                                        int kernel, const float* sim, const float* g, float* dfeat, void* stream) {
  if (!feat || !sim || !g || !dfeat || F <= 0 || E < 0 || kernel < 0 || kernel > 3) return B200GNN_ERR_BAD_ARG;
  if (E == 0) return B200GNN_OK;
  if (!src || !dst) return B200GNN_ERR_BAD_ARG;
  edge_sim_bwd_kernel<<<edge_grid(E), 256, 0, (cudaStream_t)stream>>>(feat, (int)F, src, dst, E, kernel, sim, g, dfeat);
  return check_launch();
}

// Values of the (2E + n)-entry backward matrix C (see lsp_edge_coef_kernel): the caller then runs
// b200gnn_spmm_csr_f32(C, feat) to obtain d loss / d feat without atomics.
extern "C" int b200gnn_lsp_bwd_values_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst, int64_t E,
                                          int kernel, const float* sim, const float* g, const int32_t* pos_dst,
                                          const int32_t* pos_src, const int32_t* comb_rowptr, const int32_t* diag_pos,
                                          int64_t n_nodes, float* val, float* selfc, void* stream) {
  if (!feat || !sim || !g || !val || !selfc || !comb_rowptr || !diag_pos || F <= 0 || E < 0 || n_nodes <= 0 || kernel < 0 ||
      kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (E > 0) {
    if (!src || !dst || !pos_dst || !pos_src) return B200GNN_ERR_BAD_ARG;
    lsp_edge_coef_kernel<<<edge_grid(E), 256, 0, st>>>(feat, (int)F, src, dst, E, kernel, sim, g, pos_dst, pos_src, val, selfc);
    if ((rc = check_launch())) return rc;
  }
  lsp_diag_kernel<<<edge_grid(n_nodes), 256, 0, st>>>(comb_rowptr, diag_pos, n_nodes, selfc, val);
  return check_launch();
}

// The captured LSP step's student side (kld): lsp_student_kernel, then lsp_diag_kernel and sum_partials_kernel, with the
// launches and grids of edge_sim -> lsp_segment -> lsp_bwd_values.  scratch: 2E floats (c and ra per edge).
extern "C" int b200gnn_lsp_student_f32(const float* feat, int64_t F, const int32_t* src, const int32_t* dst,
                                       const int32_t* rowptr, int64_t n_seg, int64_t E, const float* sim_t, int kernel,
                                       const int32_t* pos_dst, const int32_t* pos_src, const int32_t* comb_rowptr,
                                       const int32_t* diag_pos, int64_t n_nodes, float* sim_s, float* scratch, float* val,
                                       float* selfc, float* loss_out, float* partial, void* stream) {
  if (!feat || !src || !dst || !rowptr || !sim_t || !pos_dst || !pos_src || !comb_rowptr || !diag_pos || !sim_s || !scratch ||
      !val || !selfc || !loss_out || !partial || F <= 0 || F > B200GNN_LSP_MAX_F || E <= 0 || n_seg <= 0 || n_nodes <= 0 ||
      kernel < 0 || kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = edge_grid(n_seg);
  const float inv_E = 1.f / (float)E;
  float *c_e = scratch, *ra_e = scratch + E;
#define LSP_STUDENT(NC) \
  lsp_student_kernel<NC><<<grid, 256, 0, st>>>(feat, (int)F, src, dst, rowptr, n_seg, sim_t, kernel, inv_E, pos_dst, pos_src, \
                                               sim_s, c_e, ra_e, val, selfc, partial)
  if (F <= 32) LSP_STUDENT(1);
  else if (F <= 64) LSP_STUDENT(2);
  else if (F <= 128) LSP_STUDENT(4);
  else if (F <= 256) LSP_STUDENT(8);
  else LSP_STUDENT(16);
#undef LSP_STUDENT
  int rc;
  if ((rc = check_launch())) return rc;
  lsp_diag_kernel<<<edge_grid(n_nodes), 256, 0, st>>>(comb_rowptr, diag_pos, n_nodes, selfc, val);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, grid, 1.0 / (double)E, loss_out);
  return check_launch();
}

extern "C" int b200gnn_scatter_rows_scaled_f32(const float* src, const int64_t* idx, int64_t n, int64_t K, float scale,
                                               float* dst, int64_t ldd, const float* loss_aux, float* loss_total,
                                               void* stream) {
  if (!src || !idx || !dst || n < 0 || K <= 0 || K > INT32_MAX || ldd < K || (loss_total && !loss_aux))
    return B200GNN_ERR_BAD_ARG;
  if (n == 0 && !loss_total) return B200GNN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = edge_grid(n);
  if (K % 4 == 0 && ldd % 4 == 0 && aligned_to(src, 16) && aligned_to(dst, 16))
    scatter_rows_scaled_kernel<true><<<grid, 256, 0, st>>>(src, idx, n, (int)K, scale, dst, ldd, loss_aux, loss_total);
  else
    scatter_rows_scaled_kernel<false><<<grid, 256, 0, st>>>(src, idx, n, (int)K, scale, dst, ldd, loss_aux, loss_total);
  return check_launch();
}
