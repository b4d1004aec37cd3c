// The row passes of the captured G-CRD step (graph contrastive representation distillation, arxiv_pyg/criterion.py:129-149
// with the projection heads of arxiv_pyg/gnn.py:296-306): the on-device draw of the sampled rows, the sampled rows of both
// heads turned into InfoNCE operands, and the way back from the operand gradients to the heads' pre-activations.  The
// heads' GEMMs, BatchNorm statistics and backward, and the InfoNCE chunks themselves run on the existing kernels.
//
// Head h (s = student, t = teacher) over the n_train training rows: pre_h = G_h W_h^T + b_h (row pitch P), bn_h = [4][P]
// (mean, invstd, scale, shift of b200gnn_bn_finalize_f32), P_h = relu(pre_h * scale + shift).  Sampled position j is
// training row inds[j]; x_h[j] = scale_h * P_h[inds[j]] / max(||P_h[inds[j]]||, eps) (scale_s = 1 / nce_T, scale_t = 1).
//
// GSP (global structure preservation, arxiv_pyg/criterion.py:57-92) on the same heads uses the same two row passes:
// cosine / poly take the normalising path with scale 1 on both sides; l2 / rbf the raw path, x_h[j] = P_h[inds[j]] with
// its squared norm, and on the way back the norm term of the distance instead of the normalise backward.
#include "common.cuh"
#include "philox.cuh"

namespace b200gnn {
namespace gcrd {

constexpr int BWD_CTAS = 64;                 // 512 warps: the backward's partial slots (fixed, so the order is fixed)
constexpr int MAX_P = 256;                   // lane c owns float4 chunks c and c + 32

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, const float4& v) { *reinterpret_cast<float4*>(p) = v; }

// Philox key of every training row: word (i % 4) of block i / 4 at the step's offset.  Sorting rows by (key, row) and
// keeping the first S is a uniformly drawn S-subset up to ties of equal keys, which go to the lower row: about n^2 / 2^33
// tied pairs per step (~1 at n = 90,941), and only a pair straddling sorted position S changes the sample.
__global__ void __launch_bounds__(256) sample_keys_kernel(int64_t n, uint64_t seed, uint64_t offset, const int32_t* __restrict__ step_dev,
                                                          int64_t* __restrict__ key, int64_t* __restrict__ row) {
  const uint64_t off = offset + (step_dev ? (uint64_t)(*step_dev) : 0ull);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const uint4 r = philox4x32(seed, off, (uint64_t)i >> 2);
    const uint32_t w = (i & 3) == 0 ? r.x : (i & 3) == 1 ? r.y : (i & 3) == 2 ? r.z : r.w;
    key[i] = (int64_t)w;
    row[i] = i;
  }
}

// One head's operand row: x = sc * relu(bn(pre)) / max(||.||, eps), norm = ||relu(bn(pre))||.
// RAW: x = relu(bn(pre)), norm = its squared norm (sc and eps unused).
template <bool RAW>
__device__ __forceinline__ void operand_row(const float* __restrict__ pre, const float* __restrict__ bn, int P, float sc, float eps,
                                            float* __restrict__ x, float* __restrict__ norm, int lane) {
  float4 a[2];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int c4 = 4 * (lane + 32 * k);
    a[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < P) {
      const float4 y = ld4(pre + c4), s = ld4(bn + 2 * P + c4), h = ld4(bn + 3 * P + c4);
      a[k].x = fmaxf(fmaf(y.x, s.x, h.x), 0.f); a[k].y = fmaxf(fmaf(y.y, s.y, h.y), 0.f);
      a[k].z = fmaxf(fmaf(y.z, s.z, h.z), 0.f); a[k].w = fmaxf(fmaf(y.w, s.w, h.w), 0.f);
      ss = fmaf(a[k].x, a[k].x, ss); ss = fmaf(a[k].y, a[k].y, ss);
      ss = fmaf(a[k].z, a[k].z, ss); ss = fmaf(a[k].w, a[k].w, ss);
    }
  }
  ss = warp_sum(ss);
  if constexpr (RAW) {
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c4 = 4 * (lane + 32 * k);
      if (c4 < P) st4(x + c4, a[k]);
    }
    if (lane == 0) *norm = ss;
  } else {
    const float nrm = sqrtf(ss), inv = sc / fmaxf(nrm, eps);
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c4 = 4 * (lane + 32 * k);
      if (c4 < P) st4(x + c4, make_float4(a[k].x * inv, a[k].y * inv, a[k].z * inv, a[k].w * inv));
    }
    if (lane == 0) *norm = nrm;
  }
}

template <bool RAW>
__global__ void __launch_bounds__(256) operands_kernel(const int32_t* __restrict__ inds, int64_t S, int P,
                                                       const float* __restrict__ pre_s, const float* __restrict__ bn_s,
                                                       const float* __restrict__ pre_t, const float* __restrict__ bn_t, float inv_T,
                                                       float eps, float* __restrict__ x_s, float* __restrict__ x_t,
                                                       float* __restrict__ norm_s, float* __restrict__ norm_t) {
  const int lane = threadIdx.x & 31;
  for (int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); j < S; j += (int64_t)gridDim.x * 8) {
    const int64_t r = __ldg(inds + j);
    operand_row<RAW>(pre_s + r * P, bn_s, P, inv_T, eps, x_s + j * P, norm_s + j, lane);
    operand_row<RAW>(pre_t + r * P, bn_t, P, 1.f, eps, x_t + j * P, norm_t + j, lane);
  }
}

// What g holds on the way back: the InfoNCE operand gradient itself (G-CRD), or dG . x of the GSP chunk loop, whose
// operand gradient is 2 dG . x (normalising path) or 2 dG . x + 4 rc[j] x (raw path: the distance's norm terms).
enum BwdMode { BWD_NCE = 0, BWD_GSP_NORM = 1, BWD_GSP_RAW = 2 };

// One head's way back over the sampled rows of warp gw: the operand gradient, normalise backward (the
// row_normalize_bwd_kernel formula; none on the raw path), the ReLU mask relu(bn(pre)) > 0, times beta -> dz stored to row
// inds[j] of the zero-filled [n_train, P] dz; the warp's column sums of dz and dz * xhat (pass 1 of the BatchNorm backward)
// go to part[gw][2][P].
template <int MODE>
__device__ __forceinline__ void head_bwd(int gw, int nw, int lane, const int32_t* __restrict__ inds, int64_t S, int P,
                                         const float* __restrict__ g, const float* __restrict__ x, const float* __restrict__ nrm_in,
                                         const float* __restrict__ rc, float sc, float eps, const float* __restrict__ pre,
                                         const float* __restrict__ bn, float beta, float* __restrict__ dz, float* __restrict__ part) {
  const float inv_sc = 1.f / sc;
  float4 s[2], q[2], mu[2], is[2], scl[2], shf[2];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int c4 = 4 * (lane + 32 * k);
    s[k] = q[k] = mu[k] = is[k] = scl[k] = shf[k] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c4 < P) { mu[k] = ld4(bn + c4); is[k] = ld4(bn + P + c4); scl[k] = ld4(bn + 2 * P + c4); shf[k] = ld4(bn + 3 * P + c4); }
  }
  for (int64_t j = gw; j < S; j += nw) {
    const int64_t r = __ldg(inds + j);
    float4 gv[2], xv[2];
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c4 = 4 * (lane + 32 * k);
      gv[k] = xv[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c4 < P) {
        gv[k] = ld4(g + j * P + c4); xv[k] = ld4(x + j * P + c4);
        if constexpr (MODE != BWD_NCE) { gv[k].x *= 2.f; gv[k].y *= 2.f; gv[k].z *= 2.f; gv[k].w *= 2.f; }
        if constexpr (MODE != BWD_GSP_RAW) {
          dot = fmaf(xv[k].x * inv_sc, gv[k].x, dot); dot = fmaf(xv[k].y * inv_sc, gv[k].y, dot);
          dot = fmaf(xv[k].z * inv_sc, gv[k].z, dot); dot = fmaf(xv[k].w * inv_sc, gv[k].w, dot);
        }
      }
    }
    float inv = 0.f, rcj = 0.f;
    bool clamped = false;
    if constexpr (MODE == BWD_GSP_RAW) {
      rcj = 4.f * __ldg(rc + j);
    } else {
      dot = warp_sum(dot);
      const float nr = __ldg(nrm_in + j);
      clamped = nr < eps;
      inv = sc / fmaxf(nr, eps);
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const int c4 = 4 * (lane + 32 * k);
      if (c4 >= P) continue;
      const float4 y = ld4(pre + r * P + c4);
      float d[4] = {gv[k].x, gv[k].y, gv[k].z, gv[k].w};
      const float xs[4] = {xv[k].x, xv[k].y, xv[k].z, xv[k].w}, ys[4] = {y.x, y.y, y.z, y.w};
      const float m4[4] = {mu[k].x, mu[k].y, mu[k].z, mu[k].w}, i4[4] = {is[k].x, is[k].y, is[k].z, is[k].w};
      const float a4[4] = {scl[k].x, scl[k].y, scl[k].z, scl[k].w}, b4[4] = {shf[k].x, shf[k].y, shf[k].z, shf[k].w};
      float ps[4] = {0.f, 0.f, 0.f, 0.f}, pq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float v;
        if constexpr (MODE == BWD_GSP_RAW) v = fmaf(rcj, xs[e], d[e]);
        else v = clamped ? d[e] * inv : inv * (d[e] - xs[e] * inv_sc * dot);
        d[e] = fmaf(ys[e], a4[e], b4[e]) > 0.f ? v * beta : 0.f;
        ps[e] = d[e];
        pq[e] = d[e] * ((ys[e] - m4[e]) * i4[e]);
      }
      st4(dz + r * P + c4, make_float4(d[0], d[1], d[2], d[3]));
      s[k].x += ps[0]; s[k].y += ps[1]; s[k].z += ps[2]; s[k].w += ps[3];
      q[k].x += pq[0]; q[k].y += pq[1]; q[k].z += pq[2]; q[k].w += pq[3];
    }
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int c4 = 4 * (lane + 32 * k);
    if (c4 < P) { st4(part + (size_t)gw * 2 * P + c4, s[k]); st4(part + (size_t)gw * 2 * P + P + c4, q[k]); }
  }
}

template <int MODE>
__global__ void __launch_bounds__(256) backward_kernel(const int32_t* __restrict__ inds, int64_t S, int P, const float* __restrict__ g_s,
                                                       const float* __restrict__ g_t, const float* __restrict__ x_s,
                                                       const float* __restrict__ x_t, const float* __restrict__ norm_s,
                                                       const float* __restrict__ norm_t, const float* __restrict__ rc_s,
                                                       const float* __restrict__ rc_t, float inv_T, float eps,
                                                       const float* __restrict__ pre_s, const float* __restrict__ bn_s,
                                                       const float* __restrict__ pre_t, const float* __restrict__ bn_t, float beta,
                                                       float* __restrict__ dz_s, float* __restrict__ dz_t, float* __restrict__ part_s,
                                                       float* __restrict__ part_t, const float* __restrict__ loss_aux,
                                                       float* __restrict__ loss_total) {
  const int lane = threadIdx.x & 31, gw = blockIdx.x * 8 + (threadIdx.x >> 5), nw = gridDim.x * 8;
  head_bwd<MODE>(gw, nw, lane, inds, S, P, g_s, x_s, norm_s, rc_s, inv_T, eps, pre_s, bn_s, beta, dz_s, part_s);
  head_bwd<MODE>(gw, nw, lane, inds, S, P, g_t, x_t, norm_t, rc_t, 1.f, eps, pre_t, bn_t, beta, dz_t, part_t);
  if (loss_total && blockIdx.x == 0 && threadIdx.x == 0) loss_total[0] += beta * loss_aux[0];
}

static inline int64_t al256(int64_t b) { return (b + 255) / 256 * 256; }

}  // namespace gcrd
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int64_t b200gnn_gcrd_sample_workspace_bytes(int64_t n) {
  if (n < 1) return B200GNN_ERR_BAD_ARG;
  const int64_t sort = b200gnn_graph_sort_workspace_bytes(n);
  if (sort < 0) return sort;
  return 2 * gcrd::al256(n * 8) + sort;
}

extern "C" int b200gnn_gcrd_sample_i32(int64_t n, uint64_t seed, uint64_t offset, const int32_t* step_dev, int32_t* perm_out,
                                       void* workspace, void* stream) {
  if (n < 1 || n >= INT32_MAX || !perm_out || !workspace) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* key = (int64_t*)workspace;
  int64_t* row = (int64_t*)((char*)workspace + gcrd::al256(n * 8));
  void* sort_ws = (char*)workspace + 2 * gcrd::al256(n * 8);
  int64_t g = (n + 255) / 256;
  if (g > 132 * 8) g = 132 * 8;
  gcrd::sample_keys_kernel<<<(int)g, 256, 0, st>>>(n, seed, offset, step_dev, key, row);
  int rc = check_launch();
  if (rc) return rc;
  return b200gnn_graph_argsort_i64(key, row, n, (int64_t)1 << 32, n, perm_out, sort_ws, stream);
}

extern "C" int b200gnn_gcrd_operands_f32(const int32_t* inds, int64_t S, int64_t P, const float* pre_s, const float* bn_s,
                                         const float* pre_t, const float* bn_t, float inv_T, float eps, float* x_s, float* x_t,
                                         float* norm_s, float* norm_t, void* stream) {
  if (!inds || S < 1 || P < 4 || P % 4 || P > gcrd::MAX_P || !pre_s || !bn_s || !pre_t || !bn_t || !x_s || !x_t || !norm_s ||
      !norm_t || !(inv_T > 0.f))
    return B200GNN_ERR_BAD_ARG;
  if (!aligned_to(pre_s, 16) || !aligned_to(pre_t, 16) || !aligned_to(bn_s, 16) || !aligned_to(bn_t, 16) || !aligned_to(x_s, 16) ||
      !aligned_to(x_t, 16))
    return B200GNN_ERR_BAD_ARG;
  int64_t g = (S + 7) / 8;
  if (g > 132 * 8) g = 132 * 8;
  gcrd::operands_kernel<false><<<(int)g, 256, 0, (cudaStream_t)stream>>>(inds, S, (int)P, pre_s, bn_s, pre_t, bn_t, inv_T, eps, x_s,
                                                                         x_t, norm_s, norm_t);
  return check_launch();
}

extern "C" int64_t b200gnn_gcrd_bwd_slots(void) { return gcrd::BWD_CTAS * 8; }

extern "C" int b200gnn_gcrd_backward_f32(const int32_t* inds, int64_t S, int64_t P, const float* g_s, const float* g_t,
                                         const float* x_s, const float* x_t, const float* norm_s, const float* norm_t, float inv_T,
                                         float eps, const float* pre_s, const float* bn_s, const float* pre_t, const float* bn_t,
                                         float beta, float* dz_s, float* dz_t, float* part_s, float* part_t, const float* loss_aux,
                                         float* loss_total, void* stream) {
  if (!inds || S < 1 || P < 4 || P % 4 || P > gcrd::MAX_P || !g_s || !g_t || !x_s || !x_t || !norm_s || !norm_t || !pre_s ||
      !bn_s || !pre_t || !bn_t || !dz_s || !dz_t || !part_s || !part_t || !(inv_T > 0.f) || (loss_total && !loss_aux))
    return B200GNN_ERR_BAD_ARG;
  const void* v4[] = {g_s, g_t, x_s, x_t, pre_s, pre_t, bn_s, bn_t, dz_s, dz_t, part_s, part_t};
  for (const void* p : v4)
    if (!aligned_to(p, 16)) return B200GNN_ERR_BAD_ARG;
  gcrd::backward_kernel<gcrd::BWD_NCE><<<gcrd::BWD_CTAS, 256, 0, (cudaStream_t)stream>>>(
      inds, S, (int)P, g_s, g_t, x_s, x_t, norm_s, norm_t, nullptr, nullptr, inv_T, eps, pre_s, bn_s, pre_t, bn_t, beta, dz_s, dz_t,
      part_s, part_t, loss_aux, loss_total);
  return check_launch();
}

// GSP over the same heads (kernel 0 cosine, 1 poly: normalising path, scale 1; 2 l2, 3 rbf: raw path).
extern "C" int b200gnn_gsp_operands_f32(const int32_t* inds, int64_t S, int64_t P, int kernel, const float* pre_s, const float* bn_s,
                                        const float* pre_t, const float* bn_t, float eps, float* x_s, float* x_t, float* norm_s,
                                        float* norm_t, void* stream) {
  if (!inds || S < 1 || P < 4 || P % 4 || P > gcrd::MAX_P || kernel < 0 || kernel > 3 || !pre_s || !bn_s || !pre_t || !bn_t ||
      !x_s || !x_t || !norm_s || !norm_t || !(eps > 0.f))
    return B200GNN_ERR_BAD_ARG;
  const void* v4[] = {pre_s, pre_t, bn_s, bn_t, x_s, x_t};
  for (const void* p : v4)
    if (!aligned_to(p, 16)) return B200GNN_ERR_BAD_ARG;
  int64_t g = (S + 7) / 8;
  if (g > 132 * 8) g = 132 * 8;
  if (kernel >= 2)
    gcrd::operands_kernel<true><<<(int)g, 256, 0, (cudaStream_t)stream>>>(inds, S, (int)P, pre_s, bn_s, pre_t, bn_t, 1.f, eps, x_s, x_t,
                                                                          norm_s, norm_t);
  else
    gcrd::operands_kernel<false><<<(int)g, 256, 0, (cudaStream_t)stream>>>(inds, S, (int)P, pre_s, bn_s, pre_t, bn_t, 1.f, eps, x_s,
                                                                           x_t, norm_s, norm_t);
  return check_launch();
}

extern "C" int b200gnn_gsp_backward_f32(const int32_t* inds, int64_t S, int64_t P, int kernel, const float* g_s, const float* g_t,
                                        const float* x_s, const float* x_t, const float* norm_s, const float* norm_t,
                                        const float* rc_s, const float* rc_t, float eps, const float* pre_s, const float* bn_s,
                                        const float* pre_t, const float* bn_t, float beta, float* dz_s, float* dz_t, float* part_s,
                                        float* part_t, const float* loss_aux, float* loss_total, void* stream) {
  if (!inds || S < 1 || P < 4 || P % 4 || P > gcrd::MAX_P || kernel < 0 || kernel > 3 || !g_s || !g_t || !x_s || !x_t || !pre_s ||
      !bn_s || !pre_t || !bn_t || !dz_s || !dz_t || !part_s || !part_t || !(eps > 0.f) || (loss_total && !loss_aux))
    return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2 ? (!rc_s || !rc_t) : (!norm_s || !norm_t)) return B200GNN_ERR_BAD_ARG;
  const void* v4[] = {g_s, g_t, x_s, x_t, pre_s, pre_t, bn_s, bn_t, dz_s, dz_t, part_s, part_t};
  for (const void* p : v4)
    if (!aligned_to(p, 16)) return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2)
    gcrd::backward_kernel<gcrd::BWD_GSP_RAW><<<gcrd::BWD_CTAS, 256, 0, (cudaStream_t)stream>>>(
        inds, S, (int)P, g_s, g_t, x_s, x_t, norm_s, norm_t, rc_s, rc_t, 1.f, eps, pre_s, bn_s, pre_t, bn_t, beta, dz_s, dz_t,
        part_s, part_t, loss_aux, loss_total);
  else
    gcrd::backward_kernel<gcrd::BWD_GSP_NORM><<<gcrd::BWD_CTAS, 256, 0, (cudaStream_t)stream>>>(
        inds, S, (int)P, g_s, g_t, x_s, x_t, norm_s, norm_t, rc_s, rc_t, 1.f, eps, pre_s, bn_s, pre_t, bn_t, beta, dz_s, dz_t,
        part_s, part_t, loss_aux, loss_total);
  return check_launch();
}
