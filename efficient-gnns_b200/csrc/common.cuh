// Shared helpers for the b200gnn kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200gnn.h"

namespace b200gnn {

// Per-thread last CUDA error text + process-wide launch counter (capi.cu).
void set_cuda_error(cudaError_t e);
void count_launch(int n = 1);

inline int check_launch() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_cuda_error(e);
    return B200GNN_ERR_CUDA;
  }
  count_launch();
  return B200GNN_OK;
}

constexpr unsigned FULL_MASK = 0xffffffffu;

// One element of torch.optim.Adam (no amsgrad, no weight decay); step_size = lr / (1 - b1^t), inv_sqrt_bc2 = rsqrt(1 - b2^t).
// Shared by the flat-buffer Adam and the embedding-table Adam, which must agree bit for bit.
__device__ __forceinline__ void adam_update(float& p, float& m, float& v, float g, float b1, float b2, float eps,
                                            float step_size, float inv_sqrt_bc2) {
  const float mi = b1 * m + (1.f - b1) * g;
  const float vi = b2 * v + (1.f - b2) * g * g;
  m = mi; v = vi;
  p -= step_size * mi / (sqrtf(vi) * inv_sqrt_bc2 + eps);
}

// ---- small vector algebra so kernels can be written once over float/float2/float4
template <typename V> struct VecTraits;
template <> struct VecTraits<float> { static constexpr int W = 1; };
template <> struct VecTraits<float2> { static constexpr int W = 2; };
template <> struct VecTraits<float4> { static constexpr int W = 4; };

__device__ __forceinline__ void vzero(float& a) { a = 0.f; }
__device__ __forceinline__ void vzero(float2& a) { a.x = a.y = 0.f; }
__device__ __forceinline__ void vzero(float4& a) { a.x = a.y = a.z = a.w = 0.f; }

__device__ __forceinline__ void vfma(float& acc, float s, const float& x) { acc = fmaf(s, x, acc); }
__device__ __forceinline__ void vfma(float2& acc, float s, const float2& x) {
  acc.x = fmaf(s, x.x, acc.x); acc.y = fmaf(s, x.y, acc.y);
}
__device__ __forceinline__ void vfma(float4& acc, float s, const float4& x) {
  acc.x = fmaf(s, x.x, acc.x); acc.y = fmaf(s, x.y, acc.y);
  acc.z = fmaf(s, x.z, acc.z); acc.w = fmaf(s, x.w, acc.w);
}
__device__ __forceinline__ void vadd(float& a, const float& b) { a += b; }
__device__ __forceinline__ void vadd(float2& a, const float2& b) { a.x += b.x; a.y += b.y; }
__device__ __forceinline__ void vadd(float4& a, const float4& b) {
  a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
}
__device__ __forceinline__ void vdiv(float& a, float d) { a /= d; }
__device__ __forceinline__ void vdiv(float2& a, float d) { a.x /= d; a.y /= d; }
__device__ __forceinline__ void vdiv(float4& a, float d) { a.x /= d; a.y /= d; a.z /= d; a.w /= d; }
// acc += y ; accsq += y*y
__device__ __forceinline__ void vstat(float& s, float& q, const float& y) { s += y; q = fmaf(y, y, q); }
__device__ __forceinline__ void vstat(float2& s, float2& q, const float2& y) {
  s.x += y.x; s.y += y.y; q.x = fmaf(y.x, y.x, q.x); q.y = fmaf(y.y, y.y, q.y);
}
__device__ __forceinline__ void vstat(float4& s, float4& q, const float4& y) {
  s.x += y.x; s.y += y.y; s.z += y.z; s.w += y.w;
  q.x = fmaf(y.x, y.x, q.x); q.y = fmaf(y.y, y.y, q.y);
  q.z = fmaf(y.z, y.z, q.z); q.w = fmaf(y.w, y.w, q.w);
}

__device__ __forceinline__ float vshfl_down(float v, int d) { return __shfl_down_sync(FULL_MASK, v, d); }
__device__ __forceinline__ float2 vshfl_down(float2 v, int d) {
  return make_float2(__shfl_down_sync(FULL_MASK, v.x, d), __shfl_down_sync(FULL_MASK, v.y, d));
}
__device__ __forceinline__ float4 vshfl_down(float4 v, int d) {
  return make_float4(__shfl_down_sync(FULL_MASK, v.x, d), __shfl_down_sync(FULL_MASK, v.y, d),
                     __shfl_down_sync(FULL_MASK, v.z, d), __shfl_down_sync(FULL_MASK, v.w, d));
}

// Read-only 128/64/32-bit gathers (ld.global.nc): X rows are immutable for the
// duration of the kernel; hub rows stay hot in L1.
__device__ __forceinline__ float vldg(const float* p) { return __ldg(p); }
__device__ __forceinline__ float2 vldg(const float2* p) { return __ldg(p); }
__device__ __forceinline__ float4 vldg(const float4* p) { return __ldg(p); }

// Streaming stores (st.global.cs): outputs are written once and consumed by a
// later kernel; keep them from evicting the gathered operand out of L2.
__device__ __forceinline__ void vstcs(float* p, const float& v) { __stcs(p, v); }
__device__ __forceinline__ void vstcs(float2* p, const float2& v) { __stcs(p, v); }
__device__ __forceinline__ void vstcs(float4* p, const float4& v) { __stcs(p, v); }

// out[0] = scale * sum(partial[0..n))   (one CTA, fp64, fixed order); one copy per translation unit
static __global__ void __launch_bounds__(256) sum_partials_kernel(const float* __restrict__ partial, int n, double scale,
                                                                  float* __restrict__ out) {
  __shared__ double s[256];
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += 256) a += (double)partial[i];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int d = 128; d > 0; d >>= 1) {
    if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(s[0] * scale);
}

inline bool aligned_to(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

}  // namespace b200gnn
