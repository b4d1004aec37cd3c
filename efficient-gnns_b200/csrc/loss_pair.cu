// Building blocks of the feature-distillation criteria of arxiv_pyg/criterion.py (fitnet :24-36, AT :39-54,
// GSP/gpw :57-92, G-CRD/nce :129-149).  The S x S contractions themselves run on the wgmma GEMM
// (gemm_tf32x3.cu); the kernels here are the row / element passes around them, each producing the forward value
// and the tensor the backward GEMM needs in the same pass.  Loss scalars are reduced deterministically
// (per-CTA partials, fixed-order finalize).
#include "common.cuh"

namespace b200gnn {

__device__ __forceinline__ float warp_sum_f(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}
__device__ __forceinline__ float warp_max_f(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, d));
  return v;
}

// block-level deterministic sum of one float per thread -> partial[blockIdx.x]
__device__ __forceinline__ void block_sum_store(float v, float* partial) {
  __shared__ float s[32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  v = warp_sum_f(v);
  if (lane == 0) s[warp] = v;
  __syncthreads();
  if (warp == 0) {
    float t = lane < (int)(blockDim.x >> 5) ? s[lane] : 0.f;
    t = warp_sum_f(t);
    if (lane == 0) partial[blockIdx.x] = t;
  }
}

// ---------------------------------------------------------------- F.normalize(x, p=2, dim=-1)  (eps = 1e-12)
// warp per row; out = x / max(||x||, eps); norm_out[row] = ||x||
__global__ void __launch_bounds__(256) row_normalize_fwd_kernel(const float* __restrict__ x, int64_t n, int F, float eps,
                                                                float scale, float* __restrict__ out,
                                                                float* __restrict__ norm_out) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * 8) {
    const float* xr = x + (size_t)r * F;
    float ss = 0.f;
    for (int k = lane; k < F; k += 32) { const float v = xr[k]; ss = fmaf(v, v, ss); }
    ss = warp_sum_f(ss);
    const float nrm = sqrtf(ss);
    const float inv = scale / fmaxf(nrm, eps);
    float* o = out + (size_t)r * F;
    for (int k = lane; k < F; k += 32) o[k] = xr[k] * inv;
    if (lane == 0 && norm_out) norm_out[r] = nrm;
  }
}
// d_x = scale/max(norm,eps) * (d_out - u * (u . d_out))   with u = x/max(norm,eps) (= out/scale);
// rows with norm < eps are in the clamped regime: d_x = d_out * scale/eps.
__global__ void __launch_bounds__(256) row_normalize_bwd_kernel(const float* __restrict__ out, const float* __restrict__ norm,
                                                                const float* __restrict__ d_out, int64_t n, int F,
                                                                float eps, float scale, float* __restrict__ d_x,
                                                                int accumulate) {
  const int lane = threadIdx.x & 31;
  const float inv_scale = 1.f / scale;
  for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * 8) {
    const float* o = out + (size_t)r * F;
    const float* g = d_out + (size_t)r * F;
    float dot = 0.f;
    for (int k = lane; k < F; k += 32) dot = fmaf(o[k] * inv_scale, g[k], dot);
    dot = warp_sum_f(dot);
    const float nrm = norm[r];
    const bool clamped = nrm < eps;
    const float inv = scale / fmaxf(nrm, eps);
    float* dx = d_x + (size_t)r * F;
    for (int k = lane; k < F; k += 32) {
      const float v = clamped ? g[k] * inv : inv * (g[k] - o[k] * inv_scale * dot);
      dx[k] = accumulate ? dx[k] + v : v;
    }
  }
}

// ---------------------------------------------------------------- F.mse_loss(a, b) with d_a = 2 (a-b) w / numel
__global__ void __launch_bounds__(256) mse_fwd_bwd_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                          int64_t n, float grad_scale, float* __restrict__ d_a,
                                                          float* __restrict__ partial) {
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float d = a[i] - b[i];
    acc = fmaf(d, d, acc);
    if (d_a) d_a[i] = grad_scale * d;
  }
  block_sum_store(acc, partial);
}

// row squared norms  out[r] = sum_k x[r,k]^2  (attention transfer, criterion.py:44-45); d_x = 2 x * d_out[r]
__global__ void __launch_bounds__(256) row_sqnorm_kernel(const float* __restrict__ x, int64_t n, int F, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * 8) {
    const float* xr = x + (size_t)r * F;
    float ss = 0.f;
    for (int k = lane; k < F; k += 32) { const float v = xr[k]; ss = fmaf(v, v, ss); }
    ss = warp_sum_f(ss);
    if (lane == 0) out[r] = ss;
  }
}
__global__ void __launch_bounds__(256) row_sqnorm_bwd_kernel(const float* __restrict__ x, const float* __restrict__ d_out,
                                                             int64_t n, int F, float* __restrict__ d_x) {
  const int64_t total = n * (int64_t)F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    d_x[i] = 2.f * x[i] * d_out[i / F];
}

// ---------------------------------------------------------------- G-CRD rows: InfoNCE over Z = (fs_n ft_n^T) / tau
// One CTA per row i of the S x S logits (already divided by tau through the operand scale):
//   loss_i = logsumexp_j Z_ij - Z_ii ;   Z_ij <- (softmax_j(Z_i) - [i==j]) * w      (w = 1/S: d loss / d Z in place)
// Chunked form: Z holds rows [row_offset, row_offset + gridDim.x) of the S x S logits (row-major, S columns); the positive
// of local row r is column row_offset + r.  partial is indexed by the GLOBAL row.
__global__ void __launch_bounds__(256) nce_rows_kernel(float* __restrict__ Z, int S, float w, float* __restrict__ partial,
                                                       int row_offset, int64_t ldz) {
  __shared__ float s_red[32];
  __shared__ float s_bc[2];
  const int row = blockIdx.x + row_offset;
  float* z = Z + (size_t)blockIdx.x * ldz;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float m = -INFINITY;
  for (int j = threadIdx.x; j < S; j += blockDim.x) m = fmaxf(m, z[j]);
  m = warp_max_f(m);
  if (lane == 0) s_red[warp] = m;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? s_red[lane] : -INFINITY; t = warp_max_f(t); if (lane == 0) s_bc[0] = t; }
  __syncthreads();
  m = s_bc[0];
  float se = 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) se += expf(z[j] - m);
  se = warp_sum_f(se);
  __syncthreads();
  if (lane == 0) s_red[warp] = se;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) s_bc[1] = t; }
  __syncthreads();
  const float lse = m + logf(s_bc[1]);
  const float zii = z[row];
  __syncthreads();
  for (int j = threadIdx.x; j < S; j += blockDim.x) z[j] = (expf(z[j] - lse) - (j == row ? 1.f : 0.f)) * w;
  if (threadIdx.x == 0) partial[row] = lse - zii;
}

// ---------------------------------------------------------------- tiled transpose  out[c][r] = in[r][c]
// gridDim.y is capped at 65,535 row tiles (2,097,120 rows), so each CTA walks its row tiles with a grid stride.
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ in, int64_t rows, int64_t cols,
                                                        float* __restrict__ out) {
  __shared__ float tile[32][33];
  const int64_t c0 = (int64_t)blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int64_t r0 = (int64_t)blockIdx.y * 32; r0 < rows; r0 += (int64_t)gridDim.y * 32) {
    for (int i = ty; i < 32; i += 8)
      if (r0 + i < rows && c0 + tx < cols) tile[i][tx] = in[(size_t)(r0 + i) * cols + c0 + tx];
    __syncthreads();
    for (int i = ty; i < 32; i += 8)
      if (c0 + i < cols && r0 + tx < rows) out[(size_t)(c0 + i) * rows + r0 + tx] = tile[tx][i];
    __syncthreads();   // the tile is refilled by the next row tile
  }
}

// ---------------------------------------------------------------- GSP: pairwise-similarity MSE
// Gs = fs fs^T, Gt = ft ft^T  (S x S Gram matrices from the GEMM; for cosine/poly the operands were normalised).
// kernel: 0 cosine  sim = G ; 1 poly  sim = G^2 ; 2 l2  sim = sqrt(max(ni + nj - 2G, 0)) ; 3 rbf  sim = exp(-0.5 (ni+nj-2G))
// loss = mean (sim_s - sim_t)^2 ;  Gs <- d loss / d Gs  (so that  d fs = (dG + dG^T) fs = 2 dG fs, dG symmetric),
// and for l2/rbf rc_s[i] = sum_j d loss/d(ni)  (the norm terms of the distance).
// Row-chunk form: Gs / Gt hold rows [row0, row0 + gridDim.x) of the two S x S matrices at row pitch ld >= S; the l2/rbf
// diagonal and the ns[i] / nt[i] lookups use the global row, partial[] and rc_*[] are stored at it, and columns S..ld-1
// are set to zero (so a GEMM may contract over the padded pitch).  BOTH: Gt <- d loss / d Gt in the same pass, with the
// teacher's own coefficient sums in rc_t; its expressions are the student's with the roles of the two sides swapped, so
// the result is that of a second one-sided pass on (Gt, Gs, nt, ns).
template <bool BOTH>
__global__ void __launch_bounds__(256) gsp_pair_kernel(float* __restrict__ Gs, float* __restrict__ Gt, int64_t ld, int S,
                                                       int row0, const float* __restrict__ ns, const float* __restrict__ nt,
                                                       int kernel, float w /* 2 / S^2 */, float* __restrict__ rc_s,
                                                       float* __restrict__ rc_t, float* __restrict__ partial) {
  __shared__ float s_red[32];
  const int row = row0 + blockIdx.x;
  float* gs = Gs + (size_t)blockIdx.x * ld;
  float* gt = Gt + (size_t)blockIdx.x * ld;
  float acc = 0.f, rs = 0.f, rt = 0.f;
  const float nsi = (kernel >= 2) ? ns[row] : 0.f, nti = (kernel >= 2) ? nt[row] : 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    float ss, st, ds_dg, dt_dg, ds_dn = 0.f, dt_dn = 0.f;   // d sim / d G_ij , d sim / d n_i (= d/d n_j), per side
    const float a = gs[j], b = gt[j];
    if (kernel == 0) { ss = a; st = b; ds_dg = 1.f; dt_dg = 1.f; }
    else if (kernel == 1) { ss = a * a; st = b * b; ds_dg = 2.f * a; dt_dg = 2.f * b; }
    else {
      float d2s = fmaxf(nsi + ns[j] - 2.f * a, 0.f), d2t = fmaxf(nti + nt[j] - 2.f * b, 0.f);
      if (j == row) { d2s = 0.f; d2t = 0.f; }
      if (kernel == 2) {
        ss = sqrtf(d2s); st = sqrtf(d2t);
        const float inv_s = ss > 0.f ? 0.5f / ss : 0.f;   // d sqrt(d2)/d d2, sub-gradient 0 at 0 (torch .norm backward)
        const float inv_t = st > 0.f ? 0.5f / st : 0.f;
        ds_dg = -2.f * inv_s; ds_dn = inv_s;
        dt_dg = -2.f * inv_t; dt_dn = inv_t;
      } else {
        ss = expf(-0.5f * d2s); st = expf(-0.5f * d2t);
        ds_dg = ss; ds_dn = -0.5f * ss;
        dt_dg = st; dt_dn = -0.5f * st;
      }
    }
    const float diff = ss - st;
    acc = fmaf(diff, diff, acc);
    const float g = w * diff;                 // d loss / d sim_s
    gs[j] = g * ds_dg;
    rs += g * ds_dn;
    if (BOTH) {
      const float diff_t = st - ss;
      const float g_t = w * diff_t;           // d loss / d sim_t
      gt[j] = g_t * dt_dg;
      rt += g_t * dt_dn;
    }
  }
  for (int64_t j = (int64_t)S + threadIdx.x; j < ld; j += blockDim.x) {
    gs[j] = 0.f;
    if (BOTH) gt[j] = 0.f;
  }
  // block reductions (deterministic)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  acc = warp_sum_f(acc); rs = warp_sum_f(rs);
  if (BOTH) rt = warp_sum_f(rt);
  if (lane == 0) s_red[warp] = acc;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) partial[row] = t; }
  __syncthreads();
  if (lane == 0) s_red[warp] = rs;
  __syncthreads();
  if (warp == 0 && rc_s) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) rc_s[row] = t; }
  if (BOTH) {
    __syncthreads();
    if (lane == 0) s_red[warp] = rt;
    __syncthreads();
    if (warp == 0 && rc_t) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) rc_t[row] = t; }
  }
}

// d fs[i,:] += coef[i] * fs[i,:]     (norm terms of l2 / rbf:  d n_i / d fs_i = 2 fs_i, coefficient folded by the caller)
__global__ void __launch_bounds__(256) row_axpy_kernel(const float* __restrict__ x, const float* __restrict__ coef, int64_t n,
                                                       int F, float alpha, float* __restrict__ y) {
  const int64_t total = n * (int64_t)F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = fmaf(alpha * coef[i / F], x[i], y[i]);
}

// F.binary_cross_entropy_with_logits(z, t) (ppi_pyg/criterion.py:11,13): element loss max(z,0) - z t + log1p(exp(-|z|)),
// mean over all elements; d z = (sigmoid(z) - t) * w.  target_is_logits: t = sigmoid(target) (the teacher term of :13).
__global__ void __launch_bounds__(256) bce_logits_kernel(const float* __restrict__ z, const float* __restrict__ target,
                                                         int target_is_logits, int64_t n, float w, float* __restrict__ dz,
                                                         float* __restrict__ partial) {
  __shared__ float s_red[8];
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float x = z[i];
    float t = target[i];
    if (target_is_logits) t = 1.f / (1.f + expf(-t));
    acc += fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
    if (dz) dz[i] = (1.f / (1.f + expf(-x)) - t) * w;
  }
  acc = warp_sum_f(acc);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_red[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < 8; ++k) t += s_red[k];
    partial[blockIdx.x] = t;
  }
}

static inline int ew_grid(int64_t n, int per = 256 * 4) {
  int64_t g = (n + per - 1) / per;
  if (g > 132 * 8) g = 132 * 8;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_row_normalize_fwd_f32(const float* x, int64_t n, int64_t F, float eps, float scale, float* out,
                                             float* norm_out, void* stream) {
  if (!x || !out || n < 0 || F <= 0 || eps <= 0.f) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  row_normalize_fwd_kernel<<<ew_grid(n, 8), 256, 0, (cudaStream_t)stream>>>(x, n, (int)F, eps, scale, out, norm_out);
  return check_launch();
}
extern "C" int b200gnn_row_normalize_bwd_f32(const float* out, const float* norm, const float* d_out, int64_t n, int64_t F,
                                             float eps, float scale, float* d_x, int accumulate, void* stream) {
  if (!out || !norm || !d_out || !d_x || n < 0 || F <= 0 || eps <= 0.f) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  row_normalize_bwd_kernel<<<ew_grid(n, 8), 256, 0, (cudaStream_t)stream>>>(out, norm, d_out, n, (int)F, eps, scale, d_x,
                                                                           accumulate);
  return check_launch();
}

extern "C" int64_t b200gnn_reduce_slots(int64_t n) { return ew_grid(n); }

// loss_out[0] = mean((a-b)^2); d_a (nullable) = grad_weight * 2 (a-b) / n
extern "C" int b200gnn_mse_fwd_bwd_f32(const float* a, const float* b, int64_t n, float grad_weight, float* d_a,
                                       float* loss_out, float* partial, void* stream) {
  if (!a || !b || !loss_out || !partial || n <= 0) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ew_grid(n);
  int rc;
  mse_fwd_bwd_kernel<<<grid, 256, 0, st>>>(a, b, n, grad_weight * 2.f / (float)n, d_a, partial);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, grid, 1.0 / (double)n, loss_out);
  return check_launch();
}

// loss_out[0] = mean BCE-with-logits; d_z (nullable) = grad_weight * (sigmoid(z) - t) / n
extern "C" int b200gnn_bce_logits_fwd_bwd_f32(const float* z, const float* target, int target_is_logits, int64_t n,
                                              float grad_weight, float* d_z, float* loss_out, float* partial, void* stream) {
  if (!z || !target || !loss_out || !partial || n <= 0) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = ew_grid(n);
  int rc;
  bce_logits_kernel<<<grid, 256, 0, st>>>(z, target, target_is_logits, n, grad_weight / (float)n, d_z, partial);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, grid, 1.0 / (double)n, loss_out);
  return check_launch();
}

extern "C" int b200gnn_row_sqnorm_f32(const float* x, int64_t n, int64_t F, float* out, void* stream) {
  if (!x || !out || n < 0 || F <= 0) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  row_sqnorm_kernel<<<ew_grid(n, 8), 256, 0, (cudaStream_t)stream>>>(x, n, (int)F, out);
  return check_launch();
}
extern "C" int b200gnn_row_sqnorm_bwd_f32(const float* x, const float* d_out, int64_t n, int64_t F, float* d_x, void* stream) {
  if (!x || !d_out || !d_x || n < 0 || F <= 0) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  row_sqnorm_bwd_kernel<<<ew_grid(n * F), 256, 0, (cudaStream_t)stream>>>(x, d_out, n, (int)F, d_x);
  return check_launch();
}

// Z[S,S] in: logits (already / tau); out: d loss / d Z.  loss_out[0] = mean_i (logsumexp_j Z_ij - Z_ii).  partial: float[S].
extern "C" int b200gnn_nce_rows_f32(float* Z, int64_t S, float* loss_out, float* partial, void* stream) {
  if (!Z || !loss_out || !partial || S <= 0 || S >= INT32_MAX) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  nce_rows_kernel<<<(int)S, 256, 0, st>>>(Z, (int)S, 1.f / (float)S, partial, 0, S);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, (int)S, 1.0 / (double)S, loss_out);
  return check_launch();
}

// Row chunk of the same pass: Z = rows [row_offset, row_offset + n_rows) of the S x S logits, row pitch ldz >= S floats
// (columns S..ldz-1 are padding and are left untouched).
// The S x S matrix never exists: the caller streams chunks small enough to stay in L2 (GEMM -> this pass -> the two
// backward GEMMs), then b200gnn_nce_finish_f32 turns partial[S] into the loss.
extern "C" int b200gnn_nce_rows_chunk_f32(float* Z, int64_t ldz, int64_t n_rows, int64_t S, int64_t row_offset, float* partial,
                                          void* stream) {
  if (!Z || !partial || S <= 0 || S >= INT32_MAX || ldz < S || n_rows <= 0 || row_offset < 0 || row_offset + n_rows > S)
    return B200GNN_ERR_BAD_ARG;
  nce_rows_kernel<<<(int)n_rows, 256, 0, (cudaStream_t)stream>>>(Z, (int)S, 1.f / (float)S, partial, (int)row_offset, ldz);
  return check_launch();
}

extern "C" int b200gnn_nce_finish_f32(const float* partial, int64_t S, float* loss_out, void* stream) {
  if (!partial || !loss_out || S <= 0 || S >= INT32_MAX) return B200GNN_ERR_BAD_ARG;
  sum_partials_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(partial, (int)S, 1.0 / (double)S, loss_out);
  return check_launch();
}

extern "C" int b200gnn_transpose_f32(const float* in, int64_t rows, int64_t cols, float* out, void* stream) {
  if (!in || !out || rows <= 0 || cols <= 0) return B200GNN_ERR_BAD_ARG;
  const int64_t row_tiles = (rows + 31) / 32;
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)(row_tiles < 65535 ? row_tiles : 65535));
  transpose_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(in, rows, cols, out);
  return check_launch();
}

// Gs (in: student Gram, out: d loss / d Gs), Gt teacher Gram, ns/nt row squared norms (l2 / rbf only), rowcoef[S] out
// (l2 / rbf only: sum_j d loss / d n_i over row i; the caller doubles it for the symmetric j-side).  partial: float[S].
extern "C" int b200gnn_gsp_pair_f32(float* Gs, const float* Gt, const float* ns, const float* nt, int64_t S, int kernel,
                                    float* rowcoef, float* loss_out, float* partial, void* stream) {
  if (!Gs || !Gt || !loss_out || !partial || S <= 0 || S >= INT32_MAX || kernel < 0 || kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2 && (!ns || !nt || !rowcoef)) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  const double n2 = (double)S * (double)S;
  // the one-sided pass never stores to Gt
  gsp_pair_kernel<false><<<(int)S, 256, 0, st>>>(Gs, const_cast<float*>(Gt), S, (int)S, 0, ns, nt, kernel, (float)(2.0 / n2),
                                                 rowcoef, nullptr, partial);
  if ((rc = check_launch())) return rc;
  sum_partials_kernel<<<1, 256, 0, st>>>(partial, (int)S, 1.0 / n2, loss_out);
  return check_launch();
}

// Both gradients of a row chunk in one pass: Gs / Gt rows [row_offset, row_offset + n_rows) of the two S x S Gram
// matrices (row pitch ld >= S, a multiple of 4 when a GEMM reads them back), overwritten by d loss / d Gs and d loss / d Gt;
// columns S..ld-1 are set to zero.  partial[S] and (l2 / rbf) rc_s[S] / rc_t[S] are stored at the global rows, so
// b200gnn_gsp_finish_f32 gives the same loss bits for any chunking.
extern "C" int b200gnn_gsp_pair_chunk_f32(float* Gs, float* Gt, int64_t ld, int64_t n_rows, int64_t S, int64_t row_offset,
                                          const float* ns, const float* nt, int kernel, float* rc_s, float* rc_t, float* partial,
                                          void* stream) {
  if (!Gs || !Gt || !partial || S <= 0 || S >= INT32_MAX || ld < S || n_rows <= 0 || row_offset < 0 ||
      row_offset + n_rows > S || kernel < 0 || kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2 && (!ns || !nt || !rc_s || !rc_t)) return B200GNN_ERR_BAD_ARG;
  const double n2 = (double)S * (double)S;
  gsp_pair_kernel<true><<<(int)n_rows, 256, 0, (cudaStream_t)stream>>>(Gs, Gt, ld, (int)S, (int)row_offset, ns, nt, kernel,
                                                                      (float)(2.0 / n2), rc_s, rc_t, partial);
  return check_launch();
}

// loss_out[0] = sum(partial[0..S)) / S^2: the GSP loss from the chunk passes' partials.
extern "C" int b200gnn_gsp_finish_f32(const float* partial, int64_t S, float* loss_out, void* stream) {
  if (!partial || !loss_out || S <= 0 || S >= INT32_MAX) return B200GNN_ERR_BAD_ARG;
  const double n2 = (double)S * (double)S;
  sum_partials_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(partial, (int)S, 1.0 / n2, loss_out);
  return check_launch();
}

extern "C" int b200gnn_row_axpy_f32(const float* x, const float* coef, int64_t n, int64_t F, float alpha, float* y,
                                    void* stream) {
  if (!x || !coef || !y || n < 0 || F <= 0) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  row_axpy_kernel<<<ew_grid(n * F), 256, 0, (cudaStream_t)stream>>>(x, coef, n, (int)F, alpha, y);
  return check_launch();
}
