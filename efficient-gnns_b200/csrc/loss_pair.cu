// Building blocks of the feature-distillation criteria of arxiv_pyg/criterion.py (fitnet :24-36, AT :39-54,
// GSP/gpw :57-92, G-CRD/nce :129-149).  The S x S contractions themselves run on the wgmma GEMM
// (gemm_tf32x3.cu), except the narrow GSP contraction dG . x of a few-feature student (gsp_contract_kernel); the other
// kernels here are the row / element passes around them, each producing the forward value
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

// ---------------------------------------------------------------- row helpers
// Shared by the row passes below and the GSP rows passes, so that a fused pass computes what the eager sequence of
// row_normalize / row_sqnorm / row_axpy computes, bit for bit.  A warp owns a row; lane l visits columns l, l + 32, ...

// sum_k x[k]^2 of one row: each lane's columns in order, then the warp's butterfly
__device__ __forceinline__ float row_sumsq(const float* __restrict__ xr, int F, int lane) {
  float ss = 0.f;
  for (int k = lane; k < F; k += 32) { const float v = xr[k]; ss = fmaf(v, v, ss); }
  return warp_sum_f(ss);
}
// o = xr * scale / max(||xr||, eps); returns ||xr||
__device__ __forceinline__ float normalize_row(const float* __restrict__ xr, int F, float eps, float scale, float* __restrict__ o,
                                               int lane) {
  const float nrm = sqrtf(row_sumsq(xr, F, lane));
  const float inv = scale / fmaxf(nrm, eps);
  for (int k = lane; k < F; k += 32) o[k] = xr[k] * inv;
  return nrm;
}
// u . d_out of the normalise backward (u = out / scale); d(k) loads d_out[k]
template <class D>
__device__ __forceinline__ float normalize_bwd_dot(const float* __restrict__ o, D d, int F, float inv_scale, int lane) {
  float dot = 0.f;
  for (int k = lane; k < F; k += 32) dot = fmaf(o[k] * inv_scale, d(k), dot);
  return warp_sum_f(dot);
}
// one element of the normalise backward: inv = scale / max(norm, eps), clamped = norm < eps
__device__ __forceinline__ float normalize_bwd_elem(float o, float d, float inv_scale, float dot, float inv, bool clamped) {
  return clamped ? d * inv : inv * (d - o * inv_scale * dot);
}
// y + alpha * coef * x (row_axpy's element)
__device__ __forceinline__ float axpy_elem(float alpha, float coef, float x, float y) { return fmaf(alpha * coef, x, y); }

// ---------------------------------------------------------------- F.normalize(x, p=2, dim=-1)  (eps = 1e-12)
// warp per row; out = x / max(||x||, eps); norm_out[row] = ||x||
__global__ void __launch_bounds__(256) row_normalize_fwd_kernel(const float* __restrict__ x, int64_t n, int F, float eps,
                                                                float scale, float* __restrict__ out,
                                                                float* __restrict__ norm_out) {
  const int lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < n; r += (int64_t)gridDim.x * 8) {
    const float nrm = normalize_row(x + (size_t)r * F, F, eps, scale, out + (size_t)r * F, lane);
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
    const float dot = normalize_bwd_dot(o, [g](int k) { return g[k]; }, F, inv_scale, lane);
    const float nrm = norm[r];
    const bool clamped = nrm < eps;
    const float inv = scale / fmaxf(nrm, eps);
    float* dx = d_x + (size_t)r * F;
    for (int k = lane; k < F; k += 32) {
      const float v = normalize_bwd_elem(o[k], g[k], inv_scale, dot, inv, clamped);
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
    const float ss = row_sumsq(x + (size_t)r * F, F, lane);
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
//
// The similarity of one pair, shared by the pair passes and the similarity builder: from the Gram entry G_ij and (l2 / rbf)
// the squared norms n_i, n[j] (read only for l2 / rbf), sim and its derivatives d sim / d G_ij and d sim / d n_i
// (= d / d n_j).  diag: i == j, whose l2 / rbf distance is exactly 0 whatever rounding left in n_i + n_j - 2 G_ii.
struct PairSim {
  float sim, d_g, d_n;
};
__device__ __forceinline__ PairSim gsp_sim(int kernel, float g, float ni, const float* __restrict__ n, int j, bool diag) {
  PairSim p;
  p.d_n = 0.f;
  if (kernel == 0) { p.sim = g; p.d_g = 1.f; }
  else if (kernel == 1) { p.sim = g * g; p.d_g = 2.f * g; }
  else {
    float d2 = fmaxf(ni + n[j] - 2.f * g, 0.f);
    if (diag) d2 = 0.f;
    if (kernel == 2) {
      p.sim = sqrtf(d2);
      const float inv = p.sim > 0.f ? 0.5f / p.sim : 0.f;   // d sqrt(d2)/d d2, sub-gradient 0 at 0 (torch .norm backward)
      p.d_g = -2.f * inv; p.d_n = inv;
    } else {
      p.sim = expf(-0.5f * d2);
      p.d_g = p.sim; p.d_n = -0.5f * p.sim;
    }
  }
  return p;
}

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
    const PairSim s = gsp_sim(kernel, gs[j], nsi, ns, j, j == row), t = gsp_sim(kernel, gt[j], nti, nt, j, j == row);
    const float diff = s.sim - t.sim;
    acc = fmaf(diff, diff, acc);
    const float g = w * diff;                 // d loss / d sim_s
    gs[j] = g * s.d_g;
    rs += g * s.d_n;
    if (BOTH) {
      const float diff_t = t.sim - s.sim;
      const float g_t = w * diff_t;           // d loss / d sim_t
      gt[j] = g_t * t.d_g;
      rt += g_t * t.d_n;
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
    y[i] = axpy_elem(alpha, coef[i / F], x[i], y[i]);
}

// ---------------------------------------------------------------- GSP against a fixed teacher (PPI: gpw on out_feat)
// The teacher of the PPI step is frozen, so its similarities are built once per graph: sim[r][j] = k(G[r][j]) for rows
// [row0, row0 + gridDim.x) of the n x n teacher Gram matrix (G and sim point at the chunk's first row).
__global__ void __launch_bounds__(256) gsp_sim_kernel(const float* __restrict__ G, int64_t ldg, int n, int row0,
                                                      const float* __restrict__ sq, int kernel, float* __restrict__ sim,
                                                      int64_t lds) {
  const int row = row0 + blockIdx.x;
  const float* g = G + (size_t)blockIdx.x * ldg;
  float* s = sim + (size_t)blockIdx.x * lds;
  const float ni = kernel >= 2 ? sq[row] : 0.f;
  for (int j = threadIdx.x; j < n; j += blockDim.x) s[j] = gsp_sim(kernel, g[j], ni, sq, j, j == row).sim;
}

// gsp_pair_kernel<false> with the teacher's similarity read from the stored sim_t instead of formed from its Gram chunk:
// sample position i is node inds[i] (inds null: the identity), so sim_t is read at [inds[row]][inds[j]] while the l2 / rbf
// diagonal and every stored row are sample positions.
__global__ void __launch_bounds__(256) gsp_pair_fixed_kernel(float* __restrict__ Gs, int64_t ld, int S, int row0,
                                                             const float* __restrict__ ns, const float* __restrict__ sim_t,
                                                             int64_t ldt, const int32_t* __restrict__ inds, int kernel,
                                                             float w /* 2 / S^2 */, float* __restrict__ rc_s,
                                                             float* __restrict__ partial) {
  __shared__ float s_red[32];
  const int row = row0 + blockIdx.x;
  float* gs = Gs + (size_t)blockIdx.x * ld;
  const float* st = sim_t + (size_t)(inds ? __ldg(inds + row) : row) * ldt;
  float acc = 0.f, rs = 0.f;
  const float nsi = (kernel >= 2) ? ns[row] : 0.f;
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    const PairSim s = gsp_sim(kernel, gs[j], nsi, ns, j, j == row);
    const float diff = s.sim - st[inds ? __ldg(inds + j) : j];
    acc = fmaf(diff, diff, acc);
    const float g = w * diff;                 // d loss / d sim_s
    gs[j] = g * s.d_g;
    rs += g * s.d_n;
  }
  for (int64_t j = (int64_t)S + threadIdx.x; j < ld; j += blockDim.x) gs[j] = 0.f;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  acc = warp_sum_f(acc); rs = warp_sum_f(rs);
  if (lane == 0) s_red[warp] = acc;
  __syncthreads();
  if (warp == 0) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) partial[row] = t; }
  __syncthreads();
  if (lane == 0) s_red[warp] = rs;
  __syncthreads();
  if (warp == 0 && rc_s) { float t = lane < nw ? s_red[lane] : 0.f; t = warp_sum_f(t); if (lane == 0) rc_s[row] = t; }
}

// The operands of the fixed-teacher pair pass, straight from feature rows (no heads): x[j] = feat[inds[j]] normalised with
// F.normalize's eps and norm[j] = its norm (cosine / poly), or copied with norm[j] = its squared norm (l2 / rbf).  A warp
// per row, the arithmetic of row_normalize_fwd / row_sqnorm.
__global__ void __launch_bounds__(256) gsp_rows_operands_kernel(const float* __restrict__ feat, int64_t ldf,
                                                                const int32_t* __restrict__ inds, int64_t S, int F, int raw,
                                                                float eps, float* __restrict__ x, int64_t ldx,
                                                                float* __restrict__ norm) {
  const int lane = threadIdx.x & 31;
  for (int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); j < S; j += (int64_t)gridDim.x * 8) {
    const float* xr = feat + (size_t)(inds ? __ldg(inds + j) : j) * ldf;
    float* o = x + (size_t)j * ldx;
    float v;
    if (raw) {
      v = row_sumsq(xr, F, lane);
      for (int k = lane; k < F; k += 32) o[k] = xr[k];
    } else {
      v = normalize_row(xr, F, eps, 1.f, o, lane);
    }
    if (lane == 0) norm[j] = v;
  }
}

// The way back from g = dG . x (the chunk loop's product) to beta * d loss / d feat, stored to row inds[j] of d_feat:
// d = 2 g through the normalise backward (cosine / poly), or 2 g + 4 rc[j] x (l2 / rbf), then times beta; the
// arithmetic of the eager row_normalize_bwd / row_axpy and the autograd multiply by beta.  loss_total[0] += beta *
// loss_aux[0] as two roundings, as the eager loss[0].add_(loss_aux * beta).
__global__ void __launch_bounds__(256) gsp_rows_backward_kernel(const int32_t* __restrict__ inds, int64_t S, int F, int raw,
                                                                const float* __restrict__ g, const float* __restrict__ x,
                                                                int64_t ldx, const float* __restrict__ norm,
                                                                const float* __restrict__ rc, float eps, float beta,
                                                                float* __restrict__ d_feat, int64_t ldd,
                                                                const float* __restrict__ loss_aux,
                                                                float* __restrict__ loss_total) {
  const int lane = threadIdx.x & 31;
  for (int64_t j = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); j < S; j += (int64_t)gridDim.x * 8) {
    const float* gj = g + (size_t)j * ldx;
    const float* o = x + (size_t)j * ldx;
    float* d = d_feat + (size_t)(inds ? __ldg(inds + j) : j) * ldd;
    if (raw) {
      const float c = rc[j];
      for (int k = lane; k < F; k += 32) d[k] = axpy_elem(4.f, c, o[k], 2.f * gj[k]) * beta;
    } else {
      const float dot = normalize_bwd_dot(o, [gj](int k) { return 2.f * gj[k]; }, F, 1.f, lane);
      const float nrm = norm[j];
      const bool clamped = nrm < eps;
      const float inv = 1.f / fmaxf(nrm, eps);
      for (int k = lane; k < F; k += 32) d[k] = normalize_bwd_elem(o[k], 2.f * gj[k], 1.f, dot, inv, clamped) * beta;
    }
  }
  if (loss_total && blockIdx.x == 0 && threadIdx.x == 0) loss_total[0] = __fadd_rn(loss_total[0], __fmul_rn(loss_aux[0], beta));
}

// ---------------------------------------------------------------- GSP: the narrow contraction g = dG . x
// g[i, :F] = sum_{j<S} dG[i, j] x[j, :F] for a student side only a few features wide (F <= 128), where the 3xTF32 GEMM
// would fill one 128 x 128 output tile per 128 rows.  The S columns are cut into slabs of GC_SLAB at absolute column
// indices; a CTA takes GC_ROWS rows of one slab and walks it in tiles of GC_KT columns, ascending, accumulating in fp32
// FMA.  The tiles are staged with cp.async into two buffers (dG rows into sG, x rows into sX), so the next tile's loads
// run under this tile's FMAs.  A thread holds 4 rows x 4 features, so a CTA has 8 * F / 4 = 2F threads and
// gsp_contract_smem(F) bytes of shared memory.  Each slab's partial goes to the workspace ([slab][row][F]) and
// gsp_contract_reduce_kernel adds the slabs in ascending order; with one slab the CTA stores g itself.  So g[i] depends on
// row i of dG and on x only: not on the chunk it sits in, the row count or the SM count.
constexpr int GC_SLAB = B200GNN_GSP_CONTRACT_SLAB, GC_ROWS = 32, GC_KT = 32, GC_MAX_F = B200GNN_GSP_CONTRACT_MAX_F;
constexpr int GC_SG = GC_ROWS * (GC_KT + 1);                 // floats of one sG buffer (row pitch 33: a warp's 4-row reads)

__device__ __forceinline__ void gc_cp_async4(float* smem, const float* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void gc_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void gc_cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// column k of a thread's 4 rows (sG row pitch GC_KT + 1) times its 4 features of x row k (sX row pitch F)
__device__ __forceinline__ void gsp_contract_step(float (&acc)[4][4], const float* sg, const float* sx, int k, int F) {
  const float4 xv = *reinterpret_cast<const float4*>(sx + k * F);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float g = sg[q * (GC_KT + 1) + k];
    acc[q][0] = fmaf(g, xv.x, acc[q][0]);
    acc[q][1] = fmaf(g, xv.y, acc[q][1]);
    acc[q][2] = fmaf(g, xv.z, acc[q][2]);
    acc[q][3] = fmaf(g, xv.w, acc[q][3]);
  }
}

__global__ void __launch_bounds__(256, 1) gsp_contract_kernel(const float* __restrict__ dG, int64_t ldg, int64_t n_rows, int S,
                                                              const float* __restrict__ x, int64_t ldx, int F,
                                                              float* __restrict__ out, int64_t ldo, int64_t slab_stride) {
  extern __shared__ float4 gc_smem[];                        // two buffers of sX [GC_KT][F], then two of sG
  float* sX = reinterpret_cast<float*>(gc_smem);
  float* sG = sX + 2 * GC_KT * F;
  const int tid = threadIdx.x, nthr = blockDim.x, fgs = F >> 2;
  const int fg = tid % fgs, rg = tid / fgs;
  const int64_t r0 = (int64_t)blockIdx.x * GC_ROWS;
  const int j_begin = blockIdx.y * GC_SLAB, j_end = min(S, j_begin + GC_SLAB);
  const int n_tiles = (j_end - j_begin + GC_KT - 1) / GC_KT;
  // stage the columns [j0, j0 + kn) into buffer b: dG rows past n_rows and columns past kn are zero-filled, never read
  auto stage = [&](int b, int j0) {
    const int kn = min(GC_KT, j_end - j0);
    float* g = sG + b * GC_SG;
    for (int e = tid; e < GC_ROWS * GC_KT; e += nthr) {
      const int r = e / GC_KT, k = e % GC_KT;
      if (k < kn && r0 + r < n_rows) gc_cp_async4(g + r * (GC_KT + 1) + k, dG + (size_t)(r0 + r) * ldg + j0 + k);
      else g[r * (GC_KT + 1) + k] = 0.f;
    }
    float* xs = sX + b * GC_KT * F;
    for (int e = tid; e < kn * F; e += nthr) {
      const int k = e / F, f = e - k * F;
      gc_cp_async4(xs + k * F + f, x + (size_t)(j0 + k) * ldx + f);
    }
    gc_cp_async_commit();
  };
  float acc[4][4];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[q][c] = 0.f;
  stage(0, j_begin);
  for (int t = 0; t < n_tiles; ++t) {
    const int j0 = j_begin + t * GC_KT, kn = min(GC_KT, j_end - j0), b = t & 1;
    if (t + 1 < n_tiles) {
      stage(b ^ 1, j0 + GC_KT);
      gc_cp_async_wait<1>();
    } else {
      gc_cp_async_wait<0>();
    }
    __syncthreads();                                         // tile t is in buffer b for every thread
    const float* g = sG + b * GC_SG + rg * 4 * (GC_KT + 1);
    const float* xs = sX + b * GC_KT * F + fg * 4;
    if (kn == GC_KT) {
#pragma unroll
      for (int k = 0; k < GC_KT; ++k) gsp_contract_step(acc, g, xs, k, F);
    } else {
      for (int k = 0; k < kn; ++k) gsp_contract_step(acc, g, xs, k, F);
    }
    __syncthreads();                                         // buffer b is refilled by tile t + 2
  }
  float* o = out + (size_t)blockIdx.y * slab_stride;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int64_t row = r0 + rg * 4 + q;
    if (row < n_rows) {
      float* orow = o + (size_t)row * ldo + fg * 4;
#pragma unroll
      for (int c = 0; c < 4; ++c) orow[c] = acc[q][c];
    }
  }
}

static inline size_t gsp_contract_smem(int64_t F) { return (size_t)2 * (GC_KT * F + GC_SG) * sizeof(float); }

// g[row, f] = the slabs' partials added in ascending slab order
__global__ void __launch_bounds__(256) gsp_contract_reduce_kernel(const float* __restrict__ ws, int64_t n_rows, int F,
                                                                  int slabs, float* __restrict__ g, int64_t ldo) {
  const int64_t total = n_rows * (int64_t)F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float* p = ws + i;
    float acc = p[0];
    for (int s = 1; s < slabs; ++s) acc += p[(size_t)s * total];
    g[(i / F) * ldo + i % F] = acc;
  }
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

// The student side of b200gnn_gsp_pair_chunk_f32 alone: the same kernel, one-sided, so Gs, partial and (l2 / rbf) rc_s hold
// the bits the two-sided pass stores for them; Gt is read only.  For a frozen teacher, whose gradient nobody reads.
extern "C" int b200gnn_gsp_pair_student_chunk_f32(float* Gs, const float* Gt, int64_t ld, int64_t n_rows, int64_t S,
                                                  int64_t row_offset, const float* ns, const float* nt, int kernel, float* rc_s,
                                                  float* partial, void* stream) {
  if (!Gs || !Gt || !partial || S <= 0 || S >= INT32_MAX || ld < S || n_rows <= 0 || row_offset < 0 ||
      row_offset + n_rows > S || kernel < 0 || kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2 && (!ns || !nt || !rc_s)) return B200GNN_ERR_BAD_ARG;
  const double n2 = (double)S * (double)S;
  gsp_pair_kernel<false><<<(int)n_rows, 256, 0, (cudaStream_t)stream>>>(Gs, const_cast<float*>(Gt), ld, (int)S, (int)row_offset,
                                                                       ns, nt, kernel, (float)(2.0 / n2), rc_s, nullptr,
                                                                       partial);
  return check_launch();
}

static inline int64_t gsp_contract_slabs(int64_t S) { return (S + GC_SLAB - 1) / GC_SLAB; }

extern "C" size_t b200gnn_gsp_contract_workspace_bytes(int64_t n_rows, int64_t S, int64_t F) {
  if (n_rows <= 0 || S <= 0 || F <= 0) return 0;
  const int64_t slabs = gsp_contract_slabs(S);
  return slabs > 1 ? (size_t)slabs * (size_t)n_rows * (size_t)F * sizeof(float) : 0;
}

// g[i, :F] (pitch ldo) = sum_{j<S} dG[i, j] x[j, :F] for the n_rows rows of dG (pitch ldg >= S; its columns S.. are not
// read), x [S, F] at pitch ldx.  F a multiple of 4 up to 128.  workspace: b200gnn_gsp_contract_workspace_bytes bytes (none
// when S fits one slab).
extern "C" int b200gnn_gsp_contract_narrow_f32(const float* dG, int64_t ldg, int64_t n_rows, int64_t S, const float* x,
                                               int64_t ldx, int64_t F, float* g, int64_t ldo, void* workspace,
                                               size_t workspace_bytes, void* stream) {
  if (!dG || !x || !g || n_rows <= 0 || S <= 0 || F <= 0 || F % 4 || F > GC_MAX_F || ldg < S || ldx < F || ldo < F)
    return B200GNN_ERR_BAD_ARG;
  const int64_t slabs = gsp_contract_slabs(S), row_tiles = (n_rows + GC_ROWS - 1) / GC_ROWS;
  if (slabs > 65535 || row_tiles > INT32_MAX) return B200GNN_ERR_BAD_ARG;
  const size_t need = b200gnn_gsp_contract_workspace_bytes(n_rows, S, F);
  if (need && (!workspace || workspace_bytes < need)) return B200GNN_ERR_BAD_ARG;
  const void* al[] = {dG, x, g, workspace};
  for (const void* p : al)
    if (p && !aligned_to(p, 4)) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = static_cast<float*>(workspace);
  const dim3 grid((unsigned)row_tiles, (unsigned)slabs);
  if (slabs == 1) {
    gsp_contract_kernel<<<grid, (unsigned)(2 * F), gsp_contract_smem(F), st>>>(dG, ldg, n_rows, (int)S, x, ldx, (int)F, g, ldo, 0);
    return check_launch();
  }
  int rc;
  gsp_contract_kernel<<<grid, (unsigned)(2 * F), gsp_contract_smem(F), st>>>(dG, ldg, n_rows, (int)S, x, ldx, (int)F, ws, F,
                                                                            n_rows * F);
  if ((rc = check_launch())) return rc;
  gsp_contract_reduce_kernel<<<ew_grid(n_rows * F), 256, 0, st>>>(ws, n_rows, (int)F, (int)slabs, g, ldo);
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

// ---------------------------------------------------------------- GSP against a fixed teacher
static inline bool f32_aligned(const void* p) { return aligned_to(p, 4); }

// sim = rows [row_offset, row_offset + n_rows) of the n x n similarity matrix from the same rows of the Gram matrix
// (G at pitch ldg >= n, sim at pitch ld_sim >= n, both pointing at the chunk's first row); sq[n]: squared norms (l2 / rbf).
extern "C" int b200gnn_gsp_sim_chunk_f32(const float* G, int64_t ldg, int64_t n_rows, int64_t n, int64_t row_offset,
                                         const float* sq, int kernel, float* sim, int64_t ld_sim, void* stream) {
  if (!G || !sim || n <= 0 || n >= INT32_MAX || ldg < n || ld_sim < n || n_rows <= 0 || row_offset < 0 ||
      row_offset + n_rows > n || kernel < 0 || kernel > 3 || (kernel >= 2 && !sq))
    return B200GNN_ERR_BAD_ARG;
  if (!f32_aligned(G) || !f32_aligned(sim) || (sq && !f32_aligned(sq))) return B200GNN_ERR_BAD_ARG;
  gsp_sim_kernel<<<(int)n_rows, 256, 0, (cudaStream_t)stream>>>(G, ldg, (int)n, (int)row_offset, sq, kernel, sim, ld_sim);
  return check_launch();
}

// The student side of b200gnn_gsp_pair_chunk_f32 against a stored teacher similarity matrix sim_t [n_t, n_t] (pitch
// ld_t): Gs = rows [row_offset, row_offset + n_rows) of the S x S student Gram matrix at pitch ld >= S, overwritten by
// d loss / d Gs, columns S..ld-1 zeroed; partial[S] and (l2 / rbf) rc_s[S] at the sample rows.  inds[S] (nullable: the
// identity, S <= n_t) maps sample positions to rows of sim_t.
extern "C" int b200gnn_gsp_pair_fixed_chunk_f32(float* Gs, int64_t ld, int64_t n_rows, int64_t S, int64_t row_offset,
                                                const float* ns, const float* sim_t, int64_t ld_t, int64_t n_t,
                                                const int32_t* inds, int kernel, float* rc_s, float* partial, void* stream) {
  if (!Gs || !sim_t || !partial || S <= 0 || S >= INT32_MAX || ld < S || n_rows <= 0 || row_offset < 0 ||
      row_offset + n_rows > S || n_t <= 0 || ld_t < n_t || S > n_t || kernel < 0 || kernel > 3)
    return B200GNN_ERR_BAD_ARG;
  if (kernel >= 2 && (!ns || !rc_s)) return B200GNN_ERR_BAD_ARG;
  const void* al[] = {Gs, sim_t, partial, ns, rc_s, inds};
  for (const void* p : al)
    if (p && !f32_aligned(p)) return B200GNN_ERR_BAD_ARG;
  const double n2 = (double)S * (double)S;
  gsp_pair_fixed_kernel<<<(int)n_rows, 256, 0, (cudaStream_t)stream>>>(Gs, ld, (int)S, (int)row_offset, ns, sim_t, ld_t, inds,
                                                                      kernel, (float)(2.0 / n2), rc_s, partial);
  return check_launch();
}

// x[j] (pitch ldx) and norm[j] of feat row inds[j] (inds nullable: row j), feat at pitch ldf.
extern "C" int b200gnn_gsp_rows_operands_f32(const float* feat, int64_t ldf, const int32_t* inds, int64_t S, int64_t F,
                                             int kernel, float eps, float* x, int64_t ldx, float* norm, void* stream) {
  if (!feat || !x || !norm || S <= 0 || S >= INT32_MAX || F <= 0 || F > B200GNN_GSP_ROWS_MAX_F || ldf < F || ldx < F ||
      kernel < 0 || kernel > 3 || !(eps > 0.f))
    return B200GNN_ERR_BAD_ARG;
  const void* al[] = {feat, x, norm, inds};
  for (const void* p : al)
    if (p && !f32_aligned(p)) return B200GNN_ERR_BAD_ARG;
  gsp_rows_operands_kernel<<<ew_grid(S, 8), 256, 0, (cudaStream_t)stream>>>(feat, ldf, inds, S, (int)F, kernel >= 2, eps, x,
                                                                           ldx, norm);
  return check_launch();
}

// d_feat[inds[j]] (pitch ldd; inds nullable: row j) = beta * the operand gradient of x[j] from g[j] = (dG . x)[j];
// norm (cosine / poly) or rc (l2 / rbf) required.  loss_total[0] += beta * loss_aux[0] when loss_total is given.
extern "C" int b200gnn_gsp_rows_backward_f32(const int32_t* inds, int64_t S, int64_t F, int kernel, const float* g,
                                             const float* x, int64_t ldx, const float* norm, const float* rc, float eps,
                                             float beta, float* d_feat, int64_t ldd, const float* loss_aux,
                                             float* loss_total, void* stream) {
  if (!g || !x || !d_feat || S <= 0 || S >= INT32_MAX || F <= 0 || F > B200GNN_GSP_ROWS_MAX_F || ldx < F || ldd < F ||
      kernel < 0 || kernel > 3 || !(eps > 0.f) || (kernel >= 2 ? !rc : !norm) || (loss_total && !loss_aux))
    return B200GNN_ERR_BAD_ARG;
  const void* al[] = {inds, g, x, norm, rc, d_feat, loss_aux, loss_total};
  for (const void* p : al)
    if (p && !f32_aligned(p)) return B200GNN_ERR_BAD_ARG;
  gsp_rows_backward_kernel<<<ew_grid(S, 8), 256, 0, (cudaStream_t)stream>>>(inds, S, (int)F, kernel >= 2, g, x, ldx, norm, rc,
                                                                           eps, beta, d_feat, ldd, loss_aux, loss_total);
  return check_launch();
}
