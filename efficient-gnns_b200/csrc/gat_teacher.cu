// The training recipe around the arxiv GAT teacher (arxiv_dgl/gat.py:98-183): label inputs, the label-reuse softmax,
// the log-CE loss, split evaluation and the best-epoch snapshot.  Every kernel reads its step-dependent state (draw offset,
// loss-row count, best loss) on the device, so one epoch is one CUDA graph with no host read.
//
// Row roles (uint8 per node), written by the label-input kernel:
//   ROLE_NONE  0  not in train / val / test
//   ROLE_INPUT 1  training row fed as an input: with use_labels its one-hot label is in the input (train: the mask-true rows,
//                 eval: every training row); without labels a training row outside the loss
//   ROLE_PRED  2  training row the loss runs on (train_pred_idx, gat.py:124-131)
//   ROLE_EVAL  3  validation or test row
// Loss sums go into per-CTA fp64 partials that one CTA adds in slot order: deterministic for a fixed grid.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"

namespace b200gnn {

constexpr int TEACHER_THREADS = 256;
constexpr int TEACHER_WARPS = TEACHER_THREADS / 32;
constexpr int TEACHER_MAX_C = 256;          // classes per row: NJ = ceil(C/32) in {2, 8}
constexpr int ROLE_INPUT = 1, ROLE_PRED = 2, ROLE_EVAL = 3;
// epsilon = 1 - ln 2 and math.log(epsilon) of custom_loss_function (gat.py:21, 98-101), each rounded to fp32 once, as the
// fp32 tensor arithmetic of the reference sees them
constexpr float LOGCE_EPS = 0.306852818f;
constexpr float LOGCE_LOG_EPS = -1.18138707f;

__device__ __forceinline__ float t_warp_max(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, d));
  return v;
}
__device__ __forceinline__ float t_warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}

// The drop decision b200gnn_dropout_mask_u8 makes for flat element j at (seed, offset, p): element j is component j % 4 of
// float4 j / 4 (dropout_mask_kernel).
__device__ __forceinline__ bool drop_decision(int64_t j, float p, int p16, uint32_t thr16, uint64_t seed, uint64_t offset) {
  const uint64_t i = (uint64_t)j >> 2;
  const int comp = (int)(j & 3);
  if (p16) {
    const uint4 r = philox4x32(seed, offset, i >> 1);
    const uint32_t w = (i & 1) ? (comp < 2 ? r.z : r.w) : (comp < 2 ? r.x : r.y);
    const uint32_t u16 = (comp & 1) ? (w >> 16) : (w & 0xffffu);
    return u16 < thr16;
  }
  const uint4 r = philox4x32(seed, offset, i);
  const uint32_t u = comp == 0 ? r.x : comp == 1 ? r.y : comp == 2 ? r.z : r.w;
  return !(u32_to_unit(u) >= p);
}

// One warp per node: role, label block X[r, col0 : col0 + C] (one-hot for ROLE_INPUT rows when C > 0, zero otherwise) and
// the per-CTA count of ROLE_PRED rows.  row_pos[r]: training position (>= 0), -1 validation / test, -2 neither.
__global__ void __launch_bounds__(TEACHER_THREADS) label_inputs_kernel(
    float* __restrict__ X, int64_t ldx, int64_t col0, int C, int64_t n_rows, const int32_t* __restrict__ row_pos,
    const int64_t* __restrict__ labels, int eval, float p, int p16, uint32_t thr16, uint64_t seed, uint64_t offset,
    const int32_t* __restrict__ step_dev, uint64_t step_mul, const uint8_t* __restrict__ mask_in, int use_labels,
    uint8_t* __restrict__ role, int32_t* __restrict__ cnt_part) {
  __shared__ int s_cnt[TEACHER_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint64_t off = offset + (step_dev ? (uint64_t)(*step_dev) * step_mul : 0ull);
  int cnt = 0;
  for (int64_t r = (int64_t)blockIdx.x * TEACHER_WARPS + warp; r < n_rows; r += (int64_t)gridDim.x * TEACHER_WARPS) {
    const int pos = row_pos[r];
    int ro = pos == -1 ? ROLE_EVAL : 0;
    if (pos >= 0) {
      if (eval) {
        ro = ROLE_INPUT;
      } else {
        const bool masked = mask_in ? mask_in[pos] != 0 : drop_decision(pos, p, p16, thr16, seed, off);   // rand < mask_rate
        ro = (masked == (use_labels != 0)) ? ROLE_INPUT : ROLE_PRED;
      }
    }
    cnt += ro == ROLE_PRED;
    if (C > 0) {
      const int y = ro == ROLE_INPUT ? (int)labels[r] : -1;
      for (int c = lane; c < C; c += 32) X[(size_t)r * ldx + col0 + c] = c == y ? 1.f : 0.f;
    }
    if (lane == 0) role[r] = (uint8_t)ro;
  }
  if (lane == 0) s_cnt[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0;
    for (int w = 0; w < TEACHER_WARPS; ++w) a += s_cnt[w];
    cnt_part[blockIdx.x] = a;
  }
}

// out[r, 0:C] = softmax(logits[r, 0:C]) for the rows whose role bit is set in role_mask (every row when role is null).
template <int NJ>
__global__ void __launch_bounds__(TEACHER_THREADS) label_softmax_kernel(const float* __restrict__ logits, int64_t ld, int C,
                                                                        int64_t n_rows, const uint8_t* __restrict__ role,
                                                                        int role_mask, float* __restrict__ out, int64_t ldo) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int64_t r = (int64_t)blockIdx.x * TEACHER_WARPS + warp; r < n_rows; r += (int64_t)gridDim.x * TEACHER_WARPS) {
    if (role && !((role_mask >> role[r]) & 1)) continue;
    float z[NJ], m = -INFINITY;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = lane + 32 * j;
      z[j] = c < C ? logits[(size_t)r * ld + c] : -INFINITY;
      m = fmaxf(m, z[j]);
    }
    m = t_warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = lane + 32 * j;
      if (c < C) { z[j] = expf(z[j] - m); s += z[j]; }
    }
    s = t_warp_sum(s);
    const float inv = 1.f / s;
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = lane + 32 * j;
      if (c < C) out[(size_t)r * ldo + c] = z[j] * inv;
    }
  }
}

// Per row of the logits: cross-entropy CE = logsumexp(z) - z[y], the first-maximum argmax hit, and (GRAD) the log-CE
// gradient (softmax - onehot) * w written into drow.  NaN counts as the maximum, as in torch.argmax.
template <int NJ, bool GRAD>
__device__ __forceinline__ void logce_row(const float* __restrict__ z_row, int C, int y, float* __restrict__ drow, float inv_n,
                                          float& ce, bool& hit) {
  const int lane = threadIdx.x & 31;
  float z[NJ], m = -INFINITY, bv = -INFINITY;
  int bi = 0x7fffffff;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = lane + 32 * j;
    z[j] = c < C ? z_row[c] : -INFINITY;
    m = fmaxf(m, z[j]);
    if (c < C && bi == 0x7fffffff) { bv = z[j]; bi = c; }
    else if (c < C && (z[j] > bv || (isnan(z[j]) && !isnan(bv)))) { bv = z[j]; bi = c; }
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) {
    const float ov = __shfl_xor_sync(FULL_MASK, bv, d);
    const int oi = __shfl_xor_sync(FULL_MASK, bi, d);
    const bool o_nan = isnan(ov), s_nan = isnan(bv);
    const bool take = (o_nan && !s_nan) || (o_nan == s_nan && (ov > bv || (!(ov < bv) && oi < bi)));
    if (take) { bv = ov; bi = oi; }
  }
  m = t_warp_max(m);
  float s = 0.f, zy = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const int c = lane + 32 * j;
    if (c < C) { s += expf(z[j] - m); if (c == y) zy = z[j]; }
  }
  s = t_warp_sum(s); zy = t_warp_sum(zy);
  const float lse = logf(s);
  ce = (m + lse) - zy;
  hit = bi == y;
  if (GRAD) {
    const float w = inv_n / (LOGCE_EPS + ce);               // d/dCE of log(eps + CE), over the device row count
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int c = lane + 32 * j;
      if (c < C) drow[c] = (expf(z[j] - m - lse) - (c == y ? 1.f : 0.f)) * w;
    }
  }
}

__device__ __forceinline__ float logce_term(float ce) { return logf(LOGCE_EPS + ce) - LOGCE_LOG_EPS; }

// Sum of the label kernel's per-CTA ROLE_PRED counts (every CTA forms it; integers, so exact in any order).
__device__ __forceinline__ int64_t count_rows(const int32_t* __restrict__ cnt_part, int n_cnt) {
  __shared__ int64_t s_n[TEACHER_WARPS];
  int64_t a = 0;
  for (int i = threadIdx.x; i < n_cnt; i += TEACHER_THREADS) a += cnt_part[i];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) a += __shfl_xor_sync(FULL_MASK, a, d);
  if ((threadIdx.x & 31) == 0) s_n[threadIdx.x >> 5] = a;
  __syncthreads();
  int64_t n = 0;
  for (int w = 0; w < TEACHER_WARPS; ++w) n += s_n[w];
  return n;
}

// TRAIN: one warp per training position; every row counts for the accuracy, the ROLE_PRED rows for the loss and its
//        gradient.  partial[cta] = {sum log-CE term, hits, -, -, -, -}.
// EVAL:  one warp per position of idx = [train | val | test] (split sizes n0, n1, n2); partial[cta] = {term_s, hits_s}
//        for s = 0, 1, 2 at [s] and [3 + s].
template <int NJ, bool TRAIN>
__global__ void __launch_bounds__(TEACHER_THREADS) logce_rows_kernel(
    const float* __restrict__ logits, int64_t ld, int C, const int64_t* __restrict__ idx, int64_t n0, int64_t n1, int64_t n2,
    const int64_t* __restrict__ labels, const uint8_t* __restrict__ role, const int32_t* __restrict__ cnt_part, int n_cnt,
    float* __restrict__ dlogits, int64_t ldd, double* __restrict__ partial) {
  __shared__ double s_acc[TEACHER_WARPS][6];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float inv_n = 0.f;
  if (TRAIN) {
    const int64_t n = count_rows(cnt_part, n_cnt);
    inv_n = n > 0 ? 1.f / (float)n : 0.f;
  }
  double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  const int64_t total = n0 + n1 + n2;
  for (int64_t i = (int64_t)blockIdx.x * TEACHER_WARPS + warp; i < total; i += (int64_t)gridDim.x * TEACHER_WARPS) {
    const int64_t r = idx[i];
    const int y = (int)labels[r];
    float ce; bool hit;
    if (TRAIN) {
      const bool pred = role[r] == ROLE_PRED;
      if (pred) logce_row<NJ, true>(logits + (size_t)r * ld, C, y, dlogits + (size_t)r * ldd, inv_n, ce, hit);
      else logce_row<NJ, false>(logits + (size_t)r * ld, C, y, nullptr, 0.f, ce, hit);
      if (pred) acc[0] += (double)logce_term(ce);
      acc[1] += hit ? 1.0 : 0.0;
    } else {
      logce_row<NJ, false>(logits + (size_t)r * ld, C, y, nullptr, 0.f, ce, hit);
      const int s = i < n0 ? 0 : i < n0 + n1 ? 1 : 2;
      const double term = (double)logce_term(ce);
#pragma unroll
      for (int k = 0; k < 3; ++k)            // static indices: acc stays in registers
        if (s == k) { acc[k] += term; acc[3 + k] += hit ? 1.0 : 0.0; }
    }
  }
  if (lane == 0)
    for (int k = 0; k < 6; ++k) s_acc[warp][k] = acc[k];
  __syncthreads();
  if (threadIdx.x < 6) {
    double a = 0.0;
    for (int w = 0; w < TEACHER_WARPS; ++w) a += s_acc[w][threadIdx.x];
    partial[6 * blockIdx.x + threadIdx.x] = a;
  }
}

// One warp per output quantity k < 6: partial slots added in slot order.  TRAIN: loss_out[0] = term / n_pred,
// acc_out[0] = hits / n_train.  EVAL: acc_out[s] = hits_s / n_s, loss_out[s] = term_s / n_s.  An empty set gives NaN
// (torch.mean of nothing).
template <bool TRAIN>
__global__ void __launch_bounds__(TEACHER_THREADS) logce_finalize_kernel(const double* __restrict__ partial, int slots,
                                                                         const int32_t* __restrict__ cnt_part, int n_cnt,
                                                                         int64_t n0, int64_t n1, int64_t n2,
                                                                         float* __restrict__ loss_out, float* __restrict__ acc_out) {
  const int64_t n_pred = TRAIN ? count_rows(cnt_part, n_cnt) : 0;
  const int k = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (k >= 6 || (TRAIN && k >= 2)) return;
  if (lane == 0) {
    double a = 0.0;
    for (int s = 0; s < slots; ++s) a += partial[6 * s + k];
    if (TRAIN) {
      if (k == 0) loss_out[0] = (float)(a / (double)n_pred);
      else acc_out[0] = (float)(a / (double)n0);
    } else {
      const int sp = k % 3;
      const double n = (double)(sp == 0 ? n0 : sp == 1 ? n1 : n2);
      if (k < 3) loss_out[sp] = (float)(a / n);
      else acc_out[sp] = (float)(a / n);
    }
  }
}

struct SnapshotCopies {
  const float4* src[3];
  float4* dst[3];
  int64_t n_vec[3];
};

// if (*cand < *best): dst_i = src_i for the (up to three) buffers.  NaN never compares lower.
__global__ void __launch_bounds__(256) snapshot_copy_kernel(const float* __restrict__ cand, const float* __restrict__ best,
                                                            SnapshotCopies cp) {
  if (!(*cand < *best)) return;
  for (int b = 0; b < 3; ++b) {
    const float4* __restrict__ s = cp.src[b];
    float4* __restrict__ d = cp.dst[b];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cp.n_vec[b]; i += (int64_t)gridDim.x * blockDim.x)
      d[i] = s[i];
  }
}
__global__ void best_update_kernel(const float* __restrict__ cand, float* __restrict__ best) {
  if (*cand < *best) *best = *cand;
}

}  // namespace b200gnn

using namespace b200gnn;

extern "C" int64_t b200gnn_teacher_slots(int64_t n_items) {
  int64_t g = (n_items + TEACHER_WARPS - 1) / TEACHER_WARPS;
  if (g > 132 * 8) g = 132 * 8;
  return g < 1 ? 1 : g;
}

extern "C" int b200gnn_label_inputs_f32(float* X, int64_t ldx, int64_t col0, int64_t C, int64_t n_rows, const int32_t* row_pos,
                                        const int64_t* labels, int eval, float mask_rate, uint64_t seed, uint64_t offset,
                                        const int32_t* step_dev, uint64_t step_mul, const uint8_t* mask_in, int use_labels,
                                        uint8_t* role, int32_t* cnt_part, void* stream) {
  if (!row_pos || !role || !cnt_part || n_rows < 0 || C < 0 || mask_rate < 0.f || mask_rate >= 1.f) return B200GNN_ERR_BAD_ARG;
  if (C > 0 && (!X || !labels || col0 < 0 || ldx < col0 + C)) return B200GNN_ERR_BAD_ARG;
  if (use_labels && C == 0) return B200GNN_ERR_BAD_ARG;
  if (eval && use_labels && !labels) return B200GNN_ERR_BAD_ARG;
  uint32_t thr16 = 0;
  const int p16 = dropout_p16(mask_rate, thr16) ? 1 : 0;
  label_inputs_kernel<<<(int)b200gnn_teacher_slots(n_rows), TEACHER_THREADS, 0, (cudaStream_t)stream>>>(
      X, ldx, col0, (int)C, n_rows, row_pos, labels, eval, mask_rate, p16, thr16, seed, offset, step_dev, step_mul, mask_in,
      use_labels, role, cnt_part);
  return check_launch();
}

extern "C" int b200gnn_label_softmax_f32(const float* logits, int64_t ld, int64_t C, int64_t n_rows, const uint8_t* role,
                                         int role_mask, float* out, int64_t ldo, void* stream) {
  if (!logits || !out || C <= 0 || n_rows < 0 || ld < C || ldo < C) return B200GNN_ERR_BAD_ARG;
  if (C > TEACHER_MAX_C) return B200GNN_ERR_UNSUPPORTED;
  if (n_rows == 0) return B200GNN_OK;
  const int grid = (int)b200gnn_teacher_slots(n_rows);
  cudaStream_t st = (cudaStream_t)stream;
  if (C <= 64) label_softmax_kernel<2><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, n_rows, role, role_mask, out, ldo);
  else label_softmax_kernel<8><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, n_rows, role, role_mask, out, ldo);
  return check_launch();
}

extern "C" int b200gnn_logce_fwd_bwd_f32(const float* logits, int64_t ld, int64_t C, const int64_t* train_idx, int64_t n_train,
                                         const int64_t* labels, const uint8_t* role, const int32_t* cnt_part, int64_t n_cnt,
                                         float* dlogits, int64_t ldd, float* loss_out, float* acc_out, double* partial,
                                         void* stream) {
  if (!logits || !train_idx || !labels || !role || !cnt_part || !dlogits || !loss_out || !acc_out || !partial || C <= 0 ||
      ld < C || ldd < C || n_train < 0 || n_cnt < 1)
    return B200GNN_ERR_BAD_ARG;
  if (C > TEACHER_MAX_C) return B200GNN_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)b200gnn_teacher_slots(n_train);
  int rc;
  if (C <= 64)
    logce_rows_kernel<2, true><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, train_idx, n_train, 0, 0, labels, role,
                                                                cnt_part, (int)n_cnt, dlogits, ldd, partial);
  else
    logce_rows_kernel<8, true><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, train_idx, n_train, 0, 0, labels, role,
                                                                cnt_part, (int)n_cnt, dlogits, ldd, partial);
  if ((rc = check_launch())) return rc;
  logce_finalize_kernel<true><<<1, TEACHER_THREADS, 0, st>>>(partial, grid, cnt_part, (int)n_cnt, n_train, 0, 0, loss_out,
                                                             acc_out);
  return check_launch();
}

extern "C" int b200gnn_split_eval_f32(const float* logits, int64_t ld, int64_t C, const int64_t* idx, int64_t n0, int64_t n1,
                                      int64_t n2, const int64_t* labels, float* loss_out, float* acc_out, double* partial,
                                      void* stream) {
  if (!logits || !idx || !labels || !loss_out || !acc_out || !partial || C <= 0 || ld < C || n0 < 0 || n1 < 0 || n2 < 0)
    return B200GNN_ERR_BAD_ARG;
  if (C > TEACHER_MAX_C) return B200GNN_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)b200gnn_teacher_slots(n0 + n1 + n2);
  int rc;
  if (C <= 64)
    logce_rows_kernel<2, false><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, idx, n0, n1, n2, labels, nullptr, nullptr,
                                                                 0, nullptr, 0, partial);
  else
    logce_rows_kernel<8, false><<<grid, TEACHER_THREADS, 0, st>>>(logits, ld, (int)C, idx, n0, n1, n2, labels, nullptr, nullptr,
                                                                 0, nullptr, 0, partial);
  if ((rc = check_launch())) return rc;
  logce_finalize_kernel<false><<<1, TEACHER_THREADS, 0, st>>>(partial, grid, nullptr, 0, n0, n1, n2, loss_out, acc_out);
  return check_launch();
}

extern "C" int b200gnn_snapshot_if_better_f32(const float* cand, float* best, const float* src0, float* dst0, int64_t n0,
                                              const float* src1, float* dst1, int64_t n1, const float* src2, float* dst2,
                                              int64_t n2, void* stream) {
  if (!cand || !best) return B200GNN_ERR_BAD_ARG;
  SnapshotCopies cp;
  const float* src[3] = {src0, src1, src2};
  float* dst[3] = {dst0, dst1, dst2};
  const int64_t n[3] = {n0, n1, n2};
  int64_t most = 0;
  for (int b = 0; b < 3; ++b) {
    if (n[b] < 0 || n[b] % 4 || (n[b] > 0 && (!src[b] || !dst[b] || !aligned_to(src[b], 16) || !aligned_to(dst[b], 16))))
      return B200GNN_ERR_BAD_ARG;
    cp.src[b] = reinterpret_cast<const float4*>(src[b]);
    cp.dst[b] = reinterpret_cast<float4*>(dst[b]);
    cp.n_vec[b] = n[b] / 4;
    if (cp.n_vec[b] > most) most = cp.n_vec[b];
  }
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  int64_t g = (most + 255) / 256;
  g = g < 1 ? 1 : g > 132 * 8 ? 132 * 8 : g;
  snapshot_copy_kernel<<<(int)g, 256, 0, st>>>(cand, best, cp);
  if ((rc = check_launch())) return rc;
  best_update_kernel<<<1, 1, 0, st>>>(cand, best);
  return check_launch();
}
