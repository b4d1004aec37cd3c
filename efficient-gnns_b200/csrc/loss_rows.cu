// Row-wise losses over the training rows of the logits:
//   cross-entropy                       (arxiv_pyg/gnn.py:112, criterion.py:11)
//   logit KD, Hinton et al.             (kd_criterion, arxiv_pyg/criterion.py:8-21)
// One warp per training row; forward value and the gradient w.r.t. the FULL logits matrix are produced
// in the same pass (rows outside train_idx keep the zero the caller memset).  Loss terms are reduced
// deterministically: per-CTA partials, then one finalize CTA in fixed order.
#include "common.cuh"

namespace b200gnn {

constexpr int LOSS_THREADS = 256;
constexpr int LOSS_WARPS = LOSS_THREADS / 32;
constexpr int LOSS_MAX_C = 1024;      // classes per row: NJ = ceil(C/32) values per lane, NJ in {2, 8, 16, 32}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v = fmaxf(v, __shfl_xor_sync(FULL_MASK, v, d));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL_MASK, v, d);
  return v;
}

// partial[cta][2] = {sum_i CE_i, sum_i KL_i}
template <int LOSS_MAX_PER_LANE>
__global__ void __launch_bounds__(LOSS_THREADS) kd_rows_kernel(
    const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ train_idx, int64_t n_train,
    const int64_t* __restrict__ labels, const float* __restrict__ teacher, int64_t ldt, int C, float inv_T,
    float w_cls /* (1-alpha)/n_train */, float w_kd /* alpha*T*T/(n_train*C) */, float* __restrict__ dlogits,
    int64_t ldd, float* __restrict__ partial) {
  __shared__ float s_ce[LOSS_WARPS], s_kl[LOSS_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float ce_acc = 0.f, kl_acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * LOSS_WARPS + warp; i < n_train; i += (int64_t)gridDim.x * LOSS_WARPS) {
    const int64_t row = train_idx ? train_idx[i] : i;
    const int y = (int)labels[row];
    float z[LOSS_MAX_PER_LANE], t[LOSS_MAX_PER_LANE];
    float zmax = -INFINITY, tmax = -INFINITY;
#pragma unroll
    for (int j = 0; j < LOSS_MAX_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < C) {
        z[j] = logits[(size_t)row * ld + c];
        t[j] = teacher ? teacher[(size_t)row * ldt + c] : 0.f;
        zmax = fmaxf(zmax, z[j]); tmax = fmaxf(tmax, t[j]);
      } else { z[j] = -INFINITY; t[j] = -INFINITY; }
    }
    zmax = warp_max(zmax); tmax = warp_max(tmax);
    float se = 0.f, seT = 0.f, steT = 0.f, zy = 0.f;
#pragma unroll
    for (int j = 0; j < LOSS_MAX_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < C) {
        se += expf(z[j] - zmax);
        seT += expf((z[j] - zmax) * inv_T);
        steT += expf((t[j] - tmax) * inv_T);
        if (c == y) zy = z[j];
      }
    }
    se = warp_sum(se); seT = warp_sum(seT); steT = warp_sum(steT); zy = warp_sum(zy);
    const float lse = logf(se), lseT = logf(seT), lsteT = logf(steT);
    ce_acc += (zmax + lse) - zy;  // -log_softmax(z)[y]
    float kl = 0.f;
#pragma unroll
    for (int j = 0; j < LOSS_MAX_PER_LANE; ++j) {
      const int c = lane + 32 * j;
      if (c < C) {
        const float sm = expf(z[j] - zmax - lse);                 // softmax(z)
        float g = w_cls * (sm - (c == y ? 1.f : 0.f));
        if (teacher) {
          const float logq = (z[j] - zmax) * inv_T - lseT;        // log_softmax(z/T)
          const float logp = (t[j] - tmax) * inv_T - lsteT;       // log_softmax(t/T)
          const float p = expf(logp);
          kl += p > 0.f ? p * (logp - logq) : 0.f;
          g += w_kd * inv_T * (expf(logq) - p);
        }
        dlogits[(size_t)row * ldd + c] = g;
      }
    }
    kl_acc += warp_sum(kl);
  }
  if (lane == 0) { s_ce[warp] = ce_acc; s_kl[warp] = kl_acc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float a = 0.f, b = 0.f;
    for (int w = 0; w < LOSS_WARPS; ++w) { a += s_ce[w]; b += s_kl[w]; }
    partial[2 * blockIdx.x] = a; partial[2 * blockIdx.x + 1] = b;
  }
}

// out[3] = {loss, loss_cls, loss_kd}; one CTA, fixed-order tree => deterministic
__global__ void __launch_bounds__(256) kd_finalize_kernel(const float* __restrict__ partial, int n_part, float inv_n,
                                                          float inv_nC, float alpha, float T, int has_teacher,
                                                          float* __restrict__ out) {
  __shared__ double s_ce[256], s_kl[256];
  double ce = 0.0, kl = 0.0;
  for (int i = threadIdx.x; i < n_part; i += 256) { ce += partial[2 * i]; kl += partial[2 * i + 1]; }
  s_ce[threadIdx.x] = ce; s_kl[threadIdx.x] = kl;
  __syncthreads();
  for (int d = 128; d > 0; d >>= 1) {
    if (threadIdx.x < d) { s_ce[threadIdx.x] += s_ce[threadIdx.x + d]; s_kl[threadIdx.x] += s_kl[threadIdx.x + d]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const float loss_cls = (float)(s_ce[0] * inv_n), loss_kd = (float)(s_kl[0] * inv_nC);
    out[1] = loss_cls; out[2] = loss_kd;
    out[0] = has_teacher ? loss_kd * (alpha * T * T) + loss_cls * (1.f - alpha) : loss_cls;
  }
}

}  // namespace b200gnn

using namespace b200gnn;

extern "C" int64_t b200gnn_kd_partials(int64_t n_train) {
  int64_t g = (n_train + LOSS_WARPS - 1) / LOSS_WARPS;
  if (g > 132 * 16) g = 132 * 16;   // rows are a chain of dependent loads (idx -> label -> rows): many short warps
  return g < 1 ? 1 : g;
}

extern "C" int b200gnn_kd_loss_fwd_bwd_f32(const float* logits, int64_t ld, const int64_t* train_idx, int64_t n_train,
                                           const int64_t* labels, const float* teacher_logits, int64_t ldt, int64_t C,
                                           float alpha, float T, int64_t n_norm, float* dlogits, int64_t ldd,
                                           float* loss_out, float* partial, void* stream) {
  if (!logits || !labels || !dlogits || !loss_out || !partial || n_train < 0 || C <= 0 || ld < C || ldd < C)
    return B200GNN_ERR_BAD_ARG;
  if (C > LOSS_MAX_C) return B200GNN_ERR_UNSUPPORTED;
  if (teacher_logits && (ldt < C || T <= 0.f)) return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)b200gnn_kd_partials(n_train);
  const bool kd = teacher_logits != nullptr;
  if (n_norm <= 0) n_norm = n_train;   // sharded runs normalise by the GLOBAL number of training rows
  const float w_cls = (kd ? (1.f - alpha) : 1.f) / (float)n_norm;
  const float w_kd = kd ? alpha * T * T / ((float)n_norm * (float)C) : 0.f;
  int rc;
#define B200GNN_KD_LAUNCH(NJ)                                                                                     \
  kd_rows_kernel<NJ><<<grid, LOSS_THREADS, 0, st>>>(logits, ld, train_idx, n_train, labels, teacher_logits, ldt, \
                                                    (int)C, kd ? 1.f / T : 1.f, w_cls, w_kd, dlogits, ldd, partial)
  if (C <= 64) B200GNN_KD_LAUNCH(2);            // ogbn-arxiv: 40 classes
  else if (C <= 256) B200GNN_KD_LAUNCH(8);
  else if (C <= 512) B200GNN_KD_LAUNCH(16);     // ogbn-mag: 349 classes (mag_pyg/gnn.py:399)
  else B200GNN_KD_LAUNCH(32);
#undef B200GNN_KD_LAUNCH
  if ((rc = check_launch())) return rc;
  kd_finalize_kernel<<<1, 256, 0, st>>>(partial, grid, 1.f / (float)n_norm, 1.f / ((float)n_norm * (float)C), alpha, T,
                                      kd ? 1 : 0, loss_out);
  return check_launch();
}
