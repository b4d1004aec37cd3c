// Row passes of the SIGN student's training step (arxiv_dgl/sign.py:105-157) that are not GEMMs:
//   * the batch gather of every hop's feature rows with input dropout, plus the label and teacher-logit rows of the batch;
//   * dropout(prelu(Z)) materialised from the packed keep bits (what the PReLU GEMM prologues form in registers);
//   * column sums with a row pitch (the bias gradients, read straight out of column blocks of the concatenation).
#include "common.cuh"
#include "philox.cuh"

namespace b200gnn {
namespace sign {

constexpr int MAX_HOPS = 16;
struct HopPtrs {
  const float* x[MAX_HOPS];
};

// out[h][i][:] = dropout(feats[h][idx[i]][:]) for every hop h; the keep decision of element (i, c) of hop h is the one
// b200gnn_dropout_mask_u8(B, F, p, seed, offset + h + *step_dev * step_mul) takes.  Rows with idx outside [0, n_nodes) are
// written as zeros.  Threads past the features copy labels[idx[i]] and teacher[idx[i]][:] of the batch.
__global__ void __launch_bounds__(256) gather_kernel(const HopPtrs hp, int n_hops, int64_t n_nodes, int nvec_row,
                                                     const int64_t* __restrict__ idx, int64_t B, float p, int p16, uint32_t thr16,
                                                     uint64_t seed, uint64_t offset, const int32_t* __restrict__ step_dev,
                                                     uint64_t step_mul, float* __restrict__ out, const int64_t* __restrict__ labels,
                                                     int64_t* __restrict__ labels_out, const float* __restrict__ teacher,
                                                     int64_t ldt, int C, float* __restrict__ teacher_out) {
  if (step_dev) offset += (uint64_t)(*step_dev) * step_mul;
  const float inv_keep = p > 0.f ? 1.f / (1.f - p) : 1.f;
  const int64_t per_hop = B * nvec_row, n_feat = per_hop * n_hops;
  const int64_t n_lab = labels ? B : 0, n_t = teacher ? B * C : 0;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_feat + n_lab + n_t; t += (int64_t)gridDim.x * blockDim.x) {
    if (t < n_feat) {
      const int h = (int)(t / per_hop);
      const int64_t i = t - h * per_hop, row = i / nvec_row;
      const int cv = (int)(i - row * nvec_row);
      const int64_t node = idx[row];
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (node >= 0 && node < n_nodes) v = __ldg(reinterpret_cast<const float4*>(hp.x[h] + node * 4 * nvec_row) + cv);
      if (p > 0.f) {
        const uint64_t off = offset + (uint64_t)h;
        uchar4 m;
        if (p16) {
          const uint4 r = philox4x32(seed, off, (uint64_t)i >> 1);
          m = keep16((i & 1) ? r.z : r.x, (i & 1) ? r.w : r.y, thr16);
        } else {
          m = keep24(philox4x32(seed, off, (uint64_t)i), p);
        }
        v.x = m.x ? v.x * inv_keep : 0.f; v.y = m.y ? v.y * inv_keep : 0.f;
        v.z = m.z ? v.z * inv_keep : 0.f; v.w = m.w ? v.w * inv_keep : 0.f;
      }
      reinterpret_cast<float4*>(out)[t] = v;
    } else if (t < n_feat + n_lab) {
      const int64_t row = t - n_feat, node = idx[row];
      labels_out[row] = node >= 0 && node < n_nodes ? labels[node] : 0;
    } else {
      const int64_t e = t - n_feat - n_lab, row = e / C;
      const int c = (int)(e - row * C);
      const int64_t node = idx[row];
      teacher_out[e] = node >= 0 && node < n_nodes ? teacher[node * ldt + c] : 0.f;
    }
  }
}

// out = bit ? (z > 0 ? z : slope * z) / (1-p) : 0 — the operations of the PReLU GEMM prologues
__global__ void __launch_bounds__(256) prelu_bits_kernel(const float* __restrict__ Z, int64_t ldz, const uint32_t* __restrict__ bits,
                                                         int64_t ldbits, const float* __restrict__ slope_p, float inv_keep,
                                                         float* __restrict__ out, int64_t ldo, int64_t n_rows, int nvec_row) {
  const float slope = __ldg(slope_p);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_rows * nvec_row; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / nvec_row;
    const int cv = (int)(i - row * nvec_row);
    const float4 z = *reinterpret_cast<const float4*>(Z + row * ldz + 4 * cv);
    const uint32_t b = bits[row * ldbits + (cv >> 3)] >> (4 * (cv & 7));
    float4 y;
    y.x = (b & 1u) ? (z.x > 0.f ? z.x : slope * z.x) * inv_keep : 0.f;
    y.y = (b & 2u) ? (z.y > 0.f ? z.y : slope * z.y) * inv_keep : 0.f;
    y.z = (b & 4u) ? (z.z > 0.f ? z.z : slope * z.z) * inv_keep : 0.f;
    y.w = (b & 8u) ? (z.w > 0.f ? z.w : slope * z.w) * inv_keep : 0.f;
    *reinterpret_cast<float4*>(out + row * ldo + 4 * cv) = y;
  }
}

// Column sums of Y [n_rows, K] (pitch ldy): CTA (slot, column block) adds its rows in order into partial[slot][K], then
// colsum_ld_finalize_kernel adds the slots in order (fixed order: bitwise repeatable).
constexpr int CS_THREADS = 128;
__global__ void __launch_bounds__(CS_THREADS) colsum_ld_kernel(const float* __restrict__ Y, int64_t ldy, int64_t n_rows, int nvec_row,
                                                               float* __restrict__ partial, int slots) {
  const int cv = blockIdx.y * CS_THREADS + threadIdx.x;
  if (cv >= nvec_row) return;
  const int slot = blockIdx.x;
  const int64_t r0 = n_rows * slot / slots, r1 = n_rows * (slot + 1) / slots;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t r = r0; r < r1; ++r) {
    const float4 y = __ldg(reinterpret_cast<const float4*>(Y + r * ldy) + cv);
    a.x += y.x; a.y += y.y; a.z += y.z; a.w += y.w;
  }
  reinterpret_cast<float4*>(partial + (size_t)slot * 4 * nvec_row)[cv] = a;
}
__global__ void __launch_bounds__(256) colsum_ld_finalize_kernel(const float* __restrict__ partial, int slots, int K,
                                                                 float* __restrict__ out) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= K) return;
  float a = 0.f;
  for (int s = 0; s < slots; ++s) a += partial[(size_t)s * K + c];
  out[c] = a;
}

static inline int grid_for(int64_t n_items, int per_cta, int cap = 132 * 8) {
  int64_t g = (n_items + per_cta - 1) / per_cta;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

}  // namespace sign
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_sign_gather_f32(const float* const* feats, int32_t n_hops, int64_t n_nodes, int64_t F, const int64_t* idx,
                                       int64_t B, float p, uint64_t seed, uint64_t offset, const int32_t* step_dev,
                                       uint64_t step_mul, float* out, const int64_t* labels, int64_t* labels_out,
                                       const float* teacher, int64_t ldt, int64_t C, float* teacher_out, void* stream) {
  if (!feats || n_hops < 1 || n_hops > sign::MAX_HOPS || n_nodes < 0 || F <= 0 || F % 4 || B < 0 || p < 0.f || p >= 1.f ||
      (B > 0 && (!idx || !out)) || (labels == nullptr) != (labels_out == nullptr) ||
      (teacher == nullptr) != (teacher_out == nullptr) || (teacher && (C <= 0 || ldt < C)) || !aligned_to(out, 16))
    return B200GNN_ERR_BAD_ARG;
  sign::HopPtrs hp{};
  for (int h = 0; h < n_hops; ++h) {
    if (!feats[h] || !aligned_to(feats[h], 16)) return B200GNN_ERR_BAD_ARG;
    hp.x[h] = feats[h];
  }
  if (B == 0) return B200GNN_OK;
  uint32_t thr16 = 0;
  const int p16 = dropout_p16(p, thr16) ? 1 : 0;
  const int64_t n_items = B * (F / 4) * n_hops + (labels ? B : 0) + (teacher ? B * C : 0);
  sign::gather_kernel<<<sign::grid_for(n_items, 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      hp, n_hops, n_nodes, (int)(F / 4), idx, B, p, p16, thr16, seed, offset, step_dev, step_mul, out, labels, labels_out, teacher,
      ldt, (int)C, teacher_out);
  return check_launch();
}

extern "C" int b200gnn_prelu_bits_f32(const float* Z, int64_t ldz, const uint32_t* bits, int64_t ldbits, const float* slope, float p,
                                      float* out, int64_t ldo, int64_t n_rows, int64_t K, void* stream) {
  if (!Z || !bits || !slope || !out || n_rows < 0 || K <= 0 || K % 4 || ldz < K || ldz % 4 || ldo < K || ldo % 4 ||
      ldbits < (K + 31) / 32 || p < 0.f || p >= 1.f || !aligned_to(Z, 16) || !aligned_to(out, 16))
    return B200GNN_ERR_BAD_ARG;
  if (n_rows == 0) return B200GNN_OK;
  const float inv_keep = p > 0.f ? 1.f / (1.f - p) : 1.f;
  sign::prelu_bits_kernel<<<sign::grid_for(n_rows * (K / 4), 256 * 4), 256, 0, (cudaStream_t)stream>>>(
      Z, ldz, bits, ldbits, slope, inv_keep, out, ldo, n_rows, (int)(K / 4));
  return check_launch();
}

extern "C" int64_t b200gnn_col_sum_ld_slots(int64_t n_rows) {
  if (n_rows < 0) return B200GNN_ERR_BAD_ARG;
  const int64_t s = (n_rows + 63) / 64;
  return s < 1 ? 1 : (s > 264 ? 264 : s);
}

extern "C" int b200gnn_col_sum_ld_f32(const float* Y, int64_t ldy, int64_t n_rows, int64_t K, float* out, float* partial,
                                      int64_t slots, void* stream) {
  if (!Y || !out || !partial || n_rows < 1 || K <= 0 || K % 4 || ldy < K || ldy % 4 || !aligned_to(Y, 16) ||
      !aligned_to(partial, 16) || slots < b200gnn_col_sum_ld_slots(n_rows))
    return B200GNN_ERR_BAD_ARG;
  const int used = (int)b200gnn_col_sum_ld_slots(n_rows), nvec = (int)(K / 4);
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid(used, (nvec + sign::CS_THREADS - 1) / sign::CS_THREADS);
  sign::colsum_ld_kernel<<<grid, sign::CS_THREADS, 0, st>>>(Y, ldy, n_rows, nvec, partial, used);
  int rc = check_launch();
  if (rc) return rc;
  sign::colsum_ld_finalize_kernel<<<(int)((K + 255) / 256), 256, 0, st>>>(partial, used, (int)K, out);
  return check_launch();
}
