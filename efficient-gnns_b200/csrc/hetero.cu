// Heterogeneous input assembly (RGCN.group_input, mag_pyg/gnn.py:111-124): node i of the (sub)graph takes row
// local_idx[i] of the table of its node type — raw features for the types that have them, learned embedding tables
// (1,134,649 / 59,965 / 8,740 x 128 on ogbn-mag, mag_pyg/gnn.py:387) for the others.  The reference does one boolean
// mask + masked gather/assignment per type (4 passes over node_type, 4 [n,F] index_puts); here it is one typed gather.
// Backward: d table[t][j] = sum of d out[i] over the nodes i with (type, idx) = (t, j).  The caller passes the nodes
// sorted by (type, idx) (`order`); one warp per run of equal keys adds the run in order -> deterministic, no atomics
// (the reference's index_put_(accumulate=True) backward is atomic).
#include "common.cuh"

namespace b200gnn {

constexpr int MAX_TABLES = 16;
struct Tables {
  float* ptr[MAX_TABLES];
  int64_t rows[MAX_TABLES];
  int32_t n;
};

__global__ void __launch_bounds__(256) typed_gather_kernel(const Tables T, const int64_t* __restrict__ node_type,
                                                           const int64_t* __restrict__ local_idx, int64_t n, int F,
                                                           float* __restrict__ out, int64_t ldo, int32_t* __restrict__ err) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t i = warp; i < n; i += nwarps) {
    const int64_t t = node_type[i], j = local_idx[i];
    const float* src = nullptr;
    if (t >= 0 && t < T.n && T.ptr[t]) {
      if (j >= 0 && j < T.rows[t]) src = T.ptr[t] + (size_t)j * F;
      else if (lane == 0) *err = 1;                  // index out of range: reported, row left zero
    }
    float* dst = out + (size_t)i * ldo;
    for (int k = lane; k < F; k += 32) dst[k] = src ? __ldg(src + k) : 0.f;
  }
}

__device__ __forceinline__ bool same_key(const int64_t* nt, const int64_t* li, int64_t a, int64_t b) {
  return nt[a] == nt[b] && li[a] == li[b];
}

__global__ void __launch_bounds__(256) typed_scatter_kernel(const float* __restrict__ d_out, int64_t ldd,
                                                            const int64_t* __restrict__ node_type,
                                                            const int64_t* __restrict__ local_idx,
                                                            const int64_t* __restrict__ order, int64_t n, int F, const Tables T) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t p = warp; p < n; p += nwarps) {
    const int64_t i = order[p];
    if (p > 0 && same_key(node_type, local_idx, i, order[p - 1])) continue;   // not a run head
    const int64_t t = node_type[i], j = local_idx[i];
    if (t < 0 || t >= T.n || !T.ptr[t] || j < 0 || j >= T.rows[t]) continue;
    float* dst = T.ptr[t] + (size_t)j * F;
    for (int k0 = 0; k0 < F; k0 += 32) {
      const int k = k0 + lane;
      float acc = 0.f;
      for (int64_t q = p; q < n; ++q) {
        const int64_t r = order[q];
        if (q > p && !same_key(node_type, local_idx, r, i)) break;
        if (k < F) acc += d_out[(size_t)r * ldd + k];
      }
      if (k < F) dst[k] = acc;
    }
  }
}

// Embedding Adam without a dense gradient.  Pass 1 marks the rows of the table the batch touches: head[j] = position in
// `order` of the first node of the run with key (table_type, j).  Pass 2 sweeps the whole table, one warp per row: the
// row's gradient is its run summed exactly as typed_scatter_kernel sums it (0 for rows outside the batch), followed by
// the Adam element update of adam_kernel, and head[j] is reset to -1 for the next call.
__global__ void __launch_bounds__(256) embedding_heads_kernel(const int64_t* __restrict__ node_type,
                                                              const int64_t* __restrict__ local_idx,
                                                              const int64_t* __restrict__ order, int64_t n, int64_t table_type,
                                                              int64_t rows, int32_t* __restrict__ head) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = order[p];
    if (p > 0 && same_key(node_type, local_idx, i, order[p - 1])) continue;
    const int64_t j = local_idx[i];
    if (node_type[i] == table_type && j >= 0 && j < rows) head[j] = (int32_t)p;
  }
}

__global__ void __launch_bounds__(256) embedding_adam_kernel(const float* __restrict__ d_out, int64_t ldd,
                                                             const int64_t* __restrict__ node_type,
                                                             const int64_t* __restrict__ local_idx,
                                                             const int64_t* __restrict__ order, int64_t n, int F,
                                                             float* __restrict__ table, float* __restrict__ exp_avg,
                                                             float* __restrict__ exp_avg_sq, int64_t rows, int32_t* head,
                                                             float lr, float b1, float b2, float eps,
                                                             const int32_t* __restrict__ step) {
  const float t = (float)(*step + 1);
  const float bc1 = 1.f - powf(b1, t), bc2 = 1.f - powf(b2, t);
  const float step_size = lr / bc1, inv_sqrt_bc2 = rsqrtf(bc2);
  const int lane = threadIdx.x & 31;
  const int64_t warp = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5), nwarps = (int64_t)gridDim.x * 8;
  for (int64_t j = warp; j < rows; j += nwarps) {
    const int32_t p = head[j];
    __syncwarp();
    if (p >= 0 && lane == 0) head[j] = -1;
    const int64_t i = p >= 0 ? order[p] : 0;
    const size_t o = (size_t)j * F;
    for (int k = lane; k < F; k += 32) {
      float g = 0.f;
      if (p >= 0)
        for (int64_t q = p; q < n; ++q) {
          const int64_t r = order[q];
          if (q > p && !same_key(node_type, local_idx, r, i)) break;
          g += d_out[(size_t)r * ldd + k];
        }
      adam_update(table[o + k], exp_avg[o + k], exp_avg_sq[o + k], g, b1, b2, eps, step_size, inv_sqrt_bc2);
    }
  }
}

static inline int rows_grid(int64_t n) {
  int64_t g = (n + 7) / 8;
  if (g > 132 * 16) g = 132 * 16;
  return (int)(g < 1 ? 1 : g);
}

}  // namespace b200gnn

using namespace b200gnn;

static int fill_tables(Tables& T, float* const* tables, const int64_t* table_rows, int32_t n_tables) {
  if (n_tables <= 0 || n_tables > MAX_TABLES || !tables || !table_rows) return B200GNN_ERR_BAD_ARG;
  T.n = n_tables;
  for (int t = 0; t < n_tables; ++t) {
    if (table_rows[t] < 0) return B200GNN_ERR_BAD_ARG;
    T.ptr[t] = tables[t]; T.rows[t] = table_rows[t];
  }
  return B200GNN_OK;
}

extern "C" int b200gnn_typed_gather_f32(const float* const* tables, const int64_t* table_rows, int32_t n_tables,
                                        const int64_t* node_type, const int64_t* local_idx, int64_t n, int64_t F,
                                        float* out, int64_t ldo, int32_t* error_flag, void* stream) {
  if (n < 0 || F <= 0 || F > (1 << 20) || ldo < F || !error_flag) return B200GNN_ERR_BAD_ARG;
  Tables T;
  int rc = fill_tables(T, const_cast<float* const*>(tables), table_rows, n_tables);
  if (rc) return rc;
  if (n == 0) return B200GNN_OK;
  if (!node_type || !local_idx || !out) return B200GNN_ERR_BAD_ARG;
  typed_gather_kernel<<<rows_grid(n), 256, 0, (cudaStream_t)stream>>>(T, node_type, local_idx, n, (int)F, out, ldo, error_flag);
  return check_launch();
}

extern "C" int b200gnn_typed_scatter_f32(const float* d_out, int64_t ldd, const int64_t* node_type, const int64_t* local_idx,
                                         const int64_t* order, int64_t n, int64_t F, float* const* d_tables,
                                         const int64_t* table_rows, int32_t n_tables, void* stream) {
  if (n < 0 || F <= 0 || F > (1 << 20) || ldd < F) return B200GNN_ERR_BAD_ARG;
  Tables T;
  int rc = fill_tables(T, d_tables, table_rows, n_tables);
  if (rc) return rc;
  if (n == 0) return B200GNN_OK;
  if (!d_out || !node_type || !local_idx || !order) return B200GNN_ERR_BAD_ARG;
  typed_scatter_kernel<<<rows_grid(n), 256, 0, (cudaStream_t)stream>>>(d_out, ldd, node_type, local_idx, order, n, (int)F, T);
  return check_launch();
}

extern "C" int b200gnn_embedding_adam_f32(const float* d_out, int64_t ldd, const int64_t* node_type, const int64_t* local_idx,
                                          const int64_t* order, int64_t n, int64_t table_type, float* table, float* exp_avg,
                                          float* exp_avg_sq, int64_t rows, int64_t F, int32_t* head, float lr, float beta1,
                                          float beta2, float eps, const int32_t* step, void* stream) {
  if (n < 0 || rows < 0 || rows >= INT32_MAX || n >= INT32_MAX || F <= 0 || F > (1 << 20) || ldd < F || !step)
    return B200GNN_ERR_BAD_ARG;
  if (rows == 0) return B200GNN_OK;
  if (!table || !exp_avg || !exp_avg_sq || !head || (n > 0 && (!d_out || !node_type || !local_idx || !order)))
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (n > 0) {
    int64_t g = (n + 255) / 256;
    embedding_heads_kernel<<<(int)(g > 132 * 8 ? 132 * 8 : g), 256, 0, st>>>(node_type, local_idx, order, n, table_type, rows, head);
    if ((rc = check_launch())) return rc;
  }
  embedding_adam_kernel<<<rows_grid(rows), 256, 0, st>>>(d_out, ldd, node_type, local_idx, order, n, (int)F, table, exp_avg,
                                                         exp_avg_sq, rows, head, lr, beta1, beta2, eps, step);
  return check_launch();
}
