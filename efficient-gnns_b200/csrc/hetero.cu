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
