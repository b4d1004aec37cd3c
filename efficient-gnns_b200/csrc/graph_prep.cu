// Graph ingestion on the device (SURVEY.md §8 f2): the integer half of the reference's data path —
//   T.ToSparseTensor()            arxiv_pyg/gnn.py:236-237   sort edges by (dst, src) -> CSR of A^T
//   adj_t.to_symmetric()          arxiv_pyg/gnn.py:240       concat both directions + coalesce (sort by row*N+col, drop duplicates)
//   SparseTensor(row=col,col=row) mag_pyg/gnn.py:151         sort on construction, once per relation per inference call
//   csr2csc                       torch_sparse storage       argsort(col*M+row): the backward's CSC view
// — as hand-written kernels: a stable LSD radix sort of 64-bit keys carrying a 32-bit payload (8-bit digits; only
// the digits below the key's bit length are sorted), duplicate flags + exclusive scan + compaction, and row pointers by
// binary search.  Everything is integer work and bit-exact against oracle/graph.py (numpy).  One-off per graph: the
// kernels favour simplicity and determinism (no atomics on the output order) over the last percent of bandwidth.
#include "common.cuh"

namespace b200gnn {
namespace prep {

constexpr int RADIX_BITS = 8, RADIX = 256;
constexpr int SORT_THREADS = 256, SORT_WARPS = 8, SORT_ITEMS = 8;
constexpr int SORT_TILE = SORT_THREADS * SORT_ITEMS;       // 2048 keys per CTA; warp w owns keys [w*256, (w+1)*256) of the tile

__global__ void __launch_bounds__(256) make_keys_kernel(const int64_t* __restrict__ hi, const int64_t* __restrict__ lo, int64_t n,
                                                        uint64_t mul, uint64_t* __restrict__ keys, int32_t* __restrict__ idx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    keys[i] = (uint64_t)hi[i] * mul + (uint64_t)lo[i];
    idx[i] = (int32_t)i;
  }
}

// per-CTA digit histogram -> hist[digit][block]
__global__ void __launch_bounds__(SORT_THREADS) radix_hist_kernel(const uint64_t* __restrict__ keys, int64_t n, int shift,
                                                                  int32_t* __restrict__ hist, int nblocks) {
  __shared__ int s_h[RADIX];
  s_h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE;
  for (int i = threadIdx.x; i < SORT_TILE; i += SORT_THREADS) {
    const int64_t k = base + i;
    if (k < n) atomicAdd(&s_h[(keys[k] >> shift) & (RADIX - 1)], 1);      // counts only: order-independent
  }
  __syncthreads();
  hist[(size_t)threadIdx.x * nblocks + blockIdx.x] = s_h[threadIdx.x];
}

// exclusive scan of an int32 array in place, one CTA (n is a few hundred thousand at most: 256 digits x #tiles)
__global__ void __launch_bounds__(1024) scan_single_cta_kernel(int32_t* __restrict__ a, int64_t n) {
  __shared__ int s_w[32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int64_t b = 0; b < n; b += 1024) {
    const int64_t i = b + threadIdx.x;
    const int v = i < n ? a[i] : 0;
    int x = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(FULL_MASK, x, d); if (lane >= d) x += o; }
    if (lane == 31) s_w[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = s_w[lane], y = w;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(FULL_MASK, y, d); if (lane >= d) y += o; }
      s_w[lane] = y - w;
    }
    __syncthreads();
    const int excl = s_carry + s_w[warp] + x - v;
    if (i < n) a[i] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) s_carry = excl + v;
    __syncthreads();
  }
}

// stable scatter of one digit pass.  Element order inside a tile: warp w, round r, lane l  <->  tile index w*256 + r*32 + l.
__global__ void __launch_bounds__(SORT_THREADS) radix_scatter_kernel(const uint64_t* __restrict__ keys_in, const int32_t* __restrict__ idx_in,
                                                                     int64_t n, int shift, const int32_t* __restrict__ offs, int nblocks,
                                                                     uint64_t* __restrict__ keys_out, int32_t* __restrict__ idx_out) {
  __shared__ int s_cnt[SORT_WARPS][RADIX];       // per-warp digit counts, then running positions
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < SORT_WARPS * RADIX; i += SORT_THREADS) (&s_cnt[0][0])[i] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * SORT_TILE + warp * (32 * SORT_ITEMS);
  uint64_t key[SORT_ITEMS];
  int32_t pay[SORT_ITEMS];
  int dig[SORT_ITEMS];
#pragma unroll
  for (int r = 0; r < SORT_ITEMS; ++r) {
    const int64_t k = base + r * 32 + lane;
    const bool ok = k < n;
    key[r] = ok ? keys_in[k] : ~0ull;
    pay[r] = ok ? idx_in[k] : 0;
    dig[r] = ok ? (int)((key[r] >> shift) & (RADIX - 1)) : -1;
  }
  // phase A: per-warp digit counts
#pragma unroll
  for (int r = 0; r < SORT_ITEMS; ++r) {
    const unsigned peers = __match_any_sync(FULL_MASK, dig[r]);
    if (dig[r] >= 0 && (peers & ((1u << lane) - 1)) == 0) s_cnt[warp][dig[r]] += __popc(peers);
    __syncwarp();
  }
  __syncthreads();
  // phase B: per digit, exclusive scan over the warps + the CTA's global offset -> starting position of each warp
  {
    const int d = threadIdx.x;                   // 256 threads = 256 digits
    int run = offs[(size_t)d * nblocks + blockIdx.x];
#pragma unroll
    for (int w = 0; w < SORT_WARPS; ++w) { const int c = s_cnt[w][d]; s_cnt[w][d] = run; run += c; }
  }
  __syncthreads();
  // phase C: stable ranks round by round, scatter
#pragma unroll
  for (int r = 0; r < SORT_ITEMS; ++r) {
    const unsigned peers = __match_any_sync(FULL_MASK, dig[r]);
    int pos = 0;
    if (dig[r] >= 0) pos = s_cnt[warp][dig[r]] + __popc(peers & ((1u << lane) - 1));
    __syncwarp();
    if (dig[r] >= 0 && (peers & ((1u << lane) - 1)) == 0) s_cnt[warp][dig[r]] += __popc(peers);
    __syncwarp();
    if (dig[r] >= 0) { keys_out[pos] = key[r]; idx_out[pos] = pay[r]; }
  }
}

// flags[i] = 1 if sorted key i starts a new run
__global__ void __launch_bounds__(256) run_flags_kernel(const uint64_t* __restrict__ keys, int64_t n, int32_t* __restrict__ flags) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    flags[i] = (i == 0 || keys[i] != keys[i - 1]) ? 1 : 0;
}

// ---- device-wide exclusive scan (int32) in three kernels: block sums, scan of the sums, add back
constexpr int SCAN_TILE = 2048;
__global__ void __launch_bounds__(256) scan_block_sums_kernel(const int32_t* __restrict__ a, int64_t n, int32_t* __restrict__ sums) {
  __shared__ int s_w[8];
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE;
  int t = 0;
  for (int i = threadIdx.x; i < SCAN_TILE; i += 256) { const int64_t k = base + i; t += k < n ? a[k] : 0; }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) t += __shfl_xor_sync(FULL_MASK, t, d);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x == 0) { int s = 0; for (int w = 0; w < 8; ++w) s += s_w[w]; sums[blockIdx.x] = s; }
}
__global__ void __launch_bounds__(256) scan_apply_kernel(const int32_t* __restrict__ a, int64_t n, const int32_t* __restrict__ sums_excl,
                                                         int32_t* __restrict__ out) {
  // each thread owns 8 consecutive elements of the tile -> sequential local scan, warp scan of thread totals, warp totals
  __shared__ int s_w[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t base = (int64_t)blockIdx.x * SCAN_TILE + threadIdx.x * 8;
  int v[8], tot = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) { const int64_t k = base + j; v[j] = k < n ? a[k] : 0; tot += v[j]; }
  int x = tot;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int o = __shfl_up_sync(FULL_MASK, x, d); if (lane >= d) x += o; }
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  int wbase = 0;
  for (int w = 0; w < warp; ++w) wbase += s_w[w];
  int run = sums_excl[blockIdx.x] + wbase + x - tot;
#pragma unroll
  for (int j = 0; j < 8; ++j) { const int64_t k = base + j; if (k < n) out[k] = run; run += v[j]; }
}

// kept entry p (= run head i with pos[i] == p): row/col from the key, source index of the FIRST duplicate (stable sort)
__global__ void __launch_bounds__(256) compact_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ idx,
                                                      const int32_t* __restrict__ flags, const int32_t* __restrict__ pos, int64_t n,
                                                      uint64_t div, int64_t* __restrict__ out_hi, int64_t* __restrict__ out_lo,
                                                      int32_t* __restrict__ out_src, int64_t* __restrict__ n_out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (flags[i]) {
      const int p = pos[i];
      const uint64_t k = keys[i];
      out_hi[p] = (int64_t)(k / div);
      out_lo[p] = (int64_t)(k % div);
      if (out_src) out_src[p] = idx[i];
    }
    if (i == n - 1) *n_out = (int64_t)pos[i] + flags[i];
  }
}

// rowptr[r] = number of sorted entries with row < r  (lower bound), r = 0..n_rows
__global__ void __launch_bounds__(256) rowptr_kernel(const int64_t* __restrict__ rows, const int64_t* __restrict__ nnz_dev, int64_t nnz_host,
                                                     int64_t n_rows, int64_t* __restrict__ rowptr) {
  const int64_t nnz = nnz_dev ? *nnz_dev : nnz_host;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r <= n_rows; r += (int64_t)gridDim.x * blockDim.x) {
    int64_t lo = 0, hi = nnz;
    while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (rows[mid] < r) lo = mid + 1; else hi = mid; }
    rowptr[r] = lo;
  }
}

static inline int grid1d(int64_t n, int per = 256, int cap = 132 * 16) {
  int64_t g = (n + per - 1) / per;
  if (g > cap) g = cap;
  return (int)(g < 1 ? 1 : g);
}
static inline int key_bits(uint64_t max_key) {
  int b = 1;
  while (b < 64 && (max_key >> b)) ++b;
  return b;
}

struct Workspace {            // carved from the caller's buffer (b200gnn_graph_sort_workspace_bytes)
  uint64_t* keys[2];
  int32_t* idx[2];
  int32_t* hist;
  int32_t* flags;
  int32_t* pos;
  int32_t* sums;
};
static inline int64_t al256(int64_t b) { return (b + 255) / 256 * 256; }
static int64_t carve(Workspace* w, void* base, int64_t n) {
  const int64_t nblocks = (n + SORT_TILE - 1) / SORT_TILE, nsum = (n + SCAN_TILE - 1) / SCAN_TILE;
  int64_t off = 0;
  auto take = [&](int64_t bytes) { void* p = base ? (char*)base + off : nullptr; off += al256(bytes); return p; };
  for (int i = 0; i < 2; ++i) { void* p = take(n * 8); if (w) w->keys[i] = (uint64_t*)p; }
  for (int i = 0; i < 2; ++i) { void* p = take(n * 4); if (w) w->idx[i] = (int32_t*)p; }
  { void* p = take((int64_t)RADIX * nblocks * 4); if (w) w->hist = (int32_t*)p; }
  { void* p = take(n * 4); if (w) w->flags = (int32_t*)p; }
  { void* p = take(n * 4); if (w) w->pos = (int32_t*)p; }
  { void* p = take((nsum + 1) * 4); if (w) w->sums = (int32_t*)p; }
  return off;
}

// sorts (keys[0], idx[0]) by the low `bits` bits; returns which buffer (0/1) holds the result
static int radix_sort(Workspace& w, int64_t n, int bits, cudaStream_t st, int* rc) {
  const int nblocks = (int)((n + SORT_TILE - 1) / SORT_TILE);
  int cur = 0;
  for (int shift = 0; shift < bits; shift += RADIX_BITS) {
    radix_hist_kernel<<<nblocks, SORT_THREADS, 0, st>>>(w.keys[cur], n, shift, w.hist, nblocks);
    if ((*rc = check_launch())) return cur;
    scan_single_cta_kernel<<<1, 1024, 0, st>>>(w.hist, (int64_t)RADIX * nblocks);
    if ((*rc = check_launch())) return cur;
    radix_scatter_kernel<<<nblocks, SORT_THREADS, 0, st>>>(w.keys[cur], w.idx[cur], n, shift, w.hist, nblocks, w.keys[cur ^ 1], w.idx[cur ^ 1]);
    if ((*rc = check_launch())) return cur;
    cur ^= 1;
  }
  return cur;
}

}  // namespace prep
}  // namespace b200gnn

using namespace b200gnn;
using namespace b200gnn::prep;

extern "C" int64_t b200gnn_graph_sort_workspace_bytes(int64_t n) {
  if (n < 0) return B200GNN_ERR_BAD_ARG;
  return carve(nullptr, nullptr, n < 1 ? 1 : n);
}

// perm_out[i] = index of the entry that is i-th in the order of key = major[i]*minor_size + minor[i] (stable) —
// torch's (major*minor_size + minor).argsort(stable) of ToSparseTensor / csr2csc, SURVEY Appendix A.1.
extern "C" int b200gnn_graph_argsort_i64(const int64_t* major, const int64_t* minor, int64_t n, int64_t major_size, int64_t minor_size,
                                         int32_t* perm_out, void* workspace, void* stream) {
  if (n < 0 || major_size <= 0 || minor_size <= 0 || n >= INT32_MAX) return B200GNN_ERR_BAD_ARG;
  if (n == 0) return B200GNN_OK;
  if (!major || !minor || !perm_out || !workspace) return B200GNN_ERR_BAD_ARG;
  if ((double)major_size * (double)minor_size >= 1.8e19) return B200GNN_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w;
  carve(&w, workspace, n);
  int rc;
  make_keys_kernel<<<grid1d(n), 256, 0, st>>>(major, minor, n, (uint64_t)minor_size, w.keys[0], w.idx[0]);
  if ((rc = check_launch())) return rc;
  const int cur = radix_sort(w, n, key_bits((uint64_t)major_size * (uint64_t)minor_size - 1), st, &rc);
  if (rc) return rc;
  cudaError_t e = cudaMemcpyAsync(perm_out, w.idx[cur], (size_t)n * 4, cudaMemcpyDeviceToDevice, st);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  return B200GNN_OK;
}

// COO -> row-sorted, duplicate-free COO + rowptr: SparseTensor(row=, col=) construction + coalesce (to_symmetric's second
// half, arxiv_pyg/gnn.py:240; mag_pyg/gnn.py:151).  out_row/out_col [n] (first *nnz_out entries valid), src_out [n]
// (nullable) = input index of each kept entry (first of its duplicates), rowptr_out [n_rows+1], nnz_out: device int64.
extern "C" int b200gnn_graph_coalesce_i64(const int64_t* row, const int64_t* col, int64_t n, int64_t n_rows, int64_t n_cols,
                                          int64_t* out_row, int64_t* out_col, int32_t* src_out, int64_t* rowptr_out,
                                          int64_t* nnz_out, void* workspace, void* stream) {
  if (n < 0 || n_rows <= 0 || n_cols <= 0 || n >= INT32_MAX || !rowptr_out || !nnz_out) return B200GNN_ERR_BAD_ARG;
  if ((double)n_rows * (double)n_cols >= 1.8e19) return B200GNN_ERR_UNSUPPORTED;
  cudaStream_t st = (cudaStream_t)stream;
  int rc;
  if (n == 0) {
    cudaError_t e = cudaMemsetAsync(nnz_out, 0, 8, st);
    if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
    rowptr_kernel<<<grid1d(n_rows + 1), 256, 0, st>>>(nullptr, nullptr, 0, n_rows, rowptr_out);
    return check_launch();
  }
  if (!row || !col || !out_row || !out_col || !workspace) return B200GNN_ERR_BAD_ARG;
  Workspace w;
  carve(&w, workspace, n);
  make_keys_kernel<<<grid1d(n), 256, 0, st>>>(row, col, n, (uint64_t)n_cols, w.keys[0], w.idx[0]);
  if ((rc = check_launch())) return rc;
  const int cur = radix_sort(w, n, key_bits((uint64_t)n_rows * (uint64_t)n_cols - 1), st, &rc);
  if (rc) return rc;
  run_flags_kernel<<<grid1d(n), 256, 0, st>>>(w.keys[cur], n, w.flags);
  if ((rc = check_launch())) return rc;
  const int nsum = (int)((n + SCAN_TILE - 1) / SCAN_TILE);
  scan_block_sums_kernel<<<nsum, 256, 0, st>>>(w.flags, n, w.sums);
  if ((rc = check_launch())) return rc;
  scan_single_cta_kernel<<<1, 1024, 0, st>>>(w.sums, nsum);
  if ((rc = check_launch())) return rc;
  scan_apply_kernel<<<nsum, 256, 0, st>>>(w.flags, n, w.sums, w.pos);
  if ((rc = check_launch())) return rc;
  compact_kernel<<<grid1d(n), 256, 0, st>>>(w.keys[cur], w.idx[cur], w.flags, w.pos, n, (uint64_t)n_cols, out_row, out_col, src_out,
                                            nnz_out);
  if ((rc = check_launch())) return rc;
  rowptr_kernel<<<grid1d(n_rows + 1), 256, 0, st>>>(out_row, nnz_out, 0, n_rows, rowptr_out);
  return check_launch();
}
