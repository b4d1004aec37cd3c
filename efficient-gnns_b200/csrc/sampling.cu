// Mini-batch graph sampling on the device (SURVEY §8 f4): what the reference's GraphSAINT loader does on CPU workers with
// torch_sparse (`GraphSAINTRandomWalkSampler(homo_data, batch_size, walk_length=num_layers, num_steps, sample_coverage=0)`,
// mag_pyg/gnn.py:361-366 — roots uniform over the nodes, one uniform random walk per root, the induced subgraph of the
// visited nodes, every node / edge attribute sliced along).
//
//   random_walk     one thread per walker; step s of walker w draws word (s % 4) of Philox4x32-10(seed, offset, w * ceil(L/4)
//                   + s / 4) and moves to col[rowptr[v] + (r * deg >> 32)] — a uniform neighbour; a node without
//                   out-edges holds the walker (torch_sparse.random_walk's rule).  A pure function of (seed, offset, w), so
//                   the oracle restates it bit for bit.  The graph (4 B / edge) is L2-resident after the first step.
//   saint_subgraph  induced subgraph of a SORTED UNIQUE node set S over CSR: a node -> local-id map, one warp per selected
//                   row counting / writing the edges whose column is in S (ballot prefix: CSR order preserved, as
//                   SparseTensor.saint_subgraph keeps it), with the edge ids of the parent graph for attribute slicing.
//   induced_edges   the edges of a batch whose endpoints are both marked in a node mask, relabelled to the endpoints'
//                   ranks among the marked nodes, edge order kept (torch_geometric.utils.subgraph(mask.nonzero(), edge_index,
//                   relabel_nodes=True)[0], the LSP edge list of mag_pyg/gnn_kd_and_aux.py:240-243).  One block scans the
//                   mask into ranks; tiles of IE_TILE edges count their kept edges, one block scans the tile counts, and
//                   the fill rescans each tile with a block prefix sum, so every kept edge lands at its rank in edge order.
// Integer / index work: bit-exact against oracle/sampling.py.
#include "common.cuh"
#include "philox.cuh"

namespace b200gnn {
namespace sampling {

__global__ void __launch_bounds__(256) random_walk_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                          const int64_t* __restrict__ start, int64_t n_walks, int walk_length,
                                                          uint64_t seed, uint64_t offset, int64_t* __restrict__ out) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_walks) return;
  const int blocks_per_walk = (walk_length + 3) / 4;
  int64_t v = start[w];
  int64_t* o = out + w * (walk_length + 1);
  o[0] = v;
  uint4 r = make_uint4(0, 0, 0, 0);
  for (int s = 0; s < walk_length; ++s) {
    if ((s & 3) == 0) r = philox4x32(seed, offset, (uint64_t)w * blocks_per_walk + (s >> 2));
    const uint32_t u = (s & 3) == 0 ? r.x : (s & 3) == 1 ? r.y : (s & 3) == 2 ? r.z : r.w;
    const int32_t b = __ldg(rowptr + v), e = __ldg(rowptr + v + 1);
    const uint32_t deg = (uint32_t)(e - b);
    if (deg > 0) v = __ldg(col + b + (int32_t)(((uint64_t)u * deg) >> 32));
    o[s + 1] = v;
  }
}

__global__ void __launch_bounds__(256) fill_map_kernel(const int64_t* __restrict__ nodes, int64_t n_sel, int32_t* __restrict__ map) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_sel) map[nodes[i]] = (int32_t)i;
}

// FILL = false: counts[i] = kept edges of selected row i.  FILL = true: writes them at out_ptr[i]...
template <bool FILL>
__global__ void __launch_bounds__(256) induced_rows_kernel(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ col,
                                                           const int64_t* __restrict__ eid, const int64_t* __restrict__ nodes,
                                                           int64_t n_sel, const int32_t* __restrict__ map,
                                                           int64_t* __restrict__ counts_or_ptr, int64_t* __restrict__ out_row,
                                                           int64_t* __restrict__ out_col, int64_t* __restrict__ out_eid) {
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n_sel) return;
  const int64_t v = nodes[i];
  const int32_t b = rowptr[v], e = rowptr[v + 1];
  int64_t base = FILL ? counts_or_ptr[i] : 0;
  int64_t cnt = 0;
  for (int32_t j = b + lane; j < ((e - b + 31) / 32) * 32 + b; j += 32) {
    const int32_t c = j < e ? map[col[j]] : -1;
    const unsigned m = __ballot_sync(FULL_MASK, c >= 0);
    if (FILL && c >= 0) {
      const int64_t o = base + __popc(m & ((1u << lane) - 1));
      out_row[o] = i;
      out_col[o] = c;
      out_eid[o] = eid ? eid[j] : (int64_t)j;
    }
    base += __popc(m);
    cnt += __popc(m);
  }
  if (!FILL && lane == 0) counts_or_ptr[i] = cnt;
}

// ---- induced_edges
constexpr int IE_THREADS = 256, IE_ITEMS = 4, IE_TILE = IE_THREADS * IE_ITEMS;
constexpr int SCAN_THREADS = 1024;

// Exclusive prefix sum over the block (blockDim.x == NT); returns the thread's exclusive prefix, *total gets the block sum.
template <int NT>
__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* total) {
  __shared__ int64_t warp_sum[NT / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int64_t o = __shfl_up_sync(FULL_MASK, inc, d);
    if (lane >= d) inc += o;
  }
  if (lane == 31) warp_sum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int64_t w = lane < NT / 32 ? warp_sum[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int64_t o = __shfl_up_sync(FULL_MASK, w, d);
      if (lane >= d) w += o;
    }
    if (lane < NT / 32) warp_sum[lane] = w;                  // inclusive over warps
  }
  __syncthreads();
  const int64_t before = warp == 0 ? 0 : warp_sum[warp - 1];
  *total = warp_sum[NT / 32 - 1];
  return before + inc - v;
}

// One block: out[i] = sum_{j<i} load(j) over [0, n) in contiguous per-thread chunks (exclusive scan); total[0] = the sum.
template <typename Load>
__device__ __forceinline__ void single_block_scan(Load load, int64_t n, int64_t* __restrict__ out, int64_t* __restrict__ total) {
  const int64_t chunk = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const int64_t b = min(n, (int64_t)threadIdx.x * chunk), e = min(n, b + chunk);
  int64_t s = 0;
  for (int64_t i = b; i < e; ++i) s += load(i);
  int64_t all;
  int64_t run = block_exclusive_scan<SCAN_THREADS>(s, &all);
  for (int64_t i = b; i < e; ++i) {
    const int64_t v = load(i);
    out[i] = run;
    run += v;
  }
  if (threadIdx.x == 0) *total = all;
}

__global__ void __launch_bounds__(SCAN_THREADS) mask_rank_kernel(const uint8_t* __restrict__ mask, int64_t n,
                                                                 int64_t* __restrict__ rank, int64_t* __restrict__ n_marked) {
  single_block_scan([&](int64_t i) -> int64_t { return mask[i] != 0; }, n, rank, n_marked);
}

// Kept / out-of-range flags of the IE_ITEMS consecutive edges of this thread (bit k: edge tile·IE_TILE + t·IE_ITEMS + k).
__device__ __forceinline__ void induced_flags(const int64_t* __restrict__ ei, int64_t ld, int64_t E, const uint8_t* __restrict__ mask,
                                              int64_t n, int64_t first, unsigned& keep, int& bad) {
  keep = 0u;
  bad = 0;
#pragma unroll
  for (int k = 0; k < IE_ITEMS; ++k) {
    const int64_t j = first + k;
    if (j >= E) break;
    const int64_t s = ei[j], d = ei[ld + j];
    if (s < 0 || s >= n || d < 0 || d >= n) {
      ++bad;
      continue;
    }
    if (mask[s] && mask[d]) keep |= 1u << k;
  }
}

__global__ void __launch_bounds__(IE_THREADS) induced_count_kernel(const int64_t* __restrict__ ei, int64_t ld, int64_t E,
                                                                   const uint8_t* __restrict__ mask, int64_t n, int64_t n_tiles,
                                                                   int64_t* __restrict__ tile_cnt) {
  unsigned keep;
  int bad;
  induced_flags(ei, ld, E, mask, n, (int64_t)blockIdx.x * IE_TILE + threadIdx.x * IE_ITEMS, keep, bad);
  int64_t all_kept, all_bad;
  block_exclusive_scan<IE_THREADS>(__popc(keep), &all_kept);
  __syncthreads();                                           // warp_sum is reused by the second scan
  block_exclusive_scan<IE_THREADS>(bad, &all_bad);
  if (threadIdx.x == 0) {
    tile_cnt[blockIdx.x] = all_kept;
    tile_cnt[n_tiles + blockIdx.x] = all_bad;
  }
}

// tile_cnt [2, n_tiles] (kept, out of range) -> tile_cnt[0] := exclusive offsets of the kept edges; totals = {kept, bad}.
__global__ void __launch_bounds__(SCAN_THREADS) induced_scan_kernel(int64_t* __restrict__ tile_cnt, int64_t n_tiles,
                                                                    int64_t* __restrict__ totals) {
  int64_t s = 0;
  for (int64_t i = threadIdx.x; i < n_tiles; i += SCAN_THREADS) s += tile_cnt[n_tiles + i];
  int64_t bad;
  block_exclusive_scan<SCAN_THREADS>(s, &bad);
  __syncthreads();
  // the in-place scan reads each count before any thread overwrites it: every thread owns one contiguous chunk
  const int64_t chunk = (n_tiles + SCAN_THREADS - 1) / SCAN_THREADS;
  const int64_t b = min(n_tiles, (int64_t)threadIdx.x * chunk), e = min(n_tiles, b + chunk);
  int64_t c = 0;
  for (int64_t i = b; i < e; ++i) c += tile_cnt[i];
  int64_t kept;
  int64_t run = block_exclusive_scan<SCAN_THREADS>(c, &kept);
  for (int64_t i = b; i < e; ++i) {
    const int64_t v = tile_cnt[i];
    tile_cnt[i] = run;
    run += v;
  }
  if (threadIdx.x == 0) {
    totals[0] = kept;
    totals[1] = bad;
  }
}

__global__ void __launch_bounds__(IE_THREADS) induced_fill_kernel(const int64_t* __restrict__ ei, int64_t ld, int64_t E,
                                                                  const uint8_t* __restrict__ mask, int64_t n,
                                                                  const int64_t* __restrict__ rank, const int64_t* __restrict__ tile_off,
                                                                  int64_t* __restrict__ out, int64_t ld_out) {
  const int64_t first = (int64_t)blockIdx.x * IE_TILE + threadIdx.x * IE_ITEMS;
  unsigned keep;
  int bad;
  induced_flags(ei, ld, E, mask, n, first, keep, bad);
  int64_t all;
  int64_t o = tile_off[blockIdx.x] + block_exclusive_scan<IE_THREADS>(__popc(keep), &all);
#pragma unroll
  for (int k = 0; k < IE_ITEMS; ++k) {
    if (keep & (1u << k)) {
      out[o] = rank[ei[first + k]];
      out[ld_out + o] = rank[ei[ld + first + k]];
      ++o;
    }
  }
}

}  // namespace sampling
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_random_walk_i64(const int32_t* rowptr, const int32_t* col, int64_t n_nodes, const int64_t* start,
                                       int64_t n_walks, int32_t walk_length, uint64_t seed, uint64_t offset, int64_t* out,
                                       void* stream) {
  if (!rowptr || !start || !out || n_nodes <= 0 || n_walks < 0 || walk_length < 0 || walk_length > 4096) return B200GNN_ERR_BAD_ARG;
  if (n_walks == 0) return B200GNN_OK;
  sampling::random_walk_kernel<<<(unsigned)((n_walks + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      rowptr, col, start, n_walks, walk_length, seed, offset, out);
  return check_launch();
}

// node_map: int32 [n_nodes] workspace holding -1 everywhere on entry; the call sets map[v] = position of v in `nodes` for the
// selected nodes.  The caller restores those entries to -1 after the fill call (so one map serves every batch without an
// O(N) memset per batch).
extern "C" int b200gnn_saint_subgraph_count_i64(const int32_t* rowptr, const int32_t* col, const int64_t* nodes, int64_t n_sel,
                                                int32_t* node_map, int64_t* counts, void* stream) {
  if (!rowptr || !nodes || !node_map || !counts || n_sel < 0) return B200GNN_ERR_BAD_ARG;
  if (n_sel == 0) return B200GNN_OK;
  cudaStream_t st = (cudaStream_t)stream;
  sampling::fill_map_kernel<<<(unsigned)((n_sel + 255) / 256), 256, 0, st>>>(nodes, n_sel, node_map);
  int rc;
  if ((rc = check_launch())) return rc;
  sampling::induced_rows_kernel<false><<<(unsigned)((n_sel * 32 + 255) / 256), 256, 0, st>>>(rowptr, col, nullptr, nodes, n_sel, node_map,
                                                                                        counts, nullptr, nullptr, nullptr);
  return check_launch();
}

// out_ptr: exclusive prefix sums of `counts` (int64 [n_sel]); eid: optional parent edge ids per CSR position (NULL: the CSR
// position itself).  Outputs: local row, local column, parent edge id, CSR order.
extern "C" int b200gnn_saint_subgraph_fill_i64(const int32_t* rowptr, const int32_t* col, const int64_t* eid, const int64_t* nodes,
                                               int64_t n_sel, const int32_t* node_map, const int64_t* out_ptr, int64_t* out_row,
                                               int64_t* out_col, int64_t* out_eid, void* stream) {
  if (!rowptr || !nodes || !node_map || !out_ptr || !out_row || !out_col || !out_eid || n_sel < 0) return B200GNN_ERR_BAD_ARG;
  if (n_sel == 0) return B200GNN_OK;
  sampling::induced_rows_kernel<true><<<(unsigned)((n_sel * 32 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      rowptr, col, eid, nodes, n_sel, node_map, const_cast<int64_t*>(out_ptr), out_row, out_col, out_eid);
  return check_launch();
}

extern "C" int64_t b200gnn_induced_edges_tiles(int64_t n_edges) {
  return n_edges < 0 ? -1 : (n_edges + sampling::IE_TILE - 1) / sampling::IE_TILE;
}

// edge_index: int64 rows src (edge_index[0..E)) and dst (edge_index[ld..ld+E)); mask: uint8 / bool [n_nodes].
// rank: int64 [n_nodes + 1] workspace, on return the number of marked nodes before each node (rank[n_nodes]: all); tile_cnt: int64
// [2 * b200gnn_induced_edges_tiles(E)] workspace; totals: int64 [2] = {kept edges, edges with an endpoint outside [0, n)}.
extern "C" int b200gnn_induced_edges_count_i64(const int64_t* edge_index, int64_t ld, int64_t n_edges, const uint8_t* mask,
                                               int64_t n_nodes, int64_t* rank, int64_t* tile_cnt, int64_t* totals, void* stream) {
  if (!mask || !rank || !totals || n_nodes < 0 || n_edges < 0 || (n_edges > 0 && (!edge_index || !tile_cnt || ld < n_edges)))
    return B200GNN_ERR_BAD_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  sampling::mask_rank_kernel<<<1, sampling::SCAN_THREADS, 0, st>>>(mask, n_nodes, rank, rank + n_nodes);
  int rc;
  if ((rc = check_launch())) return rc;
  const int64_t tiles = b200gnn_induced_edges_tiles(n_edges);
  if (tiles == 0) {
    if (cudaMemsetAsync(totals, 0, 2 * sizeof(int64_t), st) != cudaSuccess) return B200GNN_ERR_CUDA;
    return B200GNN_OK;
  }
  if (tiles > 0x7fffffffLL) return B200GNN_ERR_BAD_ARG;
  sampling::induced_count_kernel<<<(unsigned)tiles, sampling::IE_THREADS, 0, st>>>(edge_index, ld, n_edges, mask, n_nodes, tiles,
                                                                                  tile_cnt);
  if ((rc = check_launch())) return rc;
  sampling::induced_scan_kernel<<<1, sampling::SCAN_THREADS, 0, st>>>(tile_cnt, tiles, totals);
  return check_launch();
}

// tile_cnt: as the count call left it; out: int64 rows (out[0..kept) relabelled sources, out[ld_out..ld_out+kept) destinations).
extern "C" int b200gnn_induced_edges_fill_i64(const int64_t* edge_index, int64_t ld, int64_t n_edges, const uint8_t* mask,
                                              int64_t n_nodes, const int64_t* rank, const int64_t* tile_cnt, int64_t* out,
                                              int64_t ld_out, void* stream) {
  if (!mask || !rank || n_nodes < 0 || n_edges < 0 || ld_out < 0 ||
      (n_edges > 0 && (!edge_index || !tile_cnt || !out || ld < n_edges)))
    return B200GNN_ERR_BAD_ARG;
  const int64_t tiles = b200gnn_induced_edges_tiles(n_edges);
  if (tiles == 0) return B200GNN_OK;
  if (tiles > 0x7fffffffLL) return B200GNN_ERR_BAD_ARG;
  sampling::induced_fill_kernel<<<(unsigned)tiles, sampling::IE_THREADS, 0, (cudaStream_t)stream>>>(
      edge_index, ld, n_edges, mask, n_nodes, rank, tile_cnt, out, ld_out);
  return check_launch();
}
