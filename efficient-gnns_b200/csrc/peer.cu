// Peer-memory data path of the node-parallel engine (SURVEY.md §8e): one process per GPU, every rank maps the other
// ranks' exchange arenas through CUDA IPC and the exchange steps of a training step are plain kernels that STORE
// straight into the consumers' buffers over NVLink/NVSwitch, followed by a flag barrier — no collective library call on
// the data path.  The reference is single-GPU (arxiv_pyg/scripts/run_gcn.sh:24-28); this is the native multi-GPU extension
// BASELINE.json's north_star asks for.
//
//   b200gnn_arena_alloc / _free        cudaMalloc'd arena (IPC handles need a cudaMalloc allocation, not a sub-block of
//                                      a caching allocator's segment)
//   b200gnn_ipc_get_handle / _open / _close   cudaIpc* wrappers (64-byte opaque handle, exchanged by the host side)
//   b200gnn_peer_copy2d_f32            n strided 2-D block copies in one launch: dst_j[r, 0:width] = src_j[r, 0:width];
//                                      dst_j may live in a peer's arena (row <-> column layout exchanges, all-gathers)
//   b200gnn_peer_barrier               every rank stores epoch e into slot [rank] of each peer's flag array
//                                      (st.release.sys after a system-scope fence), then spins until its own slots all
//                                      reached e: data written before the barrier is visible to kernels after it
#include "common.cuh"

namespace b200gnn {
namespace peer {

constexpr int MAX_WORLD = 16;
constexpr int MAX_COPIES = 16;

struct CopyParams {
  float* dst[MAX_COPIES];
  const float* src[MAX_COPIES];
  int64_t ld_dst[MAX_COPIES], ld_src[MAX_COPIES], rows[MAX_COPIES];
  int32_t n, nvec;     // nvec = width / 4
};

struct BarrierParams {
  uint64_t* flags[MAX_WORLD];   // flags[q] = rank q's flag array (MAX_WORLD slots), mapped in this process
  uint64_t* epoch;              // local device counter (number of barriers passed)
  int32_t* error;               // set to 1 if a wait gave up (a peer never arrived)
  int32_t rank, world;
  uint64_t spin_limit;
};

// signal every rank (slot [rank] of its flag array <- epoch+1, release at system scope), wait for all of ours; one warp
__device__ __forceinline__ void flag_barrier(const BarrierParams& p, int q) {
  const uint64_t e = *p.epoch + 1;
  if (q < p.world) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p.flags[q] + p.rank), "l"(e) : "memory");
    const uint64_t* mine = p.flags[p.rank] + q;
    uint64_t seen = 0, spins = 0;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(seen) : "l"(mine) : "memory");
      if (++spins > p.spin_limit) { *p.error = 1; break; }
    } while (seen < e);
  }
  __syncwarp();
  if (q == 0) *p.epoch = e;
}

// grid = (ctas_per_copy, n): copy j is spread over gridDim.x CTAs; each thread moves float4s, rows x nvec per copy
// FUSED = the exchange in ONE kernel: the CTA that finishes last (ticket counter) runs the flag barrier, so the kernel ends
// when every rank's blocks have landed here and ours have landed there.
template <bool FUSED>
__global__ void __launch_bounds__(256) copy2d_kernel(const CopyParams p, const BarrierParams bp, unsigned int* __restrict__ ticket) {
  const int j = blockIdx.y;
  const int64_t rows = p.rows[j];
  const int nvec = p.nvec;
  const float4* __restrict__ src = reinterpret_cast<const float4*>(p.src[j]);
  float4* __restrict__ dst = reinterpret_cast<float4*>(p.dst[j]);
  const int64_t lds = p.ld_src[j] / 4, ldd = p.ld_dst[j] / 4;
  const int64_t total = rows * nvec;
  // consecutive lanes move consecutive float4s (whole 512-byte warp transactions: what NVLink wants); 4 independent
  // loads in flight per thread before the stores
  for (int64_t b0 = (int64_t)blockIdx.x * 1024 + threadIdx.x; b0 < total; b0 += (int64_t)gridDim.x * 1024) {
    float4 v[4];
    int64_t r[4]; int c[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int64_t i = b0 + u * 256;
      r[u] = i / nvec; c[u] = (int)(i - r[u] * nvec);
      if (i < total) v[u] = __ldg(src + r[u] * lds + c[u]);
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (b0 + u * 256 < total) dst[r[u] * ldd + c[u]] = v[u];
  }
  if (FUSED) {
    __shared__ unsigned int s_last;
    __threadfence_system();                       // this CTA's stores (peer memory included) before its ticket
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned int total_ctas = gridDim.x * gridDim.y;
      const unsigned int t = atomicAdd(ticket, 1u);
      s_last = (t == total_ctas - 1) ? 1u : 0u;
      if (s_last) *ticket = 0u;                   // re-armed for the next launch (stream-ordered)
    }
    __syncthreads();
    if (s_last && threadIdx.x < 32) {
      __threadfence();                            // acquire side of the ticket chain
      flag_barrier(bp, threadIdx.x);
    }
  }
}

__global__ void __launch_bounds__(32) barrier_kernel(const BarrierParams p) { flag_barrier(p, threadIdx.x); }

}  // namespace peer
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_arena_alloc(int64_t bytes, void** out) {
  if (bytes <= 0 || !out) return B200GNN_ERR_BAD_ARG;
  cudaError_t e = cudaMalloc(out, (size_t)bytes);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  e = cudaMemset(*out, 0, (size_t)bytes);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  return B200GNN_OK;
}

extern "C" int b200gnn_arena_free(void* ptr) {
  if (!ptr) return B200GNN_OK;
  cudaError_t e = cudaFree(ptr);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  return B200GNN_OK;
}

extern "C" int b200gnn_ipc_get_handle(const void* dev_ptr, void* handle64) {
  if (!dev_ptr || !handle64) return B200GNN_ERR_BAD_ARG;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
  cudaIpcMemHandle_t h;
  cudaError_t e = cudaIpcGetMemHandle(&h, const_cast<void*>(dev_ptr));
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  memcpy(handle64, &h, 64);
  return B200GNN_OK;
}

extern "C" int b200gnn_ipc_open_handle(const void* handle64, void** out) {
  if (!handle64 || !out) return B200GNN_ERR_BAD_ARG;
  cudaIpcMemHandle_t h;
  memcpy(&h, handle64, 64);
  cudaError_t e = cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  return B200GNN_OK;
}

extern "C" int b200gnn_ipc_close_handle(void* ptr) {
  if (!ptr) return B200GNN_OK;
  cudaError_t e = cudaIpcCloseMemHandle(ptr);
  if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
  return B200GNN_OK;
}

static int fill_copies(peer::CopyParams& p, const b200gnn_copy2d* copies, int32_t n, int64_t width, dim3* grid) {
  if (n < 0 || n > peer::MAX_COPIES || (n > 0 && !copies) || width <= 0 || width % 4) return B200GNN_ERR_BAD_ARG;
  int64_t max_rows = 0;
  int m = 0;
  for (int j = 0; j < n; ++j) {
    const b200gnn_copy2d& c = copies[j];
    if (c.rows < 0 || (c.rows > 0 && (!c.dst || !c.src)) || c.ld_dst < width || c.ld_src < width || c.ld_dst % 4 || c.ld_src % 4 ||
        !aligned_to(c.dst, 16) || !aligned_to(c.src, 16))
      return B200GNN_ERR_BAD_ARG;
    if (c.rows == 0) continue;
    p.dst[m] = c.dst; p.src[m] = c.src; p.ld_dst[m] = c.ld_dst; p.ld_src[m] = c.ld_src; p.rows[m] = c.rows;
    if (c.rows > max_rows) max_rows = c.rows;
    ++m;
  }
  p.n = m; p.nvec = (int32_t)(width / 4);
  if (m == 0) { *grid = dim3(0, 0); return B200GNN_OK; }
  const int64_t vecs = max_rows * p.nvec;
  int64_t per = (vecs + 1023) / 1024;                 // 256 threads x 4 float4 per pass
  const int64_t cap = (132 * 8 + m - 1) / m;         // about 8 CTAs per SM over all copies
  if (per > cap) per = cap;
  if (per < 1) per = 1;
  *grid = dim3((unsigned)per, (unsigned)m);
  return B200GNN_OK;
}

static int fill_barrier(peer::BarrierParams& p, uint64_t* const* peer_flags, int32_t rank, int32_t world, uint64_t* epoch,
                        int32_t* error) {
  if (!peer_flags || !epoch || !error || world <= 0 || world > peer::MAX_WORLD || rank < 0 || rank >= world)
    return B200GNN_ERR_BAD_ARG;
  for (int q = 0; q < world; ++q) {
    if (!peer_flags[q]) return B200GNN_ERR_BAD_ARG;
    p.flags[q] = peer_flags[q];
  }
  p.epoch = epoch; p.error = error; p.rank = rank; p.world = world;
  p.spin_limit = (uint64_t)1 << 27;                   // ~ seconds: a missing peer becomes an error flag, not a hung GPU
  return B200GNN_OK;
}

extern "C" int b200gnn_peer_copy2d_f32(const b200gnn_copy2d* copies, int32_t n, int64_t width, void* stream) {
  peer::CopyParams p;
  dim3 grid;
  int rc = fill_copies(p, copies, n, width, &grid);
  if (rc || grid.x == 0) return rc;
  peer::BarrierParams none = {};
  peer::copy2d_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(p, none, nullptr);
  return check_launch();
}

extern "C" int b200gnn_peer_barrier(uint64_t* const* peer_flags, int32_t rank, int32_t world, uint64_t* epoch, int32_t* error,
                                    void* stream) {
  peer::BarrierParams p;
  int rc = fill_barrier(p, peer_flags, rank, world, epoch, error);
  if (rc) return rc;
  peer::barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(p);
  return check_launch();
}

// One exchange = one launch: the copies above, then (in the CTA that finishes last) the flag barrier.
// ticket: device uint32, zero-initialised, private to this rank (re-armed by the kernel).
extern "C" int b200gnn_peer_exchange_f32(const b200gnn_copy2d* copies, int32_t n, int64_t width, uint64_t* const* peer_flags,
                                         int32_t rank, int32_t world, uint64_t* epoch, int32_t* error, uint32_t* ticket,
                                         void* stream) {
  if (!ticket) return B200GNN_ERR_BAD_ARG;
  peer::CopyParams p;
  peer::BarrierParams bp;
  dim3 grid;
  int rc = fill_copies(p, copies, n, width, &grid);
  if (rc) return rc;
  if ((rc = fill_barrier(bp, peer_flags, rank, world, epoch, error))) return rc;
  if (grid.x == 0) {                                  // nothing to move: still a barrier
    peer::barrier_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(bp);
    return check_launch();
  }
  peer::copy2d_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(p, bp, ticket);
  return check_launch();
}
