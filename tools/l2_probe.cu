// Micro-probe: how fast can the 132 SMs of an H100 gather random rows (the SpMM access pattern), and how large a table
// stays L2-resident when every SM reads all of it?
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a tools/l2_probe.cu -o /tmp/l2_probe && /tmp/l2_probe
// Fetch instructions, each as the SpMM kernels issue it (8 warps per CTA, 3 CTAs per SM):
//   lane_cp_async  every lane copies 16-byte slices of the rows with cp.async.cg into a per-warp 8 KB shared-memory ring,
//                  groups of rows retire with cp.async.wait_group (spmm_rows_slab_kernel);
//   lane_ldg       every lane loads 16-byte slices with ld.global.nc into registers, 8 loads in flight per lane;
//   bulk           one cp.async.bulk per row into the ring, completion on mbarriers (spmm_rows_bulk_kernel's data path).
// Row indices are a hash of the position in the gather stream (no index array competing for L2).  Sweeps the table size
// (8 .. 192 MB) and the row size (128 / 256 / 1024 B); prints one JSON line per point with the gathered bytes per second.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int THREADS = 256, CTAS_PER_SM = 3, RING = 8192;

__device__ __forceinline__ uint32_t hash_idx(uint32_t i) {   // murmur3 finaliser
  i ^= i >> 16; i *= 0x85ebca6bu; i ^= i >> 13; i *= 0xc2b2ae35u; i ^= i >> 16;
  return i;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// RB = row bytes; each warp gathers rows [lo, lo + per) of the stream.
template <int RB>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM) gather_lane_cp_async(const char* __restrict__ X, uint32_t n_rows,
                                                                              int per, float* sink) {
  constexpr int P = RB / 16, D = RING / RB, G = D >= 16 ? 8 : D / 2, NG = D / G, PIECES = G * P / 32;
  static_assert(PIECES >= 1 && NG >= 2, "ring geometry");
  extern __shared__ __align__(128) char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  char* ring = smem + warp * RING;
  const uint32_t lo = (uint32_t)((blockIdx.x * THREADS + threadIdx.x) >> 5) * (uint32_t)per;
  float acc = 0.f;
  auto issue = [&](int jg, int slot0) {
    if (jg < per) {
#pragma unroll
      for (int i = 0; i < PIECES; ++i) {
        const int q = i * 32 + lane, u = q / P, off = q % P;
        const uint32_t r = hash_idx(lo + jg + u) % n_rows;
        cp_async16(ring + (slot0 + u) * RB + off * 16, X + (size_t)r * RB + off * 16);
      }
    }
    cp_async_commit();
  };
#pragma unroll
  for (int g = 0; g < NG; ++g) issue(g * G, g * G);
#pragma unroll 1
  for (int j = 0, s0 = 0; j < per; j += G, s0 = (s0 + G) & (D - 1)) {
    cp_async_wait<NG - 1>();
    __syncwarp();                                   // slices copied by other lanes are visible
#pragma unroll
    for (int u = 0; u < G; ++u)
#pragma unroll
      for (int v = 0; v < RB / 128; ++v) acc += reinterpret_cast<const float*>(ring + (s0 + u) * RB)[v * 32 + lane];
    __syncwarp();                                   // every lane has read the slots before they are refilled
    issue(j + D, s0);
  }
  cp_async_wait<0>();
  if (acc == 123.456f) sink[0] = acc;
}

template <int RB>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM) gather_lane_ldg(const char* __restrict__ X, uint32_t n_rows, int per,
                                                                         float* sink) {
  constexpr int P = RB / 16, U = 8, ROWS = U * 32 / P;   // rows per step: 8 loads per lane in flight
  const int lane = threadIdx.x & 31;
  const uint32_t lo = (uint32_t)((blockIdx.x * THREADS + threadIdx.x) >> 5) * (uint32_t)per;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
  for (int j = 0; j < per; j += ROWS) {
    float4 v[U];
#pragma unroll
    for (int i = 0; i < U; ++i) {
      const int q = i * 32 + lane, u = q / P, off = q % P;
      const uint32_t r = hash_idx(lo + j + u) % n_rows;
      v[i] = __ldg(reinterpret_cast<const float4*>(X + (size_t)r * RB + off * 16));
    }
#pragma unroll
    for (int i = 0; i < U; ++i) { acc.x += v[i].x; acc.y += v[i].y; acc.z += v[i].z; acc.w += v[i].w; }
  }
  if (acc.x == 123.456f) sink[0] = acc.x;
}

// one cp.async.bulk per row, G rows per mbarrier group (spmm_rows_bulk_kernel<2, 4>: 1 KB slots, 8 KB ring, G = 4)
template <int RB, int G>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM) gather_bulk(const char* __restrict__ X, uint32_t n_rows, int per,
                                                                     float* sink) {
  constexpr int D = RING / RB, NG = D / G;
  extern __shared__ __align__(128) char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  char* ring = smem + warp * RING;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (THREADS / 32) * RING) + warp * NG;
  if (lane < NG) mbar_init(bars + lane, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();
  const uint32_t lo = (uint32_t)((blockIdx.x * THREADS + threadIdx.x) >> 5) * (uint32_t)per;
  float acc = 0.f;
  uint32_t phases = 0;
  auto issue = [&](int jg, int slot0, int b) {
    if (jg >= per) return;
    if (lane == 0) mbar_expect_tx(bars + b, G * RB);
    if (lane < G) bulk_g2s(ring + (slot0 + lane) * RB, X + (size_t)(hash_idx(lo + jg + lane) % n_rows) * RB, RB, bars + b);
  };
#pragma unroll
  for (int g = 0; g < NG; ++g) issue(g * G, g * G, g);
  int b = 0;
#pragma unroll 1
  for (int j = 0, s0 = 0; j < per; j += G) {
    mbar_wait(bars + b, (phases >> b) & 1u);
    phases ^= 1u << b;
#pragma unroll
    for (int u = 0; u < G; ++u)
#pragma unroll
      for (int v = 0; v < RB / 128; ++v) acc += reinterpret_cast<const float*>(ring + (s0 + u) * RB)[v * 32 + lane];
    __syncwarp();
    issue(j + D, s0, b);
    s0 = (s0 + G) & (D - 1);
    b = b + 1 == NG ? 0 : b + 1;
  }
  if (acc == 123.456f) sink[0] = acc;
}

template <typename Kern>
static void run(const char* name, Kern kern, int smem, const char* X, size_t table_bytes, int rb, int n_sm, float* sink) {
  const int grid = n_sm * CTAS_PER_SM, warps = grid * THREADS / 32;
  const int per = (int)(((size_t)512 << 20) / rb / warps) / 32 * 32;   // about 512 MB gathered per launch
  const uint32_t n_rows = (uint32_t)(table_bytes / rb);
  if (smem > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  for (int it = 0; it < 2; ++it) kern<<<grid, THREADS, smem>>>(X, n_rows, per, sink);   // warm-up: the table lands in L2
  cudaEventRecord(a);
  for (int it = 0; it < 10; ++it) kern<<<grid, THREADS, smem>>>(X, n_rows, per, sink);
  cudaEventRecord(b);
  cudaEventSynchronize(b);
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  ms /= 10;
  const cudaError_t e = cudaGetLastError();
  printf("{\"probe\":\"%s\",\"table_MB\":%zu,\"row_bytes\":%d,\"GBps\":%.1f,\"err\":\"%s\"}\n", name, table_bytes >> 20, rb,
         (double)warps * per * rb / ms / 1e6, e == cudaSuccess ? "" : cudaGetErrorString(e));
  fflush(stdout);
  cudaEventDestroy(a); cudaEventDestroy(b);
}

int main() {
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("{\"device\":\"%s\",\"sms\":%d,\"l2_MB\":%.1f}\n", prop.name, prop.multiProcessorCount, prop.l2CacheSize / 1048576.0);
  const int n_sm = prop.multiProcessorCount;
  const int ring_smem = (THREADS / 32) * RING, bulk_smem = ring_smem + (THREADS / 32) * 8 * 8;
  float* sink;
  cudaMalloc(&sink, 64);
  const size_t table_mb[] = {8, 16, 24, 32, 40, 48, 64, 96, 128, 192};
  for (size_t mb : table_mb) {
    const size_t tb = mb << 20;
    char* X;
    cudaMalloc(&X, tb);
    cudaMemset(X, 0, tb);
    run("lane_cp_async", gather_lane_cp_async<128>, ring_smem, X, tb, 128, n_sm, sink);
    run("lane_cp_async", gather_lane_cp_async<256>, ring_smem, X, tb, 256, n_sm, sink);
    run("lane_cp_async", gather_lane_cp_async<1024>, ring_smem, X, tb, 1024, n_sm, sink);
    run("lane_ldg", gather_lane_ldg<128>, 0, X, tb, 128, n_sm, sink);
    run("lane_ldg", gather_lane_ldg<256>, 0, X, tb, 256, n_sm, sink);
    run("lane_ldg", gather_lane_ldg<1024>, 0, X, tb, 1024, n_sm, sink);
    cudaFree(X);
  }
  for (size_t mb : {(size_t)8, (size_t)173}) {      // today's K=256 data path: 1 KB rows of the 173 MB ARXIV-shape operand
    const size_t tb = mb << 20;
    char* X;
    cudaMalloc(&X, tb);
    cudaMemset(X, 0, tb);
    run("bulk", gather_bulk<1024, 4>, bulk_smem, X, tb, 1024, n_sm, sink);
    cudaFree(X);
  }
  return 0;
}
