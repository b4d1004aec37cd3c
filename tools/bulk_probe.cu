// Micro-probe for the SpMM data path: random row gathers with cp.async.bulk (UBLKCP) into per-warp shared-memory rings,
// completion on mbarriers, rows summed from shared memory (what the aggregation kernel does, without the CSR walk).
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/bulk_probe.cu -o /tmp/bulk_probe && /tmp/bulk_probe
// Sweeps table size (L2-resident .. DRAM), row bytes (256 / 512 / 1024), ring bytes per warp and CTAs per SM.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
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

// RB = row bytes, RING = ring bytes per warp, G = rows per barrier group
template <int RB, int RING, int G>
__global__ void __launch_bounds__(256) bulk_gather(const char* __restrict__ X, const int* __restrict__ idx, int n_idx,
                                                   float4* __restrict__ sink) {
  constexpr int D = RING / RB, NG = D / G, VPL = RB / 512 > 0 ? RB / 512 : 1;  // float4 per lane per row
  constexpr int LANES = RB >= 512 ? 32 : RB / 16;
  extern __shared__ __align__(128) char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  char* ring = smem + (size_t)warp * RING;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)(blockDim.x >> 5) * RING) + warp * NG;
  if (lane < NG) mbar_init(bars + lane, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncwarp();

  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const int per = (n_idx + nw - 1) / nw / 32 * 32;
  const int lo = min(n_idx, gw * per), hi = min(n_idx, lo + per);
  const int n = hi - lo;
  float4 acc = make_float4(0, 0, 0, 0);
  uint32_t phases = 0;
  int cI = 0;
  auto issue = [&](int jg, int slot0, int b) {
    if (jg >= n) return;
    if ((jg & 31) == 0) cI = lo + jg + lane < hi ? __ldg(idx + lo + jg + lane) : 0;
    const int cnt = min(G, n - jg);
    if (lane == 0) mbar_expect_tx(bars + b, cnt * RB);
    const int u = lane - (jg & 31);
    if (u >= 0 && u < cnt) bulk_g2s(ring + (slot0 + u) * RB, X + (size_t)cI * RB, RB, bars + b);
  };
#pragma unroll
  for (int g = 0; g < NG; ++g) issue(g * G, g * G, g);
  int b = 0;
  for (int j = 0, s0 = 0; j < n; j += G) {
    mbar_wait(bars + b, (phases >> b) & 1);
    phases ^= 1u << b;
    const int cnt = min(G, n - j);
    for (int u = 0; u < cnt; ++u) {
      if (lane < LANES) {
#pragma unroll
        for (int v = 0; v < VPL; ++v) {
          const float4 x = *reinterpret_cast<const float4*>(ring + (s0 + u) * RB + (v * 32 + lane) * 16);
          acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
        }
      }
    }
    __syncwarp();
    issue(j + D, s0, b);
    s0 = (s0 + G) & (D - 1);
    b = b + 1 == NG ? 0 : b + 1;
  }
  if (acc.x == 123.456f) sink[0] = acc;
}

static uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s; }

template <int RB, int RING, int G>
static void run(const char* X, size_t tb, const int* d_idx, int n_idx, float4* sink, int ctas_per_sm) {
  const int smem = 8 * RING + 8 * (RING / RB / G) * 8;
  cudaFuncSetAttribute(bulk_gather<RB, RING, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  bulk_gather<RB, RING, G><<<132 * ctas_per_sm, 256, smem>>>(X, d_idx, n_idx, sink);
  cudaEventRecord(a);
  for (int it = 0; it < 5; ++it) bulk_gather<RB, RING, G><<<132 * ctas_per_sm, 256, smem>>>(X, d_idx, n_idx, sink);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
  cudaError_t e = cudaGetLastError();
  printf("{\"probe\":\"bulk_gather\",\"table_MB\":%zu,\"row_bytes\":%d,\"ring_bytes\":%d,\"group\":%d,\"ctas_per_sm\":%d,"
         "\"GBps\":%.1f,\"err\":\"%s\"}\n", tb >> 20, RB, RING, G, ctas_per_sm, (double)n_idx * RB / ms / 1e6,
         e == cudaSuccess ? "" : cudaGetErrorString(e));
  fflush(stdout);
}

int main() {
  const size_t table_mb[] = {43, 87, 173, 1024};
  float4* sink; cudaMalloc(&sink, 64);
  const int n_idx = 4 << 20;
  int* h = new int[n_idx];
  int* d; cudaMalloc(&d, n_idx * 4);
  for (size_t mb : table_mb) {
    const size_t tb = mb << 20;
    char* X; cudaMalloc(&X, tb); cudaMemset(X, 0, tb);
    for (int rb : {256, 512, 1024}) {
      uint32_t s = 12345;
      const int n_rows = (int)(tb / rb);
      for (int i = 0; i < n_idx; ++i) h[i] = lcg(s) % n_rows;
      cudaMemcpy(d, h, n_idx * 4, cudaMemcpyHostToDevice);
      for (int cps : {2, 3}) {
        if (rb == 256) { run<256, 8192, 4>(X, tb, d, n_idx, sink, cps); run<256, 4096, 4>(X, tb, d, n_idx, sink, cps); }
        if (rb == 512) { run<512, 8192, 4>(X, tb, d, n_idx, sink, cps); run<512, 8192, 2>(X, tb, d, n_idx, sink, cps);
                         run<512, 4096, 2>(X, tb, d, n_idx, sink, cps); }
        if (rb == 1024) { run<1024, 8192, 2>(X, tb, d, n_idx, sink, cps); run<1024, 8192, 4>(X, tb, d, n_idx, sink, cps);
                          run<1024, 16384, 4>(X, tb, d, n_idx, sink, cps > 2 ? 2 : cps); }
      }
    }
    cudaFree(X);
  }
  return 0;
}
