// Micro-probe: how fast can the 132 SMs of an H100 gather random, L2-resident 1 KB rows (the SpMM access pattern)?
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/l2_probe.cu -o /tmp/l2_probe && /tmp/l2_probe
// Prints GB/s for a table that fits L2 (64 MB), one that does not (1 GB), and a plain streaming read.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

__global__ void gather_rows(const float4* __restrict__ X, const int* __restrict__ idx, int n_idx, int vec_per_row,
                            float4* __restrict__ sink) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  float4 acc = make_float4(0, 0, 0, 0);
  for (int base = warp * 32; base < n_idx; base += nwarps * 32) {
    int my = base + lane < n_idx ? idx[base + lane] : 0;
#pragma unroll 4
    for (int t = 0; t < 32; ++t) {
      const int r = __shfl_sync(0xffffffffu, my, t);
      for (int j = lane; j < vec_per_row; j += 32) {
        const float4 v = __ldg(X + (size_t)r * vec_per_row + j);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
  }
  if (acc.x == 123.456f) sink[0] = acc;
}

__global__ void stream_read(const float4* __restrict__ X, size_t n, float4* sink) {
  float4 acc = make_float4(0, 0, 0, 0);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(X + i);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  if (acc.x == 123.456f) sink[0] = acc;
}

static uint32_t lcg(uint32_t& s) { s = s * 1664525u + 1013904223u; return s; }

int main() {
  const int row_bytes_list[] = {1024, 512, 160};
  const size_t table_bytes_list[] = {(size_t)64 << 20, (size_t)1 << 30};
  float4* sink; cudaMalloc(&sink, 64);
  for (size_t tb : table_bytes_list) {
    float4* X; cudaMalloc(&X, tb); cudaMemset(X, 0, tb);
    for (int rb : row_bytes_list) {
      const int vec = rb / 16;
      const int n_rows = (int)(tb / rb);
      const int n_idx = 4 << 20;
      int* h = new int[n_idx]; uint32_t s = 12345;
      for (int i = 0; i < n_idx; ++i) h[i] = lcg(s) % n_rows;
      int* d; cudaMalloc(&d, n_idx * 4); cudaMemcpy(d, h, n_idx * 4, cudaMemcpyHostToDevice);
      for (int blocks_per_sm : {4, 8}) {
        cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
        gather_rows<<<132 * blocks_per_sm, 256>>>(X, d, n_idx, vec, sink);
        cudaEventRecord(a);
        for (int it = 0; it < 5; ++it) gather_rows<<<132 * blocks_per_sm, 256>>>(X, d, n_idx, vec, sink);
        cudaEventRecord(b); cudaEventSynchronize(b);
        float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
        printf("{\"probe\":\"gather\",\"table_MB\":%zu,\"row_bytes\":%d,\"ctas_per_sm\":%d,\"GBps\":%.1f}\n", tb >> 20, rb,
               blocks_per_sm, (double)n_idx * rb / ms / 1e6);
      }
      cudaFree(d); delete[] h;
    }
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    stream_read<<<132 * 8, 256>>>(X, tb / 16, sink);
    cudaEventRecord(a);
    for (int it = 0; it < 5; ++it) stream_read<<<132 * 8, 256>>>(X, tb / 16, sink);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b); ms /= 5;
    printf("{\"probe\":\"stream\",\"table_MB\":%zu,\"GBps\":%.1f}\n", tb >> 20, (double)tb / ms / 1e6);
    cudaFree(X);
  }
  return 0;
}
