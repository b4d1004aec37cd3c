// Philox4x32-10 counter-based generator (Salmon et al., SC'11), written out so the dropout mask of a
// training step is a pure function of (seed, step offset, element index) and can be replayed for parity.
#pragma once
#include <stdint.h>

namespace b200gnn {

__host__ __device__ __forceinline__ uint4 philox4x32(uint64_t seed, uint64_t offset, uint64_t index) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
  uint32_t c0 = (uint32_t)index, c1 = (uint32_t)(index >> 32), c2 = (uint32_t)offset, c3 = (uint32_t)(offset >> 32);
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  uint4 out; out.x = c0; out.y = c1; out.z = c2; out.w = c3;
  return out;
}

// uniform in [0,1) with 24 bits (exactly representable in fp32)
__host__ __device__ __forceinline__ float u32_to_unit(uint32_t x) { return (float)(x >> 8) * (1.0f / 16777216.0f); }

// The dropout keep decisions of four consecutive elements (one float4):
//   keep16: p * 65536 integral (dropout_p16), two 16-bit uniforms of a Philox word each, keep iff u16 >= p * 65536 — exact;
//   keep24: otherwise, four 24-bit uniforms of one Philox block, keep iff u >= p.
__device__ __forceinline__ uchar4 keep16(uint32_t a, uint32_t b, uint32_t thr) {
  uchar4 m;
  m.x = (a & 0xffffu) >= thr; m.y = (a >> 16) >= thr; m.z = (b & 0xffffu) >= thr; m.w = (b >> 16) >= thr;
  return m;
}
__device__ __forceinline__ uchar4 keep24(const uint4& r, float p) {
  uchar4 m;
  m.x = u32_to_unit(r.x) >= p; m.y = u32_to_unit(r.y) >= p; m.z = u32_to_unit(r.z) >= p; m.w = u32_to_unit(r.w) >= p;
  return m;
}

// p * 65536 integral (and p > 0): the 16-bit decision path is exact
static inline bool dropout_p16(float p, uint32_t& thr16) {
  const double t = (double)p * 65536.0;
  thr16 = (uint32_t)t;
  return p > 0.f && t == (double)thr16;
}

}  // namespace b200gnn
