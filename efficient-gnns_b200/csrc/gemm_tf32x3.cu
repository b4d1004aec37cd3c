// fp32-faithful dense GEMM on the Hopper tensor cores (wgmma / TMA / mbarrier), sm_90a.
//
//   C[M,N] = A[M,K] · B[N,K]^T (+ bias[N])          all fp32 in HBM, fp32 accumulation in registers
//
// The reference computes its dense contractions (GCNConv's X·W, nn.Linear, the backward dX = dY·W^T;
// arxiv_pyg/gnn.py:47,52 via PyG) in fp32 and the parity bar is 1e-5, which a single TF32 pass (10-bit
// mantissa) cannot meet.  So every product is evaluated with the 3xTF32 split
//        a·b ≈ a_hi·b_hi + a_lo·b_hi + a_hi·b_lo ,   x_hi = x rounded to tf32 (cvt.rna),
//                                                    x_lo = (x - x_hi) rounded to tf32,
// three wgmma.mma_async ... .tf32 instructions per K-step.  The dropped terms are O(2^-22) relative.  B (the small
// weight matrix) arrives pre-split from b200gnn_split_tf32_f32; A (the big activation matrix) is split on the fly in
// registers, so HBM only ever sees one fp32 copy of it.
//
// Structure (one persistent CTA per SM, 384 threads = 3 warpgroups):
//   warpgroup 0     TMA producer: one thread, cp.async.bulk.tensor 128x32 fp32 boxes (128B swizzle) of A, B_hi, B_lo
//   warpgroups 1-2  consumers, 64 rows of the 128-row tile each: every thread loads its wgmma A fragment of the stage
//                   from the A tile and splits it into (hi, lo) registers while the previous stage's wgmmas run, issues
//                   12 wgmmas per stage (A from registers, B from shared memory), then the epilogue.  A_hi / A_lo never
//                   go through shared memory, which keeps a stage's shared-memory traffic (TMA writes, the fragment
//                   loads, the B reads of the wgmmas) under its tensor-core time.
// Accumulation: the tensor core's fp32 accumulate truncates instead of rounding to nearest (tools/probe_accum.py), and its
// error grows with the number of updates of one accumulator.  Each stage's 12 wgmmas therefore go to a fresh register accumulator that is
// then added (fp32, round to nearest) into the tile's running sum: no tensor-core chain is longer than one stage.
#include <cuda.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace b200gnn {
namespace gemm {
using namespace tc;

constexpr int BM = 128, BK = 32;
constexpr int THREADS = 384;
constexpr int CONSUMER_WARPS = 8;                       // warp q owns rows [16 q, 16 q + 16) of the tile
constexpr int TILE_BYTES = BM * BK * 4;                 // 16 KB: one 128 x 32 fp32 A tile
constexpr int BAR_BYTES = 256;
constexpr int EPI_BYTES = CONSUMER_WARPS * 16 * 32 * 4; // one 16x32 staging block per consumer warp (16-byte chunks swizzled)
constexpr int STAT_MAX_N = 256;                         // fused column statistics: output width limit
constexpr int STAT_BYTES = CONSUMER_WARPS * 2 * STAT_MAX_N * 4;  // per consumer warp: [2][STAT_MAX_N] column accumulators
constexpr int XY_ROWS = 16;
constexpr int XY_SLOT_BYTES = 2 * XY_ROWS * 32 * 4;     // one 16x32 fp32 block of Xout + the same block of Y
constexpr int XY_BYTES = CONSUMER_WARPS * 2 * XY_SLOT_BYTES;  // 8 consumer warps x 2 slots (stat_mode 2 with TMA-staged operands)
constexpr int XY_BAR_OFF = 128;                         // byte offset of the 16 Xout/Y mbarriers inside the barrier block
// BatchNorm-backward epilogue: the TMA-staged Xout / Y path pays for its 64 KB with two of the four mainloop stages, which
// only narrow-K launches (epilogue-bound) win back; measured on H100 (BENCH.md): K=40 TMA ahead, K=256 the register path ahead.
constexpr int BNBWD_TMA_MAX_K = 128;

// Tile shape: BN_T output columns per tile (the wgmma N) and the number of smem stages that fit.
//   Wide  <128, 4>: 4 x 48 KB stages.
//   Narrow <48, 6>: for N <= 48 (the 40-class logits): the B tiles shrink to 6 KB, two more stages fit (the narrow
//                   GEMM is bound by the DRAM latency of A, so depth is what it needs) and the MMAs do 3/8 of the work.
//   BatchNorm-backward with TMA-staged Xout / Y <128, 2, XY_BYTES>: the 64 KB of Xout / Y leave room for 2 stages.
template <int BN_T, int NSTAGE, int EXTRA = 0>
struct Cfg {
  static constexpr int BN = BN_T, STAGES = NSTAGE;
  static constexpr int B_TILE_BYTES = BN_T * BK * 4;
  static constexpr int STAGE_BYTES = TILE_BYTES + 2 * B_TILE_BYTES;              // A, B_hi, B_lo
  static constexpr int ACC = BN_T / 2;                                            // accumulator registers per thread
  static constexpr int SMEM_BYTES = NSTAGE * STAGE_BYTES + BAR_BYTES + EPI_BYTES + STAT_BYTES + EXTRA + 1024;  // + alignment slack
  static_assert(B_TILE_BYTES % 1024 == 0 && (BN_T == 128 || BN_T == 48), "tile shape (wgmma wrappers: N = 128, 48)");
  static_assert(2 * NSTAGE * 8 <= XY_BAR_OFF, "barrier block");
  static_assert(SMEM_BYTES <= 232448, "shared memory");
};

__device__ __forceinline__ void mma(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_tf32_n128_rs(d, a, b, s); }
__device__ __forceinline__ void mma(float (&d)[24], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_tf32_n48_rs(d, a, b, s); }

// This thread's wgmma A fragments of one stage: v[k][i] = row r0 + 8 (i % 2), column 8 k + lane % 4 + 4 (i / 2) of the
// 128B-swizzled [128][32] A tile, r0 = 16 (consumer warp) + lane / 4.  The rows of one load differ in r0 % 8 = lane / 4,
// so the swizzle puts the 8 row groups in 8 different 16-byte chunks: 32 banks.  `frag` = a_frag_offset(...) + the
// tile's shared address (1024-byte aligned), so the swizzled chunk is one XOR away.
__device__ __forceinline__ uint32_t a_frag_offset(int r0, int lane) { return r0 * 128 + ((lane >> 2) << 4) + (lane & 3) * 4; }
__device__ __forceinline__ void load_a(uint32_t frag, uint32_t (&v)[BK / 8][4]) {
  asm("" : "+r"(frag));   // opaque: one XOR per load instead of 8 swizzled offsets held in registers across the epilogue
#pragma unroll
  for (int k = 0; k < BK / 8; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) v[k][i] = lds32((frag ^ ((2 * k + (i >> 1)) << 4)) + (i & 1) * 8 * 128);
}

// float index of 16-byte chunk c4 (0..7) of row r in a warp's [16][32] staging block
__device__ __forceinline__ int stg(int r, int c4) { return r * 32 + ((c4 ^ (r & 7)) << 2); }

struct Params {
  float* C;
  const float* bias;
  int64_t ldc;
  int32_t M, N, K;
  int32_t accumulate;   // C += A·B^T (+bias) instead of C = ...
  // Fused R->C layout exchange of the multi-GPU engine (hybrid.py): output columns [q*kc, (q+1)*kc) go to rank q's
  // [N, kc] buffer Cp[q] at rows row_off + m — the epilogue stores straight into the consumers' memory over NVLink
  // (peer mappings), so the exchange costs no kernel of its own and overlaps the GEMM tile by tile.  n_peer = 0: off.
  float* Cp[16];
  int32_t n_peer, kc;
  int64_t row_off;
  int32_t bcast;        // 1: every Cp[q] receives ALL columns at rows row_off + m (fused all-gather of a narrow result)
  // Fused row passes (§8 f1): column reductions over the rows of the OUTPUT, taken in the epilogue while the tile is in
  // registers, so the separate full sweeps over C disappear.  Each consumer warp keeps [2][N] running column sums in shared
  // memory over all tiles of its CTA and stores them once to stat_partial[(cta*8 + warp)][2][N] (fixed order: deterministic).
  //   stat_mode 1: (sum c, sum c^2) — the BatchNorm batch statistics of the layer output (forward);
  //   stat_mode 2: C is dOut of BN->ReLU->dropout (arxiv_pyg/gnn.py:48-50): the epilogue forms
  //                dz = dOut * [Xout > 0] / (1-p), STORES dz in place of dOut and reduces (sum dz, sum dz*xhat),
  //                xhat = (Y - mean) * invstd — pass 1 of the BatchNorm backward.
  int32_t stat_mode;
  float* stat_partial;
  const float* bn_x;    // Xout [M, ldc]  (post-dropout activation: > 0 <=> ReLU-active and kept)
  const float* bn_y;    // Y    [M, ldc]  (BatchNorm input)
  const float* bn_mean;
  const float* bn_invstd;
  float inv_keep;
  // ACT: the activation A = dropout(relu(Y * scale + shift)) of a hidden layer is recomputed from Y, the per-column
  // scale / shift of its BatchNorm and the packed keep bits (uint32 [rows][act_words], bit c % 32 of word c / 32 is the
  // dropout decision of column c) instead of being read:
  //   stat_mode 0: the A operand is Y, and every A fragment element becomes bit ? max(y * scale + shift, 0) * inv_keep : 0
  //                before its tf32 split (the same operations as b200gnn_affine_relu_dropout_f32, so the product is that of
  //                the materialised activation bit for bit);
  //   stat_mode 2: the mask [Xout > 0] of the BatchNorm-backward epilogue becomes bit && y * scale + shift > 0 (bn_x unused).
  const float* act_scale;
  const float* act_shift;
  const uint32_t* act_bits;
  int32_t act_words;
  // PRELU (SIGN's FeedForwardNet): A = dropout(prelu(Z)) with one learnable slope read from device memory, so no per-column
  // table and no limit on K:
  //   stat_mode 0: every A fragment element z becomes bit ? (z > 0 ? z : slope * z) * inv_keep : 0 before its tf32 split;
  //   stat_mode 4: C is dA, the gradient of that activation over N columns (Z = bn_y, pitch ldc, bits [M][act_words]): the
  //                epilogue STORES dz = (bit ? dA * inv_keep : 0) * (z > 0 ? 1 : slope) and reduces the slope gradient
  //                sum (bit ? dA * inv_keep : 0) * z over z <= 0 in fp64 into slope_partial[cta * 8 + warp] (fixed order).
  const float* act_slope;
  double* slope_partial;
};

// stat_mode 2: the pieces of Xout / Y one lane needs for a 32-column chunk (4 rows x 4 columns: rows it*4 + lane/8
// of the warp's 16 rows, columns 4*(lane%8)...) — the same row segments its stores cover.
template <bool ACT>
__device__ __forceinline__ void load_bn_chunk(const Params& p, int m0, int col, int q, int lane, float4 (&x)[4], float4 (&y)[4]) {
  if (col + 32 > p.N) return;
  const int sub = lane >> 3, cq = (lane & 7) * 4;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int grow = m0 + q * 16 + it * 4 + sub;
    if (grow < p.M) {
      const size_t o = (size_t)grow * p.ldc + col + cq;
      if (!ACT) x[it] = __ldg(reinterpret_cast<const float4*>(p.bn_x + o));
      y[it] = __ldg(reinterpret_cast<const float4*>(p.bn_y + o));
    }
  }
}

// ACT with stat_mode 2: this lane's keep words of a 32-column chunk (one word: chunks are 32-column aligned), rows as above
__device__ __forceinline__ void load_bits_chunk(const Params& p, int m0, int col, int q, int lane, uint32_t (&w)[4]) {
  const int sub = lane >> 3;
#pragma unroll
  for (int it = 0; it < 4; ++it) {
    const int grow = m0 + q * 16 + it * 4 + sub;
    w[it] = grow < p.M ? __ldg(p.act_bits + (size_t)grow * p.act_words + (col >> 5)) : 0u;
  }
}

// ACT with stat_mode 0: the activation of one A element from y, its column's (scale, shift) and its keep bit
__device__ __forceinline__ uint32_t act1(uint32_t y, float sc, float sh, uint32_t keep, float inv_keep) {
  return keep ? __float_as_uint(fmaxf(fmaf(__uint_as_float(y), sc, sh), 0.f) * inv_keep) : 0u;
}

// PReLU + dropout of one A element z (SIGN): the same operations as b200gnn_prelu_bits_f32
__device__ __forceinline__ uint32_t prelu1(uint32_t z, float slope, uint32_t keep, float inv_keep) {
  const float x = __uint_as_float(z);
  return keep ? __float_as_uint((x > 0.f ? x : slope * x) * inv_keep) : 0u;
}

// STAT: 0 plain, 1 / 2 the fused column reductions (Params::stat_mode), 4 the PReLU/dropout backward; PEER: the output goes
// to peer buffers (Params::Cp); ACT: the hidden activation is recomputed from Y (Params::act_bits); PRELU: the PReLU/dropout
// prologue.  Compile-time so that each instantiation carries only its own prologue and epilogue (the epilogue is the hot loop
// of the narrow-K GEMMs).
template <class C, int STAT, bool PEER, bool ACT = false, bool PRELU = false>
__global__ void __launch_bounds__(THREADS, 1)
gemm_tf32x3_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
                   const __grid_constant__ CUtensorMap tmBlo, const __grid_constant__ CUtensorMap tmX,
                   const __grid_constant__ CUtensorMap tmY, const Params p) {
  constexpr bool BNB = STAT == 2 || STAT == 3;   // BatchNorm-backward epilogue; STAT == 3: its Xout / Y blocks arrive by TMA
  constexpr bool XYTMA = STAT == 3;
  constexpr bool COLSTAT = STAT >= 1 && STAT <= 3;   // per-column reductions in the statistics block
  constexpr bool PRB = STAT == 4;                    // PReLU/dropout backward epilogue
  constexpr bool PRO = (ACT || PRELU) && !STAT;      // activation prologue on A (keep words fetched a stage ahead)
  constexpr int BN = C::BN, STAGES = C::STAGES, STAGE_BYTES = C::STAGE_BYTES, B_TILE_BYTES = C::B_TILE_BYTES, ACC = C::ACC;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full = bars;                      // TMA landed                              [STAGES]
  uint64_t* empty = bars + STAGES;            // both consumer warpgroups done with it   [STAGES]
  float* epi_smem = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + BAR_BYTES);
  float* stat_smem = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES + BAR_BYTES + EPI_BYTES);
  uint8_t* xy_smem = smem + STAGES * STAGE_BYTES + BAR_BYTES + EPI_BYTES + STAT_BYTES;
  uint64_t* xy_full = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES + XY_BAR_OFF);   // [8 warps][2 slots]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    if (XYTMA)
      for (int i = 0; i < 2 * CONSUMER_WARPS; ++i) mbar_init(&xy_full[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int num_m = (p.M + BM - 1) / BM, num_n = (p.N + BN - 1) / BN;
  const int num_tiles = num_m * num_n;
  const int num_kb = (p.K + BK - 1) / BK;

  if (warp < 4) {
    // ------------------------------------------------------------------ TMA producer
    regs_dec<40>();
    if (threadIdx.x == 0) {
      int s = 0; uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&empty[s], ph ^ 1);
          uint8_t* st = smem + s * STAGE_BYTES;
          mbar_expect_tx(&full[s], TILE_BYTES + 2 * B_TILE_BYTES);
          tma_load_2d(&tmA, &full[s], st, kb * BK, m0);
          tma_load_2d(&tmBhi, &full[s], st + TILE_BYTES, kb * BK, n0);
          tma_load_2d(&tmBlo, &full[s], st + TILE_BYTES + B_TILE_BYTES, kb * BK, n0);
          if (++s == STAGES) { s = 0; ph ^= 1; }
        }
      }
    }
    return;
  }
  regs_inc<232>();

  // -------------------------------------------------------------------- consumers
  const int q = warp - 4;                         // consumer warp: rows [16 q, 16 q + 16)
  const bool vec_ok = PEER ? true : ((p.ldc % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.C) & 15) == 0));
  float* stat = stat_smem + q * (2 * STAT_MAX_N);  // this warp's [2][N] column accumulators
  if (COLSTAT) {
    for (int i = lane; i < 2 * p.N; i += 32) stat[i] = 0.f;
    __syncwarp();
  }
  constexpr int NCHUNK = (BN + 31) / 32;
  // stat_mode 2 reads Xout and Y next to every output element; neither depends on the accumulator.
  //   STAT == 2: register path — the lane's pieces of a chunk are requested at the top of the chunk;
  //   STAT == 3: (N % 128 == 0) each warp keeps TWO chunks of Xout / Y in flight in shared memory through TMA
  //              ({32 x 16} boxes, one mbarrier per slot, refilled by lane 0 as soon as the chunk has been consumed):
  //              twice the bytes in flight and no register cost.
  uint8_t* xy = xy_smem + q * (2 * XY_SLOT_BYTES);
  uint64_t* xyb = xy_full + q * 2;
  int n_mine = 0;                                  // chunks this CTA will process (XYTMA: all chunks are whole)
  if (XYTMA) {
    for (int tt = blockIdx.x; tt < num_tiles; tt += gridDim.x) n_mine += NCHUNK;
    if (lane == 0)
      for (int g = 0; g < 2 && g < n_mine; ++g) {
        const int tt = blockIdx.x + (g / NCHUNK) * gridDim.x, cc = g % NCHUNK;
        mbar_expect_tx(&xyb[g], ACT ? XY_SLOT_BYTES / 2 : XY_SLOT_BYTES);
        if (!ACT)
          tma_load_2d(&tmX, &xyb[g], xy + g * XY_SLOT_BYTES, (tt % num_n) * BN + cc * 32, (tt / num_n) * BM + q * XY_ROWS);
        tma_load_2d(&tmY, &xyb[g], xy + g * XY_SLOT_BYTES + XY_SLOT_BYTES / 2, (tt % num_n) * BN + cc * 32,
                    (tt / num_n) * BM + q * XY_ROWS);
      }
  }
  // ACT prologue: the (scale, shift) pairs of all K columns sit in the (otherwise unused) statistics block, ordered so that a
  // thread's 8 columns of a stage, 8 k + lane % 4 + 4 j, are 4 consecutive float4 {sc(k,0), sh(k,0), sc(k,1), sh(k,1)}
  const float* act_ss = stat_smem;
  if (ACT && !STAT) {
    for (int c = threadIdx.x - 128; c < num_kb * BK; c += 256) {
      const int w = c & 31;
      const float2 v = c < p.K ? make_float2(__ldg(p.act_scale + c), __ldg(p.act_shift + c)) : make_float2(0.f, 0.f);
      *reinterpret_cast<float2*>(stat_smem + (c >> 5) * 64 + (w & 3) * 16 + (w >> 3) * 4 + ((w >> 2) & 1) * 2) = v;
    }
    named_sync(1, 256);
  }
  // keep words of this thread's two A rows (r0, r0 + 8) for the next stage: fetched one stage ahead
  const int arow = q * 16 + (lane >> 2);
  auto act_words = [&](int tile, int kb, uint32_t (&w)[2]) {
    const int r = (tile / num_n) * BM + arow;
    w[0] = r < p.M ? __ldg(p.act_bits + (size_t)r * p.act_words + kb) : 0u;
    w[1] = r + 8 < p.M ? __ldg(p.act_bits + (size_t)(r + 8) * p.act_words + kb) : 0u;
  };
  uint32_t wnext[2] = {0u, 0u};
  if (PRO && blockIdx.x < num_tiles) act_words(blockIdx.x, 0, wnext);
  const float slope = (PRELU || PRB) ? __ldg(p.act_slope) : 0.f;
  double sg = 0.0;                                 // PRB: this lane's share of the slope gradient
  float acc[ACC], sum[ACC];
  // A fragments (hi, lo) of two consecutive stages: stage kb's are written while the wgmmas of stage kb - 1, which read
  // the other set, are in flight
  uint32_t ah0[BK / 8][4], al0[BK / 8][4], ah1[BK / 8][4], al1[BK / 8][4];
  const uint32_t frag = a_frag_offset(q * 16 + (lane >> 2), lane);
  int s = 0; uint32_t ph = 0;
  int g_chunk = 0;                                 // running chunk index of this warp (XYTMA slot = g & 1, phase = (g >> 1) & 1)
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int m0 = (tile / num_n) * BM, n0 = (tile % num_n) * BN;
#pragma unroll
    for (int i = 0; i < ACC; ++i) sum[i] = acc[i] = 0.f;   // acc: not live across the previous tile's epilogue
    int prev = 0;
    auto stage = [&](int kb, uint32_t (&h)[BK / 8][4], uint32_t (&l)[BK / 8][4]) {
      uint32_t wcur[2];
      if (PRO) {
        wcur[0] = wnext[0] >> (lane & 3); wcur[1] = wnext[1] >> (lane & 3);
        if (kb + 1 < num_kb) act_words(tile, kb + 1, wnext);
        else if (tile + (int)gridDim.x < num_tiles) act_words(tile + gridDim.x, 0, wnext);
      }
      mbar_wait(&full[s], ph);
      uint8_t* st = smem + s * STAGE_BYTES;
      load_a(smem_u32(st) + frag, h);
      if (ACT && !STAT) {
        const float4* ss = reinterpret_cast<const float4*>(act_ss + kb * 64 + (lane & 3) * 16);
#pragma unroll
        for (int k = 0; k < BK / 8; ++k) {
          const float4 t = ss[k];
#pragma unroll
          for (int i = 0; i < 4; ++i)   // element i: row r0 + 8 (i % 2), column 8 k + lane % 4 + 4 (i / 2)
            h[k][i] = act1(h[k][i], (i >> 1) ? t.z : t.x, (i >> 1) ? t.w : t.y, (wcur[i & 1] >> (8 * k + 4 * (i >> 1))) & 1u,
                           p.inv_keep);
        }
      }
      if (PRELU && !STAT) {
#pragma unroll
        for (int k = 0; k < BK / 8; ++k)
#pragma unroll
          for (int i = 0; i < 4; ++i)   // element i: row r0 + 8 (i % 2), column 8 k + lane % 4 + 4 (i / 2)
            h[k][i] = prelu1(h[k][i], slope, (wcur[i & 1] >> (8 * k + 4 * (i >> 1))) & 1u, p.inv_keep);
      }
#pragma unroll
      for (int k = 0; k < BK / 8; ++k)
#pragma unroll
        for (int i = 0; i < 4; ++i) split1(h[k][i], h[k][i], l[k][i]);
      reg_fence(h); reg_fence(l);                  // split before the wait: it overlaps the previous stage's wgmmas
      if (kb > 0) {                                // the previous stage's wgmmas have retired: promote, free its stage
        wgmma_wait<0>();
        acc_fence(acc);
#pragma unroll
        for (int i = 0; i < ACC; ++i) sum[i] += acc[i];
        mbar_arrive(&empty[prev]);
      }
      wgmma_fence();
      const uint32_t sb = smem_u32(st + TILE_BYTES);
      // all 8 small correction terms of the stage first, then the 4 large ones: the accumulator is large (and its
      // truncating accumulate costs the most) for 4 of the 12 updates only
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) {
        const uint32_t koff = k * 32;              // 32 B per K-step inside the 128 B swizzle row
        mma(acc, l[k], make_desc_k128(sb + koff), k != 0);
        mma(acc, h[k], make_desc_k128(sb + B_TILE_BYTES + koff), 1);
      }
#pragma unroll
      for (int k = 0; k < BK / 8; ++k) mma(acc, h[k], make_desc_k128(sb + k * 32), 1);
      wgmma_commit();
      prev = s;
      if (++s == STAGES) { s = 0; ph ^= 1; }
    };
    for (int kb = 0; kb < num_kb; kb += 2) {
      stage(kb, ah0, al0);
      if (kb + 1 < num_kb) stage(kb + 1, ah1, al1);
    }
    wgmma_wait<0>();
    acc_fence(acc);
#pragma unroll
    for (int i = 0; i < ACC; ++i) sum[i] += acc[i];
    mbar_arrive(&empty[prev]);

    // ------------------------------------------------------------------ epilogue of rows [m0 + 16 q, m0 + 16 q + 16)
    float* tile_s = epi_smem + q * (16 * 32);
#pragma unroll
    for (int c = 0; c < NCHUNK; ++c, ++g_chunk) {
      const int col0 = n0 + c * 32;
      float4 xr[4], yr[4];
      if (STAT == 2) load_bn_chunk<ACT>(p, m0, col0, q, lane, xr, yr);
      if (PRB) load_bn_chunk<true>(p, m0, col0, q, lane, xr, yr);   // Z only
      // accumulator fragment -> staging block, so that global stores are whole 128-byte row segments
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = c * 4 + jj;
        if (j * 8 < BN) {
          const int r0 = lane >> 2, cc = jj * 8 + 2 * (lane & 3);
          *reinterpret_cast<float2*>(tile_s + stg(r0, cc >> 2) + (cc & 3)) = make_float2(sum[4 * j], sum[4 * j + 1]);
          *reinterpret_cast<float2*>(tile_s + stg(r0 + 8, cc >> 2) + (cc & 3)) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
        }
      }
      __syncwarp();
      if (vec_ok && col0 + 32 <= p.N) {
        const float* xs = reinterpret_cast<const float*>(xy + (g_chunk & 1) * XY_SLOT_BYTES);   // [16 rows][32 floats]
        const float* ys = xs + XY_ROWS * 32;
        if (XYTMA) mbar_wait(&xyb[g_chunk & 1], (uint32_t)((g_chunk >> 1) & 1));
        const int sub = lane >> 3, cq = (lane & 7) * 4;     // 4 rows per instruction, 8 lanes x float4 per row
        float4 b4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.bias) b4 = make_float4(__ldg(p.bias + col0 + cq), __ldg(p.bias + col0 + cq + 1), __ldg(p.bias + col0 + cq + 2),
                                     __ldg(p.bias + col0 + cq + 3));
        float4 s4 = make_float4(0.f, 0.f, 0.f, 0.f), q4 = s4, mu4 = s4, is4 = s4, sc4 = s4, sh4 = s4;
        if (BNB) {
          mu4 = __ldg(reinterpret_cast<const float4*>(p.bn_mean + col0 + cq));
          is4 = __ldg(reinterpret_cast<const float4*>(p.bn_invstd + col0 + cq));
        }
        uint32_t wb[4];
        if (BNB && ACT) {
          sc4 = __ldg(reinterpret_cast<const float4*>(p.act_scale + col0 + cq));
          sh4 = __ldg(reinterpret_cast<const float4*>(p.act_shift + col0 + cq));
          load_bits_chunk(p, m0, col0, q, lane, wb);
        }
        if (PRB) load_bits_chunk(p, m0, col0, q, lane, wb);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 4 + sub;
          const int grow = m0 + q * 16 + rr;
          float4 v = *reinterpret_cast<const float4*>(tile_s + stg(rr, lane & 7));
          v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
          if (PEER && grow < p.M && p.bcast) {
            for (int r = 0; r < p.n_peer; ++r)
              *reinterpret_cast<float4*>(p.Cp[r] + (size_t)(p.row_off + grow) * p.ldc + col0 + cq) = v;
          } else if (grow < p.M) {
            float4* dst;
            if (PEER) {                           // a 32-column chunk never straddles two ranks (kc % 32 == 0)
              const int r = col0 / p.kc;
              dst = reinterpret_cast<float4*>(p.Cp[r] + (size_t)(p.row_off + grow) * p.kc + (col0 - r * p.kc) + cq);
            } else {
              dst = reinterpret_cast<float4*>(p.C + (size_t)grow * p.ldc + col0 + cq);
            }
            if (!PEER && p.accumulate) { const float4 o = *dst; v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w; }
            if (STAT == 1) {
              vstat(s4, q4, v);
            } else if (BNB) {
              float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
              if (!ACT) x = XYTMA ? *reinterpret_cast<const float4*>(xs + rr * 32 + cq) : xr[it];
              const float4 y = XYTMA ? *reinterpret_cast<const float4*>(ys + rr * 32 + cq) : yr[it];
              if (ACT) {                          // Xout > 0  <=>  kept && y * scale + shift > 0
                const uint32_t b = wb[it] >> cq;
                v.x = (b & 1u) && fmaf(y.x, sc4.x, sh4.x) > 0.f ? v.x * p.inv_keep : 0.f;
                v.y = (b & 2u) && fmaf(y.y, sc4.y, sh4.y) > 0.f ? v.y * p.inv_keep : 0.f;
                v.z = (b & 4u) && fmaf(y.z, sc4.z, sh4.z) > 0.f ? v.z * p.inv_keep : 0.f;
                v.w = (b & 8u) && fmaf(y.w, sc4.w, sh4.w) > 0.f ? v.w * p.inv_keep : 0.f;
              } else {
                v.x = x.x > 0.f ? v.x * p.inv_keep : 0.f; v.y = x.y > 0.f ? v.y * p.inv_keep : 0.f;
                v.z = x.z > 0.f ? v.z * p.inv_keep : 0.f; v.w = x.w > 0.f ? v.w * p.inv_keep : 0.f;
              }
              s4.x += v.x; s4.y += v.y; s4.z += v.z; s4.w += v.w;
              q4.x = fmaf(v.x, (y.x - mu4.x) * is4.x, q4.x); q4.y = fmaf(v.y, (y.y - mu4.y) * is4.y, q4.y);
              q4.z = fmaf(v.z, (y.z - mu4.z) * is4.z, q4.z); q4.w = fmaf(v.w, (y.w - mu4.w) * is4.w, q4.w);
            } else if (PRB) {
              const float4 z = yr[it];
              const uint32_t b = wb[it] >> cq;
              const float gx = (b & 1u) ? v.x * p.inv_keep : 0.f, gy = (b & 2u) ? v.y * p.inv_keep : 0.f;
              const float gz = (b & 4u) ? v.z * p.inv_keep : 0.f, gw = (b & 8u) ? v.w * p.inv_keep : 0.f;
              if (!(z.x > 0.f)) sg += (double)(gx * z.x);
              if (!(z.y > 0.f)) sg += (double)(gy * z.y);
              if (!(z.z > 0.f)) sg += (double)(gz * z.z);
              if (!(z.w > 0.f)) sg += (double)(gw * z.w);
              v.x = z.x > 0.f ? gx : gx * slope; v.y = z.y > 0.f ? gy : gy * slope;
              v.z = z.z > 0.f ? gz : gz * slope; v.w = z.w > 0.f ? gw : gw * slope;
            }
            *dst = v;
          }
        }
        if (COLSTAT) {
          // 4 row sub-groups (lane >> 3) hold the same columns: fold them, lanes 0-7 add into the warp's accumulators
#pragma unroll
          for (int d = 8; d <= 16; d <<= 1) {
            s4.x += __shfl_xor_sync(0xffffffffu, s4.x, d); s4.y += __shfl_xor_sync(0xffffffffu, s4.y, d);
            s4.z += __shfl_xor_sync(0xffffffffu, s4.z, d); s4.w += __shfl_xor_sync(0xffffffffu, s4.w, d);
            q4.x += __shfl_xor_sync(0xffffffffu, q4.x, d); q4.y += __shfl_xor_sync(0xffffffffu, q4.y, d);
            q4.z += __shfl_xor_sync(0xffffffffu, q4.z, d); q4.w += __shfl_xor_sync(0xffffffffu, q4.w, d);
          }
          if (lane < 8) {
            float4* ps = reinterpret_cast<float4*>(stat + col0 + cq);
            float4* pq = reinterpret_cast<float4*>(stat + p.N + col0 + cq);
            float4 a0 = *ps, a1 = *pq;
            a0.x += s4.x; a0.y += s4.y; a0.z += s4.z; a0.w += s4.w;
            a1.x += q4.x; a1.y += q4.y; a1.z += q4.z; a1.w += q4.w;
            *ps = a0; *pq = a1;
          }
        }
        __syncwarp();
        if (XYTMA && lane == 0 && g_chunk + 2 < n_mine) {      // the slot has been read by every lane: refill it
          const int g = g_chunk + 2, tt = blockIdx.x + (g / NCHUNK) * gridDim.x, cc = g % NCHUNK;
          uint8_t* dst = xy + (g & 1) * XY_SLOT_BYTES;
          mbar_expect_tx(&xyb[g & 1], ACT ? XY_SLOT_BYTES / 2 : XY_SLOT_BYTES);
          if (!ACT) tma_load_2d(&tmX, &xyb[g & 1], dst, (tt % num_n) * BN + cc * 32, (tt / num_n) * BM + q * XY_ROWS);
          tma_load_2d(&tmY, &xyb[g & 1], dst + XY_SLOT_BYTES / 2, (tt % num_n) * BN + cc * 32, (tt / num_n) * BM + q * XY_ROWS);
        }
      } else {
        // ragged chunk: lane -> row lane % 16, columns [16 (lane / 16), +16) of the chunk
        const int rr = lane & 15, cb = (lane >> 4) * 16, grow = m0 + q * 16 + rr;
        if (grow < p.M && col0 + cb < p.N) {
          for (int jx = 0; jx < 16; ++jx) {
            const int cc = cb + jx, col = col0 + cc;
            if (col >= p.N) break;
            const float v = tile_s[stg(rr, cc >> 2) + (cc & 3)] + (p.bias ? __ldg(p.bias + col) : 0.f);
            if (PEER && p.bcast) {
              for (int r = 0; r < p.n_peer; ++r) p.Cp[r][(size_t)(p.row_off + grow) * p.ldc + col] = v;
            } else if (!PEER) {
              float* dst = p.C + (size_t)grow * p.ldc + col;
              *dst = v + (p.accumulate ? *dst : 0.f);
            }
          }
        }
        __syncwarp();
      }
    }
  }
  if (COLSTAT) {
    __syncwarp();
    float* out = p.stat_partial + (size_t)(blockIdx.x * CONSUMER_WARPS + q) * 2 * p.N;
    for (int i = lane; i < 2 * p.N; i += 32) out[i] = stat[i];
  }
  if (PRB) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) sg += __shfl_xor_sync(0xffffffffu, sg, d);
    if (lane == 0) p.slope_partial[blockIdx.x * CONSUMER_WARPS + q] = sg;
  }
}

// slope_grad (+)= sum of the PRB partials in slot order (one warp, fixed order: bitwise repeatable)
__global__ void __launch_bounds__(32) slope_grad_finalize_kernel(const double* __restrict__ part, int n, float* __restrict__ out,
                                                                 int accumulate) {
  double a = 0.0;
  for (int i = threadIdx.x; i < n; i += 32) a += part[i];
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d);
  if (threadIdx.x == 0) out[0] = accumulate ? out[0] + (float)a : (float)a;
}

// hi/lo split of a small matrix (weights), optionally transposed: out[c][r] when transpose.
__global__ void __launch_bounds__(256) split_tf32_kernel(const float* __restrict__ W, int64_t rows, int64_t cols,
                                                         int transpose, float* __restrict__ hi, float* __restrict__ lo) {
  const int64_t n = rows * cols;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / cols, c = i - r * cols;
    uint32_t h, l;
    split1(__float_as_uint(W[i]), h, l);
    const int64_t o = transpose ? c * rows + r : i;
    hi[o] = __uint_as_float(h);
    lo[o] = __uint_as_float(l);
  }
}

// [rows, cols] fp32 row-major with leading dimension ld -> boxes of 32 columns x box_rows rows, 128B swizzle, zero OOB fill
static bool make_map(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_rows, bool swizzle = true) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
            CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <class C, int STAT = 0, bool PEER = false, bool ACT = false, bool PRELU = false>
static int launch(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb, const Params& p,
                  cudaStream_t stream) {
  CUtensorMap tA, tBh, tBl, tX, tY;
  if (!make_map(&tA, A, p.M, p.K, lda, BM) || !make_map(&tBh, B_hi, p.N, p.K, ldb, C::BN) ||
      !make_map(&tBl, B_lo, p.N, p.K, ldb, C::BN))
    return B200GNN_ERR_UNSUPPORTED;
  tX = tA; tY = tA;                                  // placeholders unless the epilogue stages Xout / Y through TMA
  if (STAT == 3 && ((!ACT && !make_map(&tX, p.bn_x, p.M, p.N, p.ldc, XY_ROWS, false)) ||
                    !make_map(&tY, p.bn_y, p.M, p.N, p.ldc, XY_ROWS, false)))
    return B200GNN_ERR_UNSUPPORTED;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {};                    // per device and instantiation; idempotent if two threads race
  if (dev >= 0 && dev < 64 && !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(gemm_tf32x3_kernel<C, STAT, PEER, ACT, PRELU>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         C::SMEM_BYTES);
    if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
    attr_set[dev] = true;
  }
  const int tiles = ((p.M + BM - 1) / BM) * ((p.N + C::BN - 1) / C::BN);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int grid = tiles < sms ? tiles : sms;
  gemm_tf32x3_kernel<C, STAT, PEER, ACT, PRELU><<<grid, THREADS, C::SMEM_BYTES, stream>>>(tA, tBh, tBl, tX, tY, p);
  return check_launch();
}

}  // namespace gemm
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int b200gnn_split_tf32_f32(const float* W, int64_t rows, int64_t cols, int transpose, float* hi, float* lo,
                                      void* stream) {
  if (!W || !hi || !lo || rows <= 0 || cols <= 0) return B200GNN_ERR_BAD_ARG;
  const int64_t n = rows * cols;
  int grid = (int)((n + 255) / 256);
  if (grid > 132 * 8) grid = 132 * 8;
  gemm::split_tf32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(W, rows, cols, transpose, hi, lo);
  return check_launch();
}

static int g_bnbwd_variant = 0;   // A/B knob: 0 automatic, 1 force the TMA path, 2 force the register path of the BatchNorm-backward epilogue
extern "C" void b200gnn_gemm_set_bnbwd_variant(int v) { g_bnbwd_variant = v; }

// st: the fused column statistics (stat_mode 1 / 2); act: the activation recomputed from Y (Params::act_*, inv_keep) — of the
// A operand without st, of the BatchNorm-backward mask with stat_mode 2; prelu: the PReLU/dropout prologue (stat_mode 0) or
// backward epilogue (stat_mode 4) of Params::act_slope / act_bits.
static int gemm_dispatch(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb, float* C, int64_t ldc,
                         int64_t M, int64_t N, int64_t K, const float* bias, int accumulate, void* stream,
                         const gemm::Params* st = nullptr, const gemm::Params* act = nullptr,
                         const gemm::Params* prelu = nullptr) {
  if (!A || !B_hi || !B_lo || !C || M <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || ldc < N ||
      M >= INT32_MAX || N >= INT32_MAX || K >= INT32_MAX)
    return B200GNN_ERR_BAD_ARG;
  // TMA: 16-byte aligned bases and row pitches
  if (lda % 4 || ldb % 4 || !aligned_to(A, 16) || !aligned_to(B_hi, 16) || !aligned_to(B_lo, 16))
    return B200GNN_ERR_UNSUPPORTED;
  gemm::Params p{};
  p.C = C; p.bias = bias; p.ldc = ldc; p.M = (int32_t)M; p.N = (int32_t)N; p.K = (int32_t)K; p.accumulate = accumulate ? 1 : 0;
  p.n_peer = 0; p.kc = 0; p.row_off = 0; p.bcast = 0;
  if (act) {
    if (!act->act_scale || !act->act_shift || !act->act_bits || !aligned_to(act->act_scale, 16) || !aligned_to(act->act_shift, 16))
      return B200GNN_ERR_BAD_ARG;
    p.act_scale = act->act_scale; p.act_shift = act->act_shift; p.act_bits = act->act_bits; p.act_words = act->act_words;
    p.inv_keep = act->inv_keep;
  }
  if (prelu) {
    if (!prelu->act_slope || !prelu->act_bits) return B200GNN_ERR_BAD_ARG;
    p.act_slope = prelu->act_slope; p.act_bits = prelu->act_bits; p.act_words = prelu->act_words; p.inv_keep = prelu->inv_keep;
    if (prelu->stat_mode == 0) {
      if (N <= 48) return gemm::launch<gemm::Cfg<48, 6>, 0, false, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
      return gemm::launch<gemm::Cfg<128, 4>, 0, false, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
    }
    // backward epilogue: whole 32-column chunks through the vectorised epilogue only
    if (N % 32 || ldc % 4 || !aligned_to(C, 16) || !prelu->bn_y || !aligned_to(prelu->bn_y, 16) || !prelu->slope_partial)
      return B200GNN_ERR_UNSUPPORTED;
    p.stat_mode = 4; p.bn_y = prelu->bn_y; p.slope_partial = prelu->slope_partial;
    return gemm::launch<gemm::Cfg<128, 4>, 4>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
  }
  if (act && !st) {
    // (scale, shift) of all K columns in the statistics block of shared memory
    if (K > (int64_t)gemm::STAT_BYTES / 8) return B200GNN_ERR_UNSUPPORTED;
    if (N <= 48) return gemm::launch<gemm::Cfg<48, 6>, 0, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
    return gemm::launch<gemm::Cfg<128, 4>, 0, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
  }
  if (st) {
    // fused column statistics: whole 32-column chunks through the vectorised epilogue only
    if (N % 32 || N > gemm::STAT_MAX_N || N <= 48 || ldc % 4 || !aligned_to(C, 16) || !st->stat_partial) return B200GNN_ERR_UNSUPPORTED;
    p.stat_mode = st->stat_mode; p.stat_partial = st->stat_partial; p.bn_x = st->bn_x; p.bn_y = st->bn_y;
    p.bn_mean = st->bn_mean; p.bn_invstd = st->bn_invstd; p.inv_keep = st->inv_keep;
    if (p.stat_mode == 1) return gemm::launch<gemm::Cfg<128, 4>, 1>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
    // BatchNorm-backward epilogue: Xout / Y staged through TMA (two chunks in flight per warp) when every chunk is whole
    const bool tma = N % 128 == 0 && (g_bnbwd_variant == 1 || (g_bnbwd_variant == 0 && K < gemm::BNBWD_TMA_MAX_K));
    if (act)
      return tma ? gemm::launch<gemm::Cfg<128, 2, gemm::XY_BYTES>, 3, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream)
                 : gemm::launch<gemm::Cfg<128, 4>, 2, false, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
    if (tma) return gemm::launch<gemm::Cfg<128, 2, gemm::XY_BYTES>, 3>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
    return gemm::launch<gemm::Cfg<128, 4>, 2>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
  }
  if (N <= 48) return gemm::launch<gemm::Cfg<48, 6>>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
  return gemm::launch<gemm::Cfg<128, 4>>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
}

// Slots of the statistics partial buffer the fused GEMMs below fill: [slots][2][N] floats.
extern "C" int64_t b200gnn_gemm_stat_slots(int64_t M, int64_t N) {
  if (M <= 0 || N <= 0) return B200GNN_ERR_BAD_ARG;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int64_t tiles = ((M + gemm::BM - 1) / gemm::BM) * ((N + 127) / 128);
  return gemm::CONSUMER_WARPS * (tiles < sms ? tiles : sms);
}

// C = A · B^T + bias (or C += A · B^T when accumulate: the second GEMM of a SAGEConv, lin_l(mean) + lin_r(x)) with the BatchNorm
// batch statistics of the FINAL C taken in the epilogue: partial[slots][2][N] receives per-slot (sum, sum of squares) over the rows — the input of b200gnn_bn_finalize_f32 (replaces b200gnn_col_stats_f32's sweep over C).
extern "C" int b200gnn_gemm_tf32x3_stats_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                             float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                             int accumulate, float* partial, int64_t slots, void* stream) {
  if (!partial || slots < b200gnn_gemm_stat_slots(M, N) || (accumulate && bias)) return B200GNN_ERR_BAD_ARG;
  gemm::Params st{};
  st.stat_mode = 1; st.stat_partial = partial;
  return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, bias, accumulate, stream, &st);
}

// The input-gradient GEMM of a layer that follows BatchNorm -> ReLU -> dropout (arxiv_pyg/gnn.py:48-50), with pass 1 of that
// block's backward in its epilogue:  dOut = A · B^T (+ C when accumulate);  dz = dOut * [Xout > 0] / (1-p) is what is STORED
// to C, and partial[slots][2][N] receives per-slot (sum dz, sum dz * xhat), xhat = (Y - mean) * invstd.  Follow with
// b200gnn_bn_act_bwd_apply_f32(dOut = C, Xout = NULL, ...).  Xout, Y: [M, ldc] like C.
extern "C" int b200gnn_gemm_tf32x3_bnbwd_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                             float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                             const float* Xout, const float* Y, const float* mean, const float* invstd, float p_drop,
                                             float* partial, int64_t slots, void* stream) {
  if (!partial || !Xout || !Y || !mean || !invstd || p_drop < 0.f || p_drop >= 1.f || slots < b200gnn_gemm_stat_slots(M, N))
    return B200GNN_ERR_BAD_ARG;
  if (!aligned_to(Xout, 16) || !aligned_to(Y, 16) || !aligned_to(mean, 16) || !aligned_to(invstd, 16)) return B200GNN_ERR_UNSUPPORTED;
  gemm::Params st{};
  st.stat_mode = 2; st.stat_partial = partial; st.bn_x = Xout; st.bn_y = Y; st.bn_mean = mean; st.bn_invstd = invstd;
  st.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, nullptr, accumulate, stream, &st);
}

// The bnbwd GEMM above for a block whose activation is not materialised: the mask [Xout > 0] is taken from the packed keep
// bits (uint32 [M][N / 32], as written by b200gnn_dropout_bits_u32) and Y: bit && Y * scale + shift > 0.
extern "C" int b200gnn_gemm_tf32x3_bnbwd_bits_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                                  float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                                  const uint32_t* bits, const float* Y, const float* mean, const float* invstd,
                                                  const float* scale, const float* shift, float p_drop, float* partial,
                                                  int64_t slots, void* stream) {
  if (!partial || !bits || !Y || !mean || !invstd || p_drop < 0.f || p_drop >= 1.f || slots < b200gnn_gemm_stat_slots(M, N))
    return B200GNN_ERR_BAD_ARG;
  if (!aligned_to(Y, 16) || !aligned_to(mean, 16) || !aligned_to(invstd, 16)) return B200GNN_ERR_UNSUPPORTED;
  gemm::Params st{}, act{};
  st.stat_mode = 2; st.stat_partial = partial; st.bn_y = Y; st.bn_mean = mean; st.bn_invstd = invstd;
  st.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  act.act_scale = scale; act.act_shift = shift; act.act_bits = bits; act.act_words = (int32_t)((N + 31) / 32);
  act.inv_keep = st.inv_keep;
  return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, nullptr, accumulate, stream, &st, &act);
}

// C = act(Y) · B^T (+ bias), act(Y) = dropout(relu(Y * scale + shift)) with the keep decisions read from the packed bits
// (uint32 [M][ceil(K / 32)], b200gnn_dropout_bits_u32): bit for bit the GEMM of the activation
// b200gnn_affine_relu_dropout_f32 would materialise, without that [M, K] tensor.  K <= 2048.
extern "C" int b200gnn_gemm_tf32x3_act_f32(const float* Y, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                           float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                           const float* scale, const float* shift, const uint32_t* bits, float p_drop,
                                           void* stream) {
  if (p_drop < 0.f || p_drop >= 1.f) return B200GNN_ERR_BAD_ARG;
  gemm::Params act{};
  act.act_scale = scale; act.act_shift = shift; act.act_bits = bits; act.act_words = (int32_t)((K + 31) / 32);
  act.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  return gemm_dispatch(Y, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, bias, 0, stream, nullptr, &act);
}

// C = dropout(prelu(Z)) · B^T (+ bias) with the activation formed in the GEMM's registers from Z, the slope (device scalar)
// and the packed keep bits (uint32 [M][ceil(K / 32)]): bit for bit the GEMM of the activation b200gnn_prelu_bits_f32
// materialises.  Any K (no per-column table).
extern "C" int b200gnn_gemm_tf32x3_prelu_f32(const float* Z, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                             float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                             const float* slope, const uint32_t* bits, float p_drop, void* stream) {
  if (p_drop < 0.f || p_drop >= 1.f) return B200GNN_ERR_BAD_ARG;
  gemm::Params pr{};
  pr.stat_mode = 0; pr.act_slope = slope; pr.act_bits = bits; pr.act_words = (int32_t)((K + 31) / 32);
  pr.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  return gemm_dispatch(Z, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, bias, 0, stream, nullptr, nullptr, &pr);
}

// The input-gradient GEMM behind x = dropout(prelu(Z)): dA = A · B^T (+ C when accumulate); what is STORED to C is
// dZ = (bit ? dA / (1-p) : 0) * (Z > 0 ? 1 : slope), and slope_grad (+)= sum of (bit ? dA / (1-p) : 0) * Z over Z <= 0,
// reduced in fp64 per consumer warp (partial: double[slots], slots >= b200gnn_gemm_stat_slots(M, N)) and then in slot order.
// Z: [M, ldc] like C; bits: uint32 [M][N / 32]; N a multiple of 32.
extern "C" int b200gnn_gemm_tf32x3_prelu_bwd_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                                 float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, int accumulate,
                                                 const float* Z, const uint32_t* bits, const float* slope, float p_drop,
                                                 float* slope_grad, int slope_accumulate, double* partial, int64_t slots,
                                                 void* stream) {
  if (!Z || !slope_grad || !partial || p_drop < 0.f || p_drop >= 1.f || M <= 0 || N <= 0) return B200GNN_ERR_BAD_ARG;
  const int64_t used = b200gnn_gemm_stat_slots(M, N);
  if (slots < used) return B200GNN_ERR_BAD_ARG;
  gemm::Params pr{};
  pr.stat_mode = 4; pr.act_slope = slope; pr.act_bits = bits; pr.act_words = (int32_t)((N + 31) / 32);
  pr.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  pr.bn_y = Z; pr.slope_partial = partial;
  int rc = gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, nullptr, accumulate, stream, nullptr, nullptr, &pr);
  if (rc) return rc;
  gemm::slope_grad_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(partial, (int)used, slope_grad, slope_accumulate ? 1 : 0);
  return check_launch();
}

extern "C" int b200gnn_gemm_tf32x3_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                       float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, const float* bias,
                                       void* stream) {
  return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, bias, 0, stream);
}

// C += A · B^T (same kernel; the epilogue adds the tile it is about to overwrite).  Used by the chunked G-CRD backward.
extern "C" int b200gnn_gemm_tf32x3_acc_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                           float* C, int64_t ldc, int64_t M, int64_t N, int64_t K, void* stream) {
  return gemm_dispatch(A, lda, B_hi, B_lo, ldb, C, ldc, M, N, K, nullptr, 1, stream);
}

// C = A · B^T (+bias) with the output SCATTERED BY COLUMN BLOCK to `world` destination buffers: columns [q*kc, (q+1)*kc)
// -> C_ptrs[q][(row_off + m) * kc + ...] (each an [*, kc] row-major matrix; for the multi-GPU engine these are the ranks'
// C-layout buffers, peer-mapped).  kc = N / world must be a multiple of 32.  C_ptrs: HOST array of `world` device pointers.
extern "C" int b200gnn_gemm_tf32x3_scatter_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                               float* const* C_ptrs, int32_t world, int64_t row_off, int64_t M, int64_t N, int64_t K,
                                               const float* bias, void* stream) {
  if (!A || !B_hi || !B_lo || !C_ptrs || world <= 0 || world > 16 || M <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || row_off < 0 ||
      M >= INT32_MAX || N >= INT32_MAX || K >= INT32_MAX)
    return B200GNN_ERR_BAD_ARG;
  if (N % world || (N / world) % 32 || N <= 48) return B200GNN_ERR_UNSUPPORTED;
  if (lda % 4 || ldb % 4 || !aligned_to(A, 16) || !aligned_to(B_hi, 16) || !aligned_to(B_lo, 16)) return B200GNN_ERR_UNSUPPORTED;
  gemm::Params p{};
  p.C = nullptr; p.bias = bias; p.ldc = N; p.M = (int32_t)M; p.N = (int32_t)N; p.K = (int32_t)K; p.accumulate = 0;
  p.n_peer = world; p.kc = (int32_t)(N / world); p.row_off = row_off; p.bcast = 0;
  for (int q = 0; q < world; ++q) {
    if (!C_ptrs[q] || !aligned_to(C_ptrs[q], 16)) return B200GNN_ERR_BAD_ARG;
    p.Cp[q] = C_ptrs[q];
  }
  return gemm::launch<gemm::Cfg<128, 4>, 0, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
}

// C = A · B^T (+bias) stored to EVERY destination buffer C_ptrs[q] (row pitch ldc floats) at rows row_off + m: the row
// all-gather of a narrow result (the multi-GPU engine's [N, 40] logits operand) fused into the GEMM epilogue.
extern "C" int b200gnn_gemm_tf32x3_bcast_f32(const float* A, int64_t lda, const float* B_hi, const float* B_lo, int64_t ldb,
                                             float* const* C_ptrs, int32_t world, int64_t row_off, int64_t ldc, int64_t M, int64_t N,
                                             int64_t K, const float* bias, void* stream) {
  if (!A || !B_hi || !B_lo || !C_ptrs || world <= 0 || world > 16 || M <= 0 || N <= 0 || K <= 0 || lda < K || ldb < K || ldc < N ||
      row_off < 0 || M >= INT32_MAX || N >= INT32_MAX || K >= INT32_MAX)
    return B200GNN_ERR_BAD_ARG;
  if (lda % 4 || ldb % 4 || ldc % 4 || !aligned_to(A, 16) || !aligned_to(B_hi, 16) || !aligned_to(B_lo, 16)) return B200GNN_ERR_UNSUPPORTED;
  gemm::Params p{};
  p.C = C_ptrs[0]; p.bias = bias; p.ldc = ldc; p.M = (int32_t)M; p.N = (int32_t)N; p.K = (int32_t)K; p.accumulate = 0;
  p.n_peer = world; p.kc = (int32_t)N; p.row_off = row_off; p.bcast = 1;
  for (int q = 0; q < world; ++q) {
    if (!C_ptrs[q] || !aligned_to(C_ptrs[q], 16)) return B200GNN_ERR_BAD_ARG;
    p.Cp[q] = C_ptrs[q];
  }
  if (N <= 48) return gemm::launch<gemm::Cfg<48, 6>, 0, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
  return gemm::launch<gemm::Cfg<128, 4>, 0, true>(A, lda, B_hi, B_lo, ldb, p, (cudaStream_t)stream);
}
