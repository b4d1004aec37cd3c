// Weight-gradient GEMM on the Hopper tensor cores:   dW[Kin, Nout] = X[Nn, Kin]^T · G[Nn, Nout]   (fp32-faithful, 3xTF32)
//
// The contraction runs over the NODE index (Nn ~ 1.7e5) and the result is tiny (<= 256 x 256), so this is a
// split-K problem: the output is cut into 128 x 128 tiles (Kin and Nout are padded up to the tile grid by TMA zero fill;
// the padding rows and columns of the partials are dropped by the reduction), every CTA owns one tile and a contiguous range of nodes,
// streams its slices of X and G through shared memory exactly once, keeps the tile's partial in registers, and a small
// second kernel adds the per-range partials in a fixed order (deterministic, no atomics).
//
// Both operands are "MN-major" (the contraction index is the slow one in memory).  X^T is the wgmma A operand, which
// comes from registers: TMA lands X as 16 boxes of [32 nodes][8 columns], and every consumer thread loads its fragment
// straight from them (conflict-free: the 4 nodes of one load are 32 bytes apart) and splits it in registers.  G is the
// B operand, which wgmma reads from shared memory K-major only, so the consumers transpose it as they split: TMA lands
// [32 nodes][128 columns] of G and the 256 consumer threads write (hi, lo) as [128 rows][32 nodes] K-major tiles with
// the 128-byte swizzle, the layout of gemm_tf32x3.cu.  The transposed tiles and the X fragments are double-buffered,
// so the split of node block i overlaps the wgmmas of block i-1.  Accumulation as in gemm_tf32x3.cu: each block's 12
// wgmmas go to a fresh register accumulator that is added (fp32, round to nearest) into the running partial.
//
// 384 threads: warpgroup 0 = TMA producer (one thread), warpgroups 1-2 = consumers, 64 rows of the tile each.
#include "common.cuh"
#include "tc_common.cuh"

namespace b200gnn {
namespace wgrad {
using namespace tc;

constexpr int BKN = 32;                       // nodes per stage: one 128-byte K-major row of the transposed operands
constexpr int TM = 128, TN = 128;             // output tile (rows of dW = columns of X, columns of dW = columns of G)
constexpr int THREADS = 384;
constexpr int STAGES = 5;
constexpr int X_BOX = 8;                         // X lands as TM / X_BOX boxes of [BKN nodes][X_BOX columns]
constexpr int RAW_BYTES = BKN * (TM + TN) * 4;   // 32 KB: X and G blocks as TMA lands them
constexpr int OP_BYTES = 128 * BKN * 4;          // 16 KB: one transposed operand, [128 rows][32 nodes]
constexpr int T_BYTES = 2 * OP_BYTES;            // G_hi, G_lo
constexpr int SS_BYTES = TM / 2 * 16;             // ACT: {scale, shift} of the tile's column pairs (c, c + 8)
constexpr int SMEM_BYTES = STAGES * RAW_BYTES + 2 * T_BYTES + 256 + SS_BYTES + 1024;
constexpr int MAX_RANGES = 132;                  // node ranges (workspace partials): one CTA per SM over all tiles
// The workspace holds at most the partials of the largest shape of the 128/256-wide layers (132 ranges of 256 x 256);
// wider outputs have more tiles, fill the SMs with fewer ranges and get proportionally fewer partial slots.
constexpr int64_t MAX_PARTIAL_FLOATS = (int64_t)MAX_RANGES * 256 * 256;
constexpr int MAX_KIN = 2048, MAX_NOUT = 512;
static_assert(SMEM_BYTES <= 232448, "shared memory");

struct Params {
  float* partial;   // [n_ranges][Kpad][Npad], Kpad = Kin rounded up to 128, Npad = Nout rounded up to 32 (TMA zero fill)
  int32_t Nn, Kin, Kpad, Nout, Npad, num_kb;
  int32_t n_tn, n_ranges;   // column tiles of dW, node ranges
  // ACT: X is the BatchNorm input Y of a hidden layer and the operand is its activation, recomputed in registers from Y, the
  // per-column scale / shift and the packed keep bits (uint32 [Nn][act_words]) exactly as gemm_tf32x3.cu's ACT prologue does
  const float* act_scale;
  const float* act_shift;
  const uint32_t* act_bits;
  int32_t act_words;
  float inv_keep;
};

template <bool ACT>
__global__ void __launch_bounds__(THREADS, 1)
wgrad_tf32x3_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmG, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* tbuf = smem + STAGES * RAW_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(tbuf + 2 * T_BYTES);
  uint64_t* empty = full + STAGES;
  float4* act_ss = reinterpret_cast<float4*>(tbuf + 2 * T_BYTES + 256);

  const int tiles = (p.Kpad / TM) * p.n_tn;
  const int tile = (int)blockIdx.x % tiles, range = (int)blockIdx.x / tiles;
  const int mt = tile / p.n_tn, nt = tile % p.n_tn;
  const int kb0 = (int)((int64_t)p.num_kb * range / p.n_ranges);
  const int kb1 = (int)((int64_t)p.num_kb * (range + 1) / p.n_ranges);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    regs_dec<40>();
    if (threadIdx.x == 0) {
      int s = 0; uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty[s], ph ^ 1);
        uint8_t* st = smem + s * RAW_BYTES;
        mbar_expect_tx(&full[s], RAW_BYTES);
        for (int j = 0; j < TM / X_BOX; ++j)
          tma_load_2d(&tmX, &full[s], st + j * BKN * X_BOX * 4, mt * TM + j * X_BOX, kb * BKN);
        tma_load_2d(&tmG, &full[s], st + BKN * TM * 4, nt * TN, kb * BKN);
        if (++s == STAGES) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  regs_inc<232>();

  const int cw = (warp >> 2) - 1;             // warpgroup: rows [64 cw, 64 cw + 64) of the tile
  const int ct = threadIdx.x - 128;           // 0..255
  // X^T fragment of this thread: register i of k-step k is row (column of X) 64 cw + 16 (warp % 4) + lane / 4 + 8 (i % 2),
  // node 8 k + lane % 4 + 4 (i / 2), i.e. box 8 cw + 2 (warp % 4) + i % 2, column lane / 4 of the box
  const uint32_t xfrag = (8 * cw + 2 * (warp & 3)) * (BKN * X_BOX * 4) + (lane & 3) * (X_BOX * 4) + (lane >> 2) * 4;
  // ACT: this thread's two X columns c0, c0 + 8 (one keep word: c0 % 32 < 24); their (scale, shift) wait in shared memory
  // as act_ss[pair] = {sc(c0), sh(c0), sc(c0 + 8), sh(c0 + 8)}; lane l fetches the word of node 32 kb + l one block ahead,
  // and the lanes that need it read it by shuffle
  const int pair = cw * 32 + (warp & 3) * 8 + (lane >> 2);
  const int c0 = mt * TM + cw * 64 + (warp & 3) * 16 + (lane >> 2);
  uint32_t wnext = 0u;
  auto act_word = [&](int kb) {
    const int node = kb * BKN + lane;
    return node < p.Nn && (c0 >> 5) < p.act_words ? __ldg(p.act_bits + (size_t)node * p.act_words + (c0 >> 5)) : 0u;
  };
  if (ACT) {
    if (ct < TM / 2) {
      const int c = mt * TM + (ct >> 3) * 16 + (ct & 7);   // pair ct: columns c, c + 8
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < p.Kin) { v.x = __ldg(p.act_scale + c); v.y = __ldg(p.act_shift + c); }
      if (c + 8 < p.Kin) { v.z = __ldg(p.act_scale + c + 8); v.w = __ldg(p.act_shift + c + 8); }
      act_ss[ct] = v;
    }
    if (kb0 < kb1) wnext = act_word(kb0);
    named_sync(1, 256);
  }
  float acc[64], sum[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) sum[i] = acc[i] = 0.f;
  uint32_t xh0[BKN / 8][4], xl0[BKN / 8][4], xh1[BKN / 8][4], xl1[BKN / 8][4];   // X fragments of two consecutive blocks
  int s = 0; uint32_t ph = 0;
  auto block = [&](int i, uint32_t (&h)[BKN / 8][4], uint32_t (&l)[BKN / 8][4]) {
    uint32_t wcur = 0u;
    if (ACT) {
      wcur = wnext;
      if (kb0 + i + 1 < kb1) wnext = act_word(kb0 + i + 1);
    }
    mbar_wait(&full[s], ph);
    float4 ss = make_float4(0.f, 0.f, 0.f, 0.f);
    int l4 = lane & 3;
    if (ACT) {
      ss = act_ss[pair];
      asm volatile("" : "+r"(l4));             // shuffle source lanes formed per block, not held in 8 registers
    }
    const uint32_t sraw = smem_u32(smem + s * RAW_BYTES);
    const float* rg = reinterpret_cast<const float*>(smem + s * RAW_BYTES + BKN * TM * 4);   // [32 nodes][128]
    uint8_t* T = tbuf + (i & 1) * T_BYTES;
    // transpose + split of G: item = (row r, 4-node chunk c); consecutive threads take consecutive rows, so the
    // reads are conflict-free and the 16-byte swizzled writes of 8 consecutive rows cover all banks
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int idx = u * 256 + ct;
      const int r = idx & 127, c = idx >> 7;
      const float* src = rg + (4 * c) * 128 + r;
      const uint4 v = make_uint4(__float_as_uint(src[0]), __float_as_uint(src[128]), __float_as_uint(src[256]),
                                 __float_as_uint(src[384]));
      uint4 hv, lv;
      split4(v, hv, lv);
      *reinterpret_cast<uint4*>(T + swz128(r, c)) = hv;
      *reinterpret_cast<uint4*>(T + OP_BYTES + swz128(r, c)) = lv;
    }
#pragma unroll
    for (int k = 0; k < BKN / 8; ++k)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        // register j: column c0 + 8 (j % 2), node 8 k + lane % 4 + 4 (j / 2) of the block
        uint32_t v = lds32(sraw + xfrag + (j & 1) * (BKN * X_BOX * 4) + (8 * k + 4 * (j >> 1)) * (X_BOX * 4));
        if (ACT) {
          const uint32_t w = __shfl_sync(0xffffffffu, wcur, 8 * k + l4 + 4 * (j >> 1));
          const float y = fmaxf(fmaf(__uint_as_float(v), (j & 1) ? ss.z : ss.x, (j & 1) ? ss.w : ss.y), 0.f) * p.inv_keep;
          v = (w >> ((c0 & 31) + 8 * (j & 1))) & 1u ? __float_as_uint(y) : 0u;
        }
        split1(v, h[k][j], l[k][j]);
      }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    mbar_arrive(&empty[s]);                    // the raw block has been read
    if (i > 0) {                               // block i-1's wgmmas have retired: promote
      wgmma_wait<0>();
      acc_fence(acc);
#pragma unroll
      for (int j = 0; j < 64; ++j) sum[j] += acc[j];
    }
    named_sync(1, 256);                        // T[i & 1] complete; every warpgroup is done with T[(i + 1) & 1]
    reg_fence(h); reg_fence(l);
    wgmma_fence();
    const uint32_t sa = smem_u32(T);
#pragma unroll
    for (int k = 0; k < BKN / 8; ++k) {        // the small correction terms first (see gemm_tf32x3.cu)
      const uint32_t koff = k * 32;
      wgmma_tf32_n128_rs(acc, l[k], make_desc_k128(sa + koff), k != 0);
      wgmma_tf32_n128_rs(acc, h[k], make_desc_k128(sa + OP_BYTES + koff), 1);
    }
#pragma unroll
    for (int k = 0; k < BKN / 8; ++k) wgmma_tf32_n128_rs(acc, h[k], make_desc_k128(sa + k * 32), 1);
    wgmma_commit();
    if (++s == STAGES) { s = 0; ph ^= 1; }
  };
  for (int i = 0; i < kb1 - kb0; i += 2) {
    block(i, xh0, xl0);
    if (i + 1 < kb1 - kb0) block(i + 1, xh1, xl1);
  }
  if (kb1 > kb0) {
    wgmma_wait<0>();
    acc_fence(acc);
#pragma unroll
    for (int j = 0; j < 64; ++j) sum[j] += acc[j];
  }
  // fragment -> partial: rows mt*128 + 64 cw + 16 (warp % 4) + lane/4 (+8), columns nt*128 + 8 j + 2 (lane % 4)
  float* out = p.partial + (size_t)range * p.Kpad * p.Npad;
  const int row0 = mt * TM + cw * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = nt * TN + 8 * j + 2 * (lane & 3);
    if (col < p.Npad) {
      *reinterpret_cast<float2*>(out + (size_t)row0 * p.Npad + col) = make_float2(sum[4 * j], sum[4 * j + 1]);
      *reinterpret_cast<float2*>(out + (size_t)(row0 + 8) * p.Npad + col) = make_float2(sum[4 * j + 2], sum[4 * j + 3]);
    }
  }
}

// dW[r][c] = sum over CTAs of partial[cta][r][c], dropping the padding rows and columns.  32 float4 columns x 8 groups per
// CTA: group g adds partials g, g+8, ... and the groups are combined in order through shared memory (fixed order,
// deterministic; 8x shorter dependent chains than one thread per element).
constexpr int RED_VECS = 32, RED_GROUPS = 8;
__global__ void __launch_bounds__(RED_VECS * RED_GROUPS) wgrad_reduce_kernel(const float4* __restrict__ partial, int n_part,
                                                                             int Kin, int Kpad, int Nout, int Npad,
                                                                             float* __restrict__ out) {
  __shared__ float4 sh[RED_GROUPS][RED_VECS];
  const int64_t n_vec = (int64_t)Kpad * Npad / 4;
  const int v = threadIdx.x % RED_VECS, g = threadIdx.x / RED_VECS;
  const int64_t i = (int64_t)blockIdx.x * RED_VECS + v;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < n_vec)
    for (int c = g; c < n_part; c += RED_GROUPS) {
      const float4 x = __ldcs(partial + (size_t)c * n_vec + i);
      acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
    }
  sh[g][v] = acc;
  __syncthreads();
  if (g != 0 || i >= n_vec) return;
  const int row = (int)(i / (Npad / 4)), c4 = (int)(i % (Npad / 4)) * 4;
  if (c4 >= Nout || row >= Kin) return;
#pragma unroll
  for (int j = 1; j < RED_GROUPS; ++j) {
    const float4 x = sh[j][v];
    acc.x += x.x; acc.y += x.y; acc.z += x.z; acc.w += x.w;
  }
  *reinterpret_cast<float4*>(out + (size_t)row * Nout + c4) = acc;   // Nout % 4 == 0
}

// [rows, width] fp32 row-major (ld): boxes of box_cols columns x BKN rows, no swizzle, zero fill past the last row / column
static bool make_map_rows(CUtensorMap* m, const float* base, int64_t rows, int64_t width, int64_t ld, int box_cols) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {(cuuint64_t)width, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_cols, (cuuint32_t)BKN};
  cuuint32_t estr[2] = {1, 1};
  return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int64_t pad_k(int64_t Kin) { return (Kin + TM - 1) / TM * TM; }
static int64_t pad_n(int64_t Nout) { return (Nout + 31) / 32 * 32; }
// node ranges the workspace has room for: MAX_RANGES for every output up to 256 x 256
static int range_cap(int64_t Kin, int64_t Nout) {
  const int64_t c = MAX_PARTIAL_FLOATS / (pad_k(Kin) * pad_n(Nout));
  return (int)(c > MAX_RANGES ? MAX_RANGES : (c < 1 ? 1 : c));
}

}  // namespace wgrad
}  // namespace b200gnn

using namespace b200gnn;

extern "C" int64_t b200gnn_wgrad_workspace_floats(int64_t Kin, int64_t Nout) {
  if (Kin <= 0 || Nout <= 0) return B200GNN_ERR_BAD_ARG;
  if (Kin > wgrad::MAX_KIN || Nout > wgrad::MAX_NOUT) return B200GNN_ERR_UNSUPPORTED;
  return wgrad::range_cap(Kin, Nout) * wgrad::pad_k(Kin) * wgrad::pad_n(Nout);
}

template <bool ACT>
static int wgrad_launch(const float* X, int64_t ldx, const float* G, int64_t ldg, float* dW, int64_t Nn, int64_t Kin, int64_t Nout,
                        float* workspace, const wgrad::Params& act, void* stream) {
  if (!X || !G || !dW || !workspace || Nn <= 0 || Kin <= 0 || Nout <= 0 || ldx < Kin || ldg < Nout || Nn >= INT32_MAX)
    return B200GNN_ERR_BAD_ARG;
  // tensor-core tiling: Kin a multiple of 4 up to 2048 (padded to 128), Nout a multiple of 4 up to 512 (padded to 32), both
  // by TMA zero fill; 16-byte alignment
  if (Kin % 4 || Kin > wgrad::MAX_KIN || Nout % 4 || Nout > wgrad::MAX_NOUT || ldx % 4 || ldg % 4 || !aligned_to(X, 16) || !aligned_to(G, 16) ||
      !aligned_to(dW, 16) || !aligned_to(workspace, 16))
    return B200GNN_ERR_UNSUPPORTED;
  CUtensorMap tX, tG;
  if (!wgrad::make_map_rows(&tX, X, Nn, Kin, ldx, wgrad::X_BOX) || !wgrad::make_map_rows(&tG, G, Nn, Nout, ldg, wgrad::TN))
    return B200GNN_ERR_UNSUPPORTED;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  static bool attr_set[64] = {};                    // per device
  if (dev >= 0 && dev < 64 && !attr_set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(wgrad::wgrad_tf32x3_kernel<ACT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         wgrad::SMEM_BYTES);
    if (e != cudaSuccess) { set_cuda_error(e); return B200GNN_ERR_CUDA; }
    attr_set[dev] = true;
  }
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaStream_t st = (cudaStream_t)stream;
  wgrad::Params p = act;
  p.partial = workspace; p.Nn = (int32_t)Nn; p.Kin = (int32_t)Kin; p.Nout = (int32_t)Nout;
  p.Kpad = (int32_t)wgrad::pad_k(Kin);
  p.Npad = (int32_t)wgrad::pad_n(Nout);
  p.num_kb = (int32_t)((Nn + wgrad::BKN - 1) / wgrad::BKN);
  p.n_tn = (p.Npad + wgrad::TN - 1) / wgrad::TN;
  const int tiles = (int)(p.Kpad / wgrad::TM) * p.n_tn;
  int ranges = sms / tiles;                          // one CTA per SM over all tiles
  const int cap = wgrad::range_cap(Kin, Nout);       // the workspace holds this many partials
  if (ranges > cap) ranges = cap;
  if (ranges > p.num_kb) ranges = p.num_kb;
  if (ranges < 1) ranges = 1;
  p.n_ranges = ranges;
  int rc;
  wgrad::wgrad_tf32x3_kernel<ACT><<<tiles * ranges, wgrad::THREADS, wgrad::SMEM_BYTES, st>>>(tX, tG, p);
  if ((rc = check_launch())) return rc;
  const int64_t n_vec = (int64_t)p.Kpad * p.Npad / 4;
  wgrad::wgrad_reduce_kernel<<<(int)((n_vec + wgrad::RED_VECS - 1) / wgrad::RED_VECS), wgrad::RED_VECS * wgrad::RED_GROUPS, 0, st>>>(
      reinterpret_cast<const float4*>(workspace), ranges, (int)Kin, p.Kpad, (int)Nout, p.Npad, dW);
  return check_launch();
}

extern "C" int b200gnn_gemm_wgrad_tf32x3_f32(const float* X, int64_t ldx, const float* G, int64_t ldg, float* dW,
                                             int64_t Nn, int64_t Kin, int64_t Nout, float* workspace, void* stream) {
  return wgrad_launch<false>(X, ldx, G, ldg, dW, Nn, Kin, Nout, workspace, wgrad::Params{}, stream);
}

// dW = act(Y)^T · G with act(Y) = dropout(relu(Y * scale + shift)) recomputed from Y and the packed keep bits
// (uint32 [Nn][ceil(Kin / 32)], b200gnn_dropout_bits_u32): bit for bit the weight gradient of the materialised activation.
extern "C" int b200gnn_gemm_wgrad_tf32x3_act_f32(const float* Y, int64_t ldx, const float* G, int64_t ldg, float* dW,
                                                 int64_t Nn, int64_t Kin, int64_t Nout, const float* scale, const float* shift,
                                                 const uint32_t* bits, float p_drop, float* workspace, void* stream) {
  if (!scale || !shift || !bits || p_drop < 0.f || p_drop >= 1.f) return B200GNN_ERR_BAD_ARG;
  wgrad::Params act{};
  act.act_scale = scale; act.act_shift = shift; act.act_bits = bits; act.act_words = (int32_t)((Kin + 31) / 32);
  act.inv_keep = p_drop > 0.f ? 1.f / (1.f - p_drop) : 1.f;
  return wgrad_launch<true>(Y, ldx, G, ldg, dW, Nn, Kin, Nout, workspace, act, stream);
}
