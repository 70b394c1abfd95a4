// Residual GEMM fused with the LayerNorm that follows it (sm_90a, wgmma + TMA).
//
//   x[M, D]  (fp32, in place)  <-  x + A[M, K] * W[D, K]^T + bias            (timm Block: x = x + attn(..) / mlp(..))
//   xn[M, D] (bf16)            <-  LayerNorm(x_new; gamma, beta, eps)         (norm2 / next block's norm1 / final norm)
//
// Why: as separate kernels the attention-projection and fc2 GEMMs are bound by the fp32 read-modify-write of the
// residual stream and the LayerNorm re-reads it from HBM; here each updated row is normalised while it is still in
// registers.
//
// Warpgroup 0 is the TMA producer; warpgroups 1 and 2 accumulate with wgmma, so a row's values sit in two column parts
// (two warpgroups, or two CTAs):
//   pass 1: v = (acc + bias) + x is stored back to x and kept in the accumulator registers; row sums are reduced over
//           the quad of lanes that holds a row, then over the column parts through shared memory;
//   pass 2: the same for the squared deviations from the mean (two-pass variance, as layernorm_kernel);
//   pass 3: normalise, pack to bf16, store xn.
// Rounding points are those of the unfused pair (residual-accumulate GEMM epilogue + layernorm_kernel): fp32 x, bf16 xn.
//
// MODE 0: one CTA per 64-row tile, all D columns; warpgroup w accumulates columns [D/2 w, D/2 (w + 1)).
// MODE 1: a cluster of two CTAs on 128 rows; each CTA loads half of the W tile and multicasts it into both, so every W
//         byte is fetched once per 128 rows.  Same work per row as MODE 0: bit-identical results.
// MODE 2 (D = 384): persistent; a cluster of two CTAs walks 64-row tiles with the grid's stride.  CTA r computes the
//         columns [192 r, 192 r + 192) (wgmma m64n192k16), staging its own A rows and only its half of W.  The two MMA
//         warpgroups of a CTA take the cluster's tiles in turn ("ping-pong", as in gemm.cuh): one warpgroup's epilogue
//         runs under the other's main loop.  The producer TMA-loads each tile's x slice into the warpgroup's own
//         shared-memory buffer ahead of the main loop.  The row statistics of the column parts are exchanged through
//         distributed shared memory.  Their summation order reproduces the kernel each K used before (see
//         gln_pair_epilogue).
#pragma once
#include "gemm.cuh"

namespace pq {

struct GemmLnParams {
  int M, K;
  const float* bias;     // [D] or nullptr
  const float* gamma;    // [D]
  const float* beta;     // [D]
  float eps;
  int num_m_tiles;       // tiles of kTileM rows (MODE 2: walked by the clusters with the grid's stride)
};

constexpr int GLN_THREADS = 384;
constexpr int GLN_BLOCK_M = 64;

// MODE 0 / 1
template <int D, int MODE>
struct GemmLnCfg {
  static_assert(MODE == 0 || MODE == 1, "MODE");
  static constexpr int kCG = MODE == 0 ? 1 : 2;                       // CTAs per cluster
  static constexpr int kTileM = GLN_BLOCK_M * kCG;                    // rows per cluster
  static constexpr int kCols = D;                                     // columns per CTA
  static constexpr int kNW = kCols / 2;                               // columns per MMA warpgroup
  static constexpr int kParts = 2;                                    // column parts of a row
  static constexpr int kABox = GLN_BLOCK_M;                           // A rows per TMA box
  static constexpr int kLoadRows = MODE == 1 ? D / 2 : kCols;         // W rows this CTA loads per k-block
  static constexpr int kBox = kLoadRows > 256 ? kLoadRows / 2 : kLoadRows;   // TMA box rows (at most 256)
  static constexpr int kABytes = GLN_BLOCK_M * GEMM_BLOCK_K * 2;      // 8 KB
  static constexpr int kBBytes = kCols * GEMM_BLOCK_K * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kParamBytes = 3 * kCols * 4 + 2 * kParts * GLN_BLOCK_M * 4;   // bias, gamma, beta; row partials
  static constexpr int kBarBytes = 256;
  static constexpr int kStagesRaw = (232448 - 1024 - kBarBytes - kParamBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + kParamBytes + kBarBytes + 1024;
  static_assert(D == 192 || D == 384, "embed_dim");
  static_assert(kNW % 16 == 0 && kNW <= 256, "wgmma N");
  static_assert((kNW * GEMM_BLOCK_K * 2) % 1024 == 0 && (kBox * GEMM_BLOCK_K * 2) % 1024 == 0, "1024-B aligned operand tiles");
  static_assert(kStages >= 3, "pipeline depth");
};

// MODE 2.  Shared memory: 3 operand stages (A 64 x 64 + W 192 x 64), one x slice per MMA warpgroup (2 x 48 KB), the
// parameters.
template <int D>
struct GemmLnCfg<D, 2> {
  static_assert(D == 384, "the persistent column-split kernel is built for D = 384");
  static constexpr int kCG = 2;                                       // CTAs per cluster: the two column halves
  static constexpr int kTileM = GLN_BLOCK_M;                          // 64 rows per tile
  static constexpr int kCols = D / 2;                                 // columns per CTA; one m64n192 per warpgroup
  static constexpr int kABox = GLN_BLOCK_M;                           // A rows per TMA box
  static constexpr int kBox = kCols;                                  // W rows per TMA box
  static constexpr int kABytes = GLN_BLOCK_M * GEMM_BLOCK_K * 2;      // 8 KB
  static constexpr int kBBytes = kCols * GEMM_BLOCK_K * 2;            // 24 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = 3;
  static constexpr int kXBoxCols = 32;                                // fp32 x boxes: one 128-B swizzle row wide
  static constexpr int kXBoxBytes = GLN_BLOCK_M * kXBoxCols * 4;      // 8 KB
  static constexpr int kXBytes = GLN_BLOCK_M * kCols * 4;             // 48 KB: one warpgroup's tile
  static constexpr int kParamBytes = 3 * kCols * 4 + 2 * 2 * 4 * GLN_BLOCK_M * 4;   // bias, gamma, beta; [wg][round][part][row]
  static constexpr int kBarBytes = 256;
  static constexpr int kSmemBytes = kStages * kStageBytes + 2 * kXBytes + kParamBytes + kBarBytes + 1024;
  static_assert(kSmemBytes <= 232448, "shared memory");
};

// Row statistics of MODE 2 are summed over four 96-column parts from this K on (the order of the column-split kernel
// that ran fc2 before), over two 192-column parts below it (the order of the full-row kernel, MODE 0, that ran
// attn.proj).  Selected by K only: a row's bits do not depend on the batch.
constexpr int GLN_PARTS4_MIN_K = 768;

// Sum of one row's column parts, in a fixed order (every thread of every CTA that holds the row gets the same bits).
template <int PARTS>
__device__ __forceinline__ float gln_row_total(const float* s_part, int r) {
  float t = s_part[r] + s_part[GLN_BLOCK_M + r];
  if constexpr (PARTS == 4) t += s_part[2 * GLN_BLOCK_M + r] + s_part[3 * GLN_BLOCK_M + r];
  return t;
}

// Epilogue shared by the full-row fused kernels (MODE 0 / 1, mlp_ln.cuh): `acc` holds the 64 x NW block of one MMA
// warpgroup (rows m0.., columns wg * NW..); x += acc + bias in place, then xn = bf16(LayerNorm(x)) over the D columns of
// a row, whose two column parts are combined through s_part.
template <int D, int NW>
__device__ __forceinline__ void gln_epilogue(float (&acc)[NW / 2], float* __restrict__ x, __nv_bfloat16* __restrict__ xn, int M,
                                             float eps, int m0, int wg, const float* s_bias, const float* s_gamma,
                                             const float* s_beta, float* s_part) {
  constexpr int kNW = NW;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int lr = (t >> 5) * 16 + (lane >> 2);        // local rows lr, lr + 8
  const bool ok_a = m0 + lr < M, ok_b = m0 + lr + 8 < M;
  float* xa = x + static_cast<long long>(m0 + lr) * D + wg * kNW + 2 * (lane & 3);
  float* xb = xa + 8ll * D;

  // pass 1: residual update, row sums
  float sa = 0.f, sb = 0.f;
#pragma unroll
  for (int i = 0; i < kNW / 8; ++i) {
    const int cl = wg * kNW + i * 8 + 2 * (lane & 3);   // column
    const float b0 = s_bias[cl], b1 = s_bias[cl + 1];
    float2 xo = ok_a ? *reinterpret_cast<const float2*>(xa + i * 8) : make_float2(0.f, 0.f);
    acc[4 * i] = (acc[4 * i] + b0) + xo.x;
    acc[4 * i + 1] = (acc[4 * i + 1] + b1) + xo.y;
    if (ok_a) *reinterpret_cast<float2*>(xa + i * 8) = make_float2(acc[4 * i], acc[4 * i + 1]);
    xo = ok_b ? *reinterpret_cast<const float2*>(xb + i * 8) : make_float2(0.f, 0.f);
    acc[4 * i + 2] = (acc[4 * i + 2] + b0) + xo.x;
    acc[4 * i + 3] = (acc[4 * i + 3] + b1) + xo.y;
    if (ok_b) *reinterpret_cast<float2*>(xb + i * 8) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    sa += acc[4 * i] + acc[4 * i + 1];
    sb += acc[4 * i + 2] + acc[4 * i + 3];
  }
  float mean_a = 0.f, mean_b = 0.f, rstd_a = 0.f, rstd_b = 0.f;
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    if (round == 1) {                                // pass 2: squared deviations from the mean
      sa = 0.f;
      sb = 0.f;
#pragma unroll
      for (int i = 0; i < kNW / 8; ++i) {
        const float a0 = acc[4 * i] - mean_a, a1 = acc[4 * i + 1] - mean_a;
        const float d0 = acc[4 * i + 2] - mean_b, d1 = acc[4 * i + 3] - mean_b;
        sa += a0 * a0 + a1 * a1;
        sb += d0 * d0 + d1 * d1;
      }
    }
    sa += __shfl_xor_sync(0xffffffffu, sa, 1);
    sa += __shfl_xor_sync(0xffffffffu, sa, 2);
    sb += __shfl_xor_sync(0xffffffffu, sb, 1);
    sb += __shfl_xor_sync(0xffffffffu, sb, 2);
    float* slot = s_part + (round * 2 + wg) * GLN_BLOCK_M;
    if ((lane & 3) == 0) {
      slot[lr] = sa;
      slot[lr + 8] = sb;
    }
    asm volatile("bar.sync 1, 256;" ::: "memory");   // the two MMA warpgroups
    const float* tot = s_part + round * 2 * GLN_BLOCK_M;
    const float ta = gln_row_total<2>(tot, lr), tb = gln_row_total<2>(tot, lr + 8);
    if (round == 0) {
      mean_a = ta * (1.0f / D);
      mean_b = tb * (1.0f / D);
    } else {
      rstd_a = 1.0f / sqrtf(ta * (1.0f / D) + eps);
      rstd_b = 1.0f / sqrtf(tb * (1.0f / D) + eps);
    }
  }
  // pass 3: normalise, bf16
  uint32_t* na = reinterpret_cast<uint32_t*>(xn + static_cast<long long>(m0 + lr) * D + wg * kNW + 2 * (lane & 3));
  uint32_t* nb = na + 4ll * D;
#pragma unroll
  for (int i = 0; i < kNW / 8; ++i) {
    const int cl = wg * kNW + i * 8 + 2 * (lane & 3);
    const float g0 = s_gamma[cl], g1 = s_gamma[cl + 1], e0 = s_beta[cl], e1 = s_beta[cl + 1];
    if (ok_a) na[i * 4] = pack_bf16((acc[4 * i] - mean_a) * rstd_a * g0 + e0, (acc[4 * i + 1] - mean_a) * rstd_a * g1 + e1);
    if (ok_b) nb[i * 4] = pack_bf16((acc[4 * i + 2] - mean_b) * rstd_b * g0 + e0, (acc[4 * i + 3] - mean_b) * rstd_b * g1 + e1);
  }
}

// Epilogue of MODE 2 for one MMA warpgroup: `acc` holds rows m0 + [0, 64) x the CTA's columns c0 + [0, D/2); their x
// slice is in the warpgroup's shared-memory buffer (xs: D/64 TMA boxes of [64 rows][32] fp32, 128B swizzle).  The x
// buffer is released on x_empty as soon as it has been read.  The row statistics are summed per column part in the order
// of the kernel that ran this K before: PARTS = 4, 96-column parts (rank 2 + half), each thread keeping one sum per
// half; PARTS = 2, one 192-column part per CTA, with the in-thread order of a MODE 0 warpgroup.  The partials go to both
// CTAs' s_part (this warpgroup's [round][part][row]); stat_bar[round] collects the arrivals of this warpgroup and of the
// peer CTA's warpgroup with the same rows (completing once per tile of the warpgroup, parity `par`).
template <int D, int PARTS>
__device__ __forceinline__ void gln_pair_epilogue(float (&acc)[D / 4], const uint8_t* xs, float* __restrict__ x,
                                                  __nv_bfloat16* __restrict__ xn, int M, float eps, int m0, int c0,
                                                  uint32_t rank, const float* s_bias, const float* s_gamma,
                                                  const float* s_beta, float* s_part, uint64_t* stat_bar, uint32_t par,
                                                  uint64_t* x_empty) {
  using Cfg = GemmLnCfg<D, 2>;
  constexpr int kI = Cfg::kCols / 8;                  // accumulator groups of 8 columns
  constexpr int kH = PARTS / 2;                       // column parts per thread
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int lr = (t >> 5) * 16 + (lane >> 2);         // local rows lr, lr + 8
  const bool ok_a = m0 + lr < M, ok_b = m0 + lr + 8 < M;
  float* xa = x + static_cast<long long>(m0 + lr) * D + c0 + 2 * (lane & 3);
  float* xb = xa + 8ll * D;
  // 128B swizzle: 16-B chunk c of row r sits at chunk c ^ (r % 8); r % 8 = lane / 4 for both rows
  const uint8_t* xsa = xs + lr * 128 + (lane & 1) * 8;
  const uint8_t* xsb = xsa + 8 * 128;
  const uint32_t peer = rank ^ 1u;

  // pass 1: residual update, row sums
  float sa[kH], sb[kH];
#pragma unroll
  for (int h = 0; h < kH; ++h) { sa[h] = 0.f; sb[h] = 0.f; }
#pragma unroll
  for (int i = 0; i < kI; ++i) {
    const int h = i / (kI / kH);
    const int cl = i * 8 + 2 * (lane & 3);            // column inside this CTA's part
    const float b0 = s_bias[cl], b1 = s_bias[cl + 1];
    const int off = (i >> 2) * Cfg::kXBoxBytes + ((((i & 3) * 2 + ((lane >> 1) & 1)) ^ (lane >> 2)) << 4);
    float2 xo = *reinterpret_cast<const float2*>(xsa + off);
    acc[4 * i] = (acc[4 * i] + b0) + xo.x;
    acc[4 * i + 1] = (acc[4 * i + 1] + b1) + xo.y;
    if (ok_a) *reinterpret_cast<float2*>(xa + i * 8) = make_float2(acc[4 * i], acc[4 * i + 1]);
    xo = *reinterpret_cast<const float2*>(xsb + off);
    acc[4 * i + 2] = (acc[4 * i + 2] + b0) + xo.x;
    acc[4 * i + 3] = (acc[4 * i + 3] + b1) + xo.y;
    if (ok_b) *reinterpret_cast<float2*>(xb + i * 8) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    sa[h] += acc[4 * i] + acc[4 * i + 1];
    sb[h] += acc[4 * i + 2] + acc[4 * i + 3];
  }
  mbar_arrive(x_empty);                               // the producer may load the next tile's x slice
  float mean_a = 0.f, mean_b = 0.f, rstd_a = 0.f, rstd_b = 0.f;
#pragma unroll
  for (int round = 0; round < 2; ++round) {
    if (round == 1) {                                 // pass 2: squared deviations from the mean
#pragma unroll
      for (int h = 0; h < kH; ++h) { sa[h] = 0.f; sb[h] = 0.f; }
#pragma unroll
      for (int i = 0; i < kI; ++i) {
        const int h = i / (kI / kH);
        const float a0 = acc[4 * i] - mean_a, a1 = acc[4 * i + 1] - mean_a;
        const float d0 = acc[4 * i + 2] - mean_b, d1 = acc[4 * i + 3] - mean_b;
        sa[h] += a0 * a0 + a1 * a1;
        sb[h] += d0 * d0 + d1 * d1;
      }
    }
    float* slots = s_part + round * PARTS * GLN_BLOCK_M;
#pragma unroll
    for (int h = 0; h < kH; ++h) {
      sa[h] += __shfl_xor_sync(0xffffffffu, sa[h], 1);
      sa[h] += __shfl_xor_sync(0xffffffffu, sa[h], 2);
      sb[h] += __shfl_xor_sync(0xffffffffu, sb[h], 1);
      sb[h] += __shfl_xor_sync(0xffffffffu, sb[h], 2);
      float* slot = slots + (static_cast<int>(rank & 1u) * kH + h) * GLN_BLOCK_M;
      if ((lane & 3) == 0) {
        slot[lr] = sa[h];
        slot[lr + 8] = sb[h];
        st_cluster_f32(mapa_cluster(smem_u32(slot + lr), peer), sa[h]);
        st_cluster_f32(mapa_cluster(smem_u32(slot + lr + 8), peer), sb[h]);
      }
    }
    mbar_arrive(&stat_bar[round]);
    mbar_arrive_cluster(mapa_cluster(smem_u32(&stat_bar[round]), peer));
    mbar_wait_cluster(&stat_bar[round], par);
    const float ta = gln_row_total<PARTS>(slots, lr), tb = gln_row_total<PARTS>(slots, lr + 8);
    if (round == 0) {
      mean_a = ta * (1.0f / D);
      mean_b = tb * (1.0f / D);
    } else {
      rstd_a = 1.0f / sqrtf(ta * (1.0f / D) + eps);
      rstd_b = 1.0f / sqrtf(tb * (1.0f / D) + eps);
    }
  }
  // pass 3: normalise, bf16
  uint32_t* na = reinterpret_cast<uint32_t*>(xn + static_cast<long long>(m0 + lr) * D + c0 + 2 * (lane & 3));
  uint32_t* nb = na + 4ll * D;
#pragma unroll
  for (int i = 0; i < kI; ++i) {
    const int cl = i * 8 + 2 * (lane & 3);
    const float g0 = s_gamma[cl], g1 = s_gamma[cl + 1], e0 = s_beta[cl], e1 = s_beta[cl + 1];
    if (ok_a) na[i * 4] = pack_bf16((acc[4 * i] - mean_a) * rstd_a * g0 + e0, (acc[4 * i + 1] - mean_a) * rstd_a * g1 + e1);
    if (ok_b) nb[i * 4] = pack_bf16((acc[4 * i + 2] - mean_b) * rstd_b * g0 + e0, (acc[4 * i + 3] - mean_b) * rstd_b * g1 + e1);
  }
}

// MODE 2 (see the top of the file).  Grid: clusters of two CTAs; cluster c takes the 64-row tiles c, c + clusters, ...
// and its j-th tile goes to MMA warpgroup j % 2 of both CTAs.  CTA r computes columns [192 r, 192 r + 192) and loads its
// own A and W boxes: no operand is multicast, so a stage is free as soon as the warpgroup that read it releases it, and
// neither CTA's ring waits on the other's.  Barriers: full/empty per operand stage, x_full[wg] / x_empty[wg] for the
// warpgroups' x buffers, stat_bar[wg][round] for the row statistics of the warpgroup's rows.  Both CTAs walk every tile
// of their cluster, also rows past M (TMA zero-fills them, the stores are guarded).
template <int D>
__device__ __forceinline__ void gln_pair_persistent(const CUtensorMap* tmA, const CUtensorMap* tmB, const CUtensorMap* tmX,
                                                    float* __restrict__ x, __nv_bfloat16* __restrict__ xn,
                                                    const GemmLnParams& p) {
  using Cfg = GemmLnCfg<D, 2>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;
  uint8_t* xs = smem + Cfg::kStages * Cfg::kStageBytes;  // [wg][48 KB]
  float* s_bias = reinterpret_cast<float*>(xs + 2 * Cfg::kXBytes);
  float* s_gamma = s_bias + Cfg::kCols;
  float* s_beta = s_gamma + Cfg::kCols;
  float* s_part = s_beta + Cfg::kCols;                 // [wg][round][4 parts][64 rows]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_bias) + Cfg::kParamBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  uint64_t* x_full = empty_bar + Cfg::kStages;         // [wg]
  uint64_t* x_empty = x_full + 2;                      // [wg]
  uint64_t* stat_bar = x_empty + 2;                    // [wg][round]

  const uint32_t rank = cluster_ctarank();
  const int cluster = static_cast<int>(blockIdx.x / Cfg::kCG), clusters = static_cast<int>(gridDim.x / Cfg::kCG);
  const int c0 = static_cast<int>(rank & 1u) * Cfg::kCols;   // first column of this CTA
  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;

  grid_dep_launch();
  if (threadIdx.x == 0) {
    prefetch_tmap(tmA);
    prefetch_tmap(tmB);
    prefetch_tmap(tmX);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);                     // the one warpgroup that reads the stage
    }
    for (int w = 0; w < 2; ++w) {
      mbar_init(&x_full[w], 1);
      mbar_init(&x_empty[w], 128);                     // every thread of the warpgroup
    }
    for (int i = 0; i < 4; ++i) mbar_init(&stat_bar[i], 2 * 128);   // a warpgroup and its peer's
    fence_mbar_init();
  }
  // bias / gamma / beta are weights (never written by a preceding kernel): stage them before the dependency wait
  for (int j = threadIdx.x; j < Cfg::kCols; j += GLN_THREADS) {
    s_bias[j] = (p.bias != nullptr) ? __ldg(p.bias + c0 + j) : 0.0f;
    s_gamma[j] = __ldg(p.gamma + c0 + j);
    s_beta[j] = __ldg(p.beta + c0 + j);
  }
  cluster_sync_all();
  grid_dep_wait();

  if (threadIdx.x < 128) {
    // ===================== TMA producer: the cluster's tiles in order, running ahead across tiles =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      int j = 0;
      for (int tile = cluster; tile < p.num_m_tiles; tile += clusters, ++j) {
        const int m0 = tile * Cfg::kTileM;
        // the x slice first: its buffer was freed by pass 1 of the warpgroup's previous tile's epilogue, and the
        // warpgroup finishes that epilogue before it needs this tile's operands
        const int w = j & 1;
        mbar_wait_mma(&x_empty[w], ((j >> 1) & 1) ^ 1u);
        mbar_expect_tx(&x_full[w], Cfg::kXBytes);
#pragma unroll
        for (int b = 0; b < Cfg::kCols / Cfg::kXBoxCols; ++b)
          tma_load_2d(xs + w * Cfg::kXBytes + b * Cfg::kXBoxBytes, tmX, &x_full[w], c0 + b * Cfg::kXBoxCols, m0);
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, tmA, &full_bar[stage], kb * GEMM_BLOCK_K, m0);
          tma_load_2d(sa + Cfg::kABytes, tmB, &full_bar[stage], kb * GEMM_BLOCK_K, c0);
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA warpgroup wg: the cluster's tiles wg, wg + 2, ... (ping-pong) =====================
    setmaxnreg_inc<232>();                              // 96 accumulators, and the epilogue's state next to them
    const int wg = (threadIdx.x >> 7) - 1;
    const bool parts4 = p.K >= GLN_PARTS4_MIN_K;
    const bool leader = (threadIdx.x & 127) == 0;
    uint8_t* xw = xs + wg * Cfg::kXBytes;
    int stage = 0;
    uint32_t phase = 0, par = 0;
    if (wg == 1) ring_advance(stage, phase, num_kb, Cfg::kStages);   // tile 0 belongs to warpgroup 0
#pragma unroll 1
    for (int tile = cluster + wg * clusters; tile < p.num_m_tiles; tile += 2 * clusters) {
      const int m0 = tile * Cfg::kTileM;
      // ordered main loops: wait until the other warpgroup has issued every MMA of the cluster's previous tile
      if (tile != cluster) named_bar_sync(1 + wg, 256);
      float acc[Cfg::kCols / 2];
#pragma unroll
      for (int i = 0; i < Cfg::kCols / 2; ++i) acc[i] = 0.0f;
      int prev = -1;
#pragma unroll 1
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_mma(&full_bar[stage], phase);
        const uint32_t base = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint64_t da = make_desc_k_sw128(base);
        const uint64_t db = make_desc_k_sw128(base + Cfg::kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)
          wgmma_bf16<Cfg::kCols>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                                 static_cast<uint32_t>((kb | k) != 0));
        wgmma_commit();
        if (prev >= 0) {                                 // the MMAs of this k-block are queued: free the previous stage
          wgmma_wait<1>();
          if (leader) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
      }
      if (tile + clusters < p.num_m_tiles) named_bar_arrive(1 + (wg ^ 1), 256);   // the other warpgroup may start its main loop
      wgmma_wait<0>();
      wgmma_reg_fence(acc);
      if (leader) mbar_arrive(&empty_bar[prev]);
      ring_advance(stage, phase, num_kb, Cfg::kStages);            // skip the other warpgroup's next tile
      mbar_wait_mma(&x_full[wg], par);
      if (parts4)
        gln_pair_epilogue<D, 4>(acc, xw, x, xn, p.M, p.eps, m0, c0, rank, s_bias, s_gamma, s_beta,
                                s_part + wg * 2 * 4 * GLN_BLOCK_M, stat_bar + 2 * wg, par, &x_empty[wg]);
      else
        gln_pair_epilogue<D, 2>(acc, xw, x, xn, p.M, p.eps, m0, c0, rank, s_bias, s_gamma, s_beta,
                                s_part + wg * 2 * 4 * GLN_BLOCK_M, stat_bar + 2 * wg, par, &x_empty[wg]);
      par ^= 1u;
    }
  }
  // a CTA of a pair must not exit while its peer may still write to its shared memory or arrive on its barriers
  cluster_sync_all();
}

template <int D, int MODE>
__global__ void __launch_bounds__(GLN_THREADS, 1)
gemm_ln_fused_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmX, float* __restrict__ x, __nv_bfloat16* __restrict__ xn,
                     const GemmLnParams p) {
  if constexpr (MODE == 2) {
    gln_pair_persistent<D>(&tmA, &tmB, &tmX, x, xn, p);
  } else {
    // tmX is used by MODE 2 only
    using Cfg = GemmLnCfg<D, MODE>;
    constexpr int kNW = Cfg::kNW;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw_addr = smem_u32(smem_raw);
    const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
    uint8_t* smem = smem_raw + pad;
    float* s_bias = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
    float* s_gamma = s_bias + Cfg::kCols;
    float* s_beta = s_gamma + Cfg::kCols;
    float* s_part = s_beta + Cfg::kCols;               // [2 rounds][kParts][64 rows]
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_bias) + Cfg::kParamBytes);
    uint64_t* empty_bar = full_bar + Cfg::kStages;

    const uint32_t rank = (MODE == 1) ? cluster_ctarank() : 0u;
    const int cluster = blockIdx.x / Cfg::kCG;
    const int m0 = cluster * Cfg::kTileM + static_cast<int>(rank) * GLN_BLOCK_M;
    const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;

    grid_dep_launch();
    if (threadIdx.x == 0) {
      prefetch_tmap(&tmA);
      prefetch_tmap(&tmB);
      for (int s = 0; s < Cfg::kStages; ++s) {
        mbar_init(&full_bar[s], 1);
        mbar_init(&empty_bar[s], MODE == 1 ? 4 : 2);
      }
      fence_mbar_init();
    }
    // bias / gamma / beta are weights (never written by a preceding kernel): stage them before the dependency wait
    for (int j = threadIdx.x; j < Cfg::kCols; j += GLN_THREADS) {
      s_bias[j] = (p.bias != nullptr) ? __ldg(p.bias + j) : 0.0f;
      s_gamma[j] = __ldg(p.gamma + j);
      s_beta[j] = __ldg(p.beta + j);
    }
    if constexpr (MODE == 1) cluster_sync_all(); else __syncthreads();
    grid_dep_wait();

    if (threadIdx.x < 128) {
      // ===================== TMA producer =====================
      if (threadIdx.x == 0) {
        int stage = 0;
        uint32_t phase = 0;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * GEMM_BLOCK_K, m0);
          if constexpr (MODE == 1) {
            const int r = static_cast<int>(rank);
            tma_load_2d_mcast(sb + r * Cfg::kLoadRows * GEMM_BLOCK_K * 2, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K,
                              r * Cfg::kLoadRows, 0x3);
          } else {
#pragma unroll
            for (int b = 0; b < Cfg::kLoadRows / Cfg::kBox; ++b)
              tma_load_2d(sb + b * Cfg::kBox * GEMM_BLOCK_K * 2, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K, b * Cfg::kBox);
          }
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
        }
      }
      __syncwarp();
    } else {
      // ===================== MMA warpgroups: columns [kNW wg, kNW wg + kNW) =====================
      const int wg = (threadIdx.x >> 7) - 1;
      float acc[kNW / 2];
#pragma unroll
      for (int i = 0; i < kNW / 2; ++i) acc[i] = 0.0f;
      int stage = 0;
      uint32_t phase = 0;
      wg_mainloop<kNW, MODE == 1>(acc, smem, Cfg::kStageBytes, 0, Cfg::kABytes + wg * kNW * GEMM_BLOCK_K * 2, full_bar,
                                  empty_bar, Cfg::kStages, num_kb, stage, phase);
      gln_epilogue<D, kNW>(acc, x, xn, p.M, p.eps, m0, wg, s_bias, s_gamma, s_beta, s_part);
    }
    // a CTA of a pair must not exit while its peer may still write to its shared memory or arrive on its barriers
    if constexpr (MODE == 1) cluster_sync_all();
  }
}

}  // namespace pq
