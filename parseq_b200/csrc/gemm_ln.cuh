// Residual GEMM fused with the LayerNorm that follows it (sm_90a, wgmma + TMA).
//
//   x[M, D]  (fp32, in place)  <-  x + A[M, K] * W[D, K]^T + bias            (timm Block: x = x + attn(..) / mlp(..))
//   xn[M, D] (bf16)            <-  LayerNorm(x_new; gamma, beta, eps)         (norm2 / next block's norm1 / final norm)
//
// Why: as separate kernels the attention-projection and fc2 GEMMs are bound by the fp32 read-modify-write of the
// residual stream and the LayerNorm re-reads it from HBM; here each updated row is normalised while it is still in
// registers.
//
// A CTA owns 64 rows.  Warpgroup 0 is the TMA producer; warpgroups 1 and 2 each accumulate half of the CTA's columns
// for all 64 rows (wgmma m64 x N x k16), so a row's values sit in two warpgroups (and, for MODE 2, two CTAs):
//   pass 1: v = (acc + bias) + x is stored back to x and kept in the accumulator registers; row sums are reduced over
//           the quad of lanes that holds a row, then over the column parts through shared memory;
//   pass 2: the same for the squared deviations from the mean (two-pass variance, as layernorm_kernel);
//   pass 3: normalise, pack to bf16, store xn.
// Rounding points are those of the unfused pair (residual-accumulate GEMM epilogue + layernorm_kernel): fp32 x, bf16 xn.
//
// MODE 0: one CTA per 64-row tile, all D columns.
// MODE 1: a cluster of two CTAs on 128 rows; each CTA loads half of the W tile and multicasts it into both, so every W
//         byte is fetched once per 128 rows.  Same work per row as MODE 0: bit-identical results.
// MODE 2: a cluster of two CTAs on 64 rows, each CTA computing half of the columns (half of W per CTA, a ring twice as
//         deep); the row statistics of the four column parts are exchanged through distributed shared memory.
#pragma once
#include "gemm.cuh"

namespace pq {

struct GemmLnParams {
  int M, K;
  const float* bias;     // [D] or nullptr
  const float* gamma;    // [D]
  const float* beta;     // [D]
  float eps;
  int num_m_tiles;       // clusters (MODE 1 / 2) or CTAs (MODE 0)
};

constexpr int GLN_THREADS = 384;
constexpr int GLN_BLOCK_M = 64;

template <int D, int MODE>
struct GemmLnCfg {
  static_assert(MODE >= 0 && MODE <= 2, "MODE");
  static constexpr int kCG = MODE == 0 ? 1 : 2;                       // CTAs per cluster
  static constexpr int kCols = MODE == 2 ? D / 2 : D;                 // columns per CTA
  static constexpr int kNW = kCols / 2;                               // columns per MMA warpgroup
  static constexpr int kParts = MODE == 2 ? 4 : 2;                    // column parts of a row
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

// Sum of one row's column parts, in a fixed order (every thread of every CTA that holds the row gets the same bits).
template <int PARTS>
__device__ __forceinline__ float gln_row_total(const float* s_part, int r) {
  float t = s_part[r] + s_part[GLN_BLOCK_M + r];
  if constexpr (PARTS == 4) t += s_part[2 * GLN_BLOCK_M + r] + s_part[3 * GLN_BLOCK_M + r];
  return t;
}

// Epilogue shared by the fused kernels (this file, mlp_ln.cuh): `acc` holds the 64 x NW block of one MMA warpgroup
// (rows m0.., columns c0 + wg * NW..); x += acc + bias in place, then xn = bf16(LayerNorm(x)) over the D columns of a row,
// whose PARTS column parts are combined through s_part (and, for SPLIT, through the peer CTA's s_part: stat_bar).
template <int D, int NW, int PARTS, bool SPLIT>
__device__ __forceinline__ void gln_epilogue(float (&acc)[NW / 2], float* __restrict__ x, __nv_bfloat16* __restrict__ xn, int M,
                                             float eps, int m0, int c0, int wg, uint32_t rank, const float* s_bias,
                                             const float* s_gamma, const float* s_beta, float* s_part, uint64_t* stat_bar) {
  constexpr int kNW = NW;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int lr = (t >> 5) * 16 + (lane >> 2);        // local rows lr, lr + 8
  const bool ok_a = m0 + lr < M, ok_b = m0 + lr + 8 < M;
  float* xa = x + static_cast<long long>(m0 + lr) * D + c0 + wg * kNW + 2 * (lane & 3);
  float* xb = xa + 8ll * D;
  const int part = (SPLIT ? static_cast<int>(rank) * 2 : 0) + wg;
  const uint32_t peer = rank ^ 1u;

  // pass 1: residual update, row sums
  float sa = 0.f, sb = 0.f;
#pragma unroll
  for (int i = 0; i < kNW / 8; ++i) {
    const int cl = wg * kNW + i * 8 + 2 * (lane & 3);   // column inside this CTA's part
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
    float* slot = s_part + (round * PARTS + part) * GLN_BLOCK_M;
    if ((lane & 3) == 0) {
      slot[lr] = sa;
      slot[lr + 8] = sb;
      if constexpr (SPLIT) {
        st_cluster_f32(mapa_cluster(smem_u32(slot + lr), peer), sa);
        st_cluster_f32(mapa_cluster(smem_u32(slot + lr + 8), peer), sb);
      }
    }
    if constexpr (SPLIT) {
      mbar_arrive(&stat_bar[round]);
      mbar_arrive_cluster(mapa_cluster(smem_u32(&stat_bar[round]), peer));
      mbar_wait_cluster(&stat_bar[round], 0);
    } else {
      asm volatile("bar.sync 1, 256;" ::: "memory");   // the two MMA warpgroups
    }
    const float* tot = s_part + round * PARTS * GLN_BLOCK_M;
    const float ta = gln_row_total<PARTS>(tot, lr), tb = gln_row_total<PARTS>(tot, lr + 8);
    if (round == 0) {
      mean_a = ta * (1.0f / D);
      mean_b = tb * (1.0f / D);
    } else {
      rstd_a = 1.0f / sqrtf(ta * (1.0f / D) + eps);
      rstd_b = 1.0f / sqrtf(tb * (1.0f / D) + eps);
    }
  }
  // pass 3: normalise, bf16
  uint32_t* na = reinterpret_cast<uint32_t*>(xn + static_cast<long long>(m0 + lr) * D + c0 + wg * kNW + 2 * (lane & 3));
  uint32_t* nb = na + 4ll * D;
#pragma unroll
  for (int i = 0; i < kNW / 8; ++i) {
    const int cl = wg * kNW + i * 8 + 2 * (lane & 3);
    const float g0 = s_gamma[cl], g1 = s_gamma[cl + 1], e0 = s_beta[cl], e1 = s_beta[cl + 1];
    if (ok_a) na[i * 4] = pack_bf16((acc[4 * i] - mean_a) * rstd_a * g0 + e0, (acc[4 * i + 1] - mean_a) * rstd_a * g1 + e1);
    if (ok_b) nb[i * 4] = pack_bf16((acc[4 * i + 2] - mean_b) * rstd_b * g0 + e0, (acc[4 * i + 3] - mean_b) * rstd_b * g1 + e1);
  }
}

template <int D, int MODE>
__global__ void __launch_bounds__(GLN_THREADS, 1)
gemm_ln_fused_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     float* __restrict__ x, __nv_bfloat16* __restrict__ xn, const GemmLnParams p) {
  using Cfg = GemmLnCfg<D, MODE>;
  constexpr int kNW = Cfg::kNW;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;
  float* s_bias = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  float* s_gamma = s_bias + Cfg::kCols;
  float* s_beta = s_gamma + Cfg::kCols;
  float* s_part = s_beta + Cfg::kCols;                 // [2 rounds][kParts][64 rows]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_bias) + Cfg::kParamBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  uint64_t* stat_bar = empty_bar + Cfg::kStages;       // [2 rounds] (MODE 2): the partials of both CTAs have landed

  const uint32_t rank = (MODE != 0) ? cluster_ctarank() : 0u;
  const int cluster = blockIdx.x / Cfg::kCG;
  const int m0 = (MODE == 1) ? cluster * 2 * GLN_BLOCK_M + static_cast<int>(rank) * GLN_BLOCK_M : cluster * GLN_BLOCK_M;
  const int c0 = (MODE == 2) ? static_cast<int>(rank) * Cfg::kCols : 0;   // first column of this CTA
  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;

  grid_dep_launch();
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], MODE == 1 ? 4 : 2);
    }
    mbar_init(&stat_bar[0], 2 * 256);                  // every MMA thread of both CTAs
    mbar_init(&stat_bar[1], 2 * 256);
    fence_mbar_init();
  }
  // bias / gamma / beta are weights (never written by a preceding kernel): stage them before the dependency wait
  for (int j = threadIdx.x; j < Cfg::kCols; j += GLN_THREADS) {
    s_bias[j] = (p.bias != nullptr) ? __ldg(p.bias + c0 + j) : 0.0f;
    s_gamma[j] = __ldg(p.gamma + c0 + j);
    s_beta[j] = __ldg(p.beta + c0 + j);
  }
  if constexpr (MODE != 0) cluster_sync_all(); else __syncthreads();
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
            tma_load_2d(sb + b * Cfg::kBox * GEMM_BLOCK_K * 2, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K, c0 + b * Cfg::kBox);
        }
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA warpgroups: columns [kNW wg, kNW wg + kNW) of this CTA's part =====================
    const int wg = (threadIdx.x >> 7) - 1;
    float acc[kNW / 2];
#pragma unroll
    for (int i = 0; i < kNW / 2; ++i) acc[i] = 0.0f;
    int stage = 0;
    uint32_t phase = 0;
    wg_mainloop<kNW, MODE == 1>(acc, smem, Cfg::kStageBytes, 0, Cfg::kABytes + wg * kNW * GEMM_BLOCK_K * 2, full_bar,
                                empty_bar, Cfg::kStages, num_kb, stage, phase);
    gln_epilogue<D, kNW, Cfg::kParts, MODE == 2>(acc, x, xn, p.M, p.eps, m0, c0, wg, rank, s_bias, s_gamma, s_beta, s_part,
                                                stat_bar);
  }
  // a CTA of a pair must not exit while its peer may still write to its shared memory or arrive on its barriers
  if constexpr (MODE != 0) cluster_sync_all();
}

}  // namespace pq
