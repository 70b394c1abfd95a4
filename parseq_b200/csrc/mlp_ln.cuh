// The whole MLP of a timm Block + the LayerNorm that follows it in one kernel (sm_90a, wgmma + TMA):
//
//   x[M, D]  (fp32, in place)  <-  x + GELU(xn W1^T + b1) W2^T + b2        (H = 4 D hidden columns)
//   xn_out   (bf16)            <-  LayerNorm(x_new; gamma, beta, eps)      (may alias xn)
//
// A CTA owns 64 rows; their xn tile stays in shared memory for the whole kernel.  The hidden activation never reaches
// HBM: it is produced 64 columns at a time (fc1: each MMA warpgroup computes 32 of them, GELU, bf16, into a swizzled
// shared-memory chunk, double-buffered) and consumed at once as one 64-wide k-block of fc2, whose accumulators (each
// warpgroup half of the D output columns) live in registers across all H / 64 chunks.  The weights stream through one
// TMA ring in a fixed order: per chunk, the D / 64 k-blocks of its W1 rows, then the two column halves of its W2 block.
// Same k order and rounding points as the two-kernel path (GEMM with the GELU epilogue, then gemm_ln.cuh MODE 0):
// bit-identical results.
//
// CG = 2: a cluster of two CTAs on 128 rows; each CTA loads half of every weight box and multicasts it into both.
#pragma once
#include "gemm_ln.cuh"

namespace pq {

struct MlpLnParams {
  int M;
  const float* b1;       // [4D]
  const float* b2;       // [D]
  const float* gamma;    // [D]
  const float* beta;     // [D]
  float eps;
  int num_m_tiles;       // clusters of CG CTAs
};

constexpr int MLP_THREADS = 384;

template <int D, int CG>
struct MlpLnCfg {
  static constexpr int kH = 4 * D;
  static constexpr int kKC = D / 64;                                  // fc1 k-blocks per hidden chunk
  static constexpr int kChunks = kH / 64;                             // hidden chunks = fc2 k-blocks
  static constexpr int kW1Rows = 64 / CG;                             // W1 box rows loaded by one CTA
  static constexpr int kW2Rows = D / 2 / CG;                          // W2 box rows loaded by one CTA
  static constexpr int kW1Bytes = 64 * 64 * 2;
  static constexpr int kW2Bytes = (D / 2) * 64 * 2;
  static constexpr int kSlotBytes = kW2Bytes > kW1Bytes ? kW2Bytes : kW1Bytes;
  static constexpr int kXsBytes = kKC * 64 * 64 * 2;                  // the CTA's xn rows
  static constexpr int kHidBytes = 2 * 64 * 64 * 2;                   // two hidden chunks
  static constexpr int kParamBytes = (kH + 3 * D) * 4 + 2 * 2 * GLN_BLOCK_M * 4;   // b1, b2, gamma, beta; row partials
  static constexpr int kBarBytes = 256;
  static constexpr int kStagesRaw = (232448 - 1024 - kBarBytes - kXsBytes - kHidBytes - kParamBytes) / kSlotBytes;
  static constexpr int kStages = kStagesRaw > 8 ? 8 : kStagesRaw;
  static constexpr int kSmemBytes = kXsBytes + kHidBytes + kStages * kSlotBytes + kParamBytes + kBarBytes + 1024;
  static_assert(D == 192 || D == 384, "embed_dim");
  static_assert((kW1Rows * 128) % 1024 == 0 && (kW2Rows * 128) % 1024 == 0 && kSlotBytes % 1024 == 0, "1024-B aligned boxes");
  static_assert(kStages >= 4, "pipeline depth");
};

template <int D, int CG>
__global__ void __launch_bounds__(MLP_THREADS, 1)
mlp_ln_fused_kernel(const __grid_constant__ CUtensorMap tmXn, const __grid_constant__ CUtensorMap tmW1,
                    const __grid_constant__ CUtensorMap tmW2, float* __restrict__ x, __nv_bfloat16* __restrict__ xn_out,
                    const MlpLnParams p) {
  using Cfg = MlpLnCfg<D, CG>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* xs = smem_raw + pad;                                       // [kKC][64 rows][128 B], 1024-B aligned
  uint8_t* hid = xs + Cfg::kXsBytes;                                  // [2][64 rows][128 B]
  uint8_t* ring = hid + Cfg::kHidBytes;
  float* s_b1 = reinterpret_cast<float*>(ring + Cfg::kStages * Cfg::kSlotBytes);
  float* s_b2 = s_b1 + Cfg::kH;
  float* s_gamma = s_b2 + D;
  float* s_beta = s_gamma + D;
  float* s_part = s_beta + D;                                         // [2 rounds][2 parts][64 rows]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_b1) + Cfg::kParamBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;
  uint64_t* xs_bar = empty_bar + Cfg::kStages;

  const uint32_t rank = (CG == 2) ? cluster_ctarank() : 0u;
  const int m0 = (blockIdx.x / CG) * (GLN_BLOCK_M * CG) + static_cast<int>(rank) * GLN_BLOCK_M;

  grid_dep_launch();
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmXn);
    prefetch_tmap(&tmW1);
    prefetch_tmap(&tmW2);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CG);
    }
    mbar_init(xs_bar, 1);
    fence_mbar_init();
  }
  for (int j = threadIdx.x; j < Cfg::kH; j += MLP_THREADS) s_b1[j] = __ldg(p.b1 + j);
  for (int j = threadIdx.x; j < D; j += MLP_THREADS) {
    s_b2[j] = __ldg(p.b2 + j);
    s_gamma[j] = __ldg(p.gamma + j);
    s_beta[j] = __ldg(p.beta + j);
  }
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
  grid_dep_wait();

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    if (threadIdx.x == 0) {
      mbar_expect_tx(xs_bar, Cfg::kXsBytes);
      for (int c = 0; c < Cfg::kKC; ++c) tma_load_2d(xs + c * 8192, &tmXn, xs_bar, c * 64, m0);
      const int r = static_cast<int>(rank);
      int stage = 0;
      uint32_t phase = 0;
      auto next_slot = [&](int bytes) -> uint8_t* {
        mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
        mbar_expect_tx(&full_bar[stage], bytes);
        return ring + stage * Cfg::kSlotBytes;
      };
      auto advance = [&]() { if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; } };
      for (int j = 0; j < Cfg::kChunks; ++j) {
        for (int c = 0; c < Cfg::kKC; ++c) {                         // W1 rows [64 j, 64 j + 64), k-block c
          uint8_t* dst = next_slot(Cfg::kW1Bytes) + r * Cfg::kW1Rows * 128;
          if constexpr (CG == 2) tma_load_2d_mcast(dst, &tmW1, &full_bar[stage], c * 64, j * 64 + r * Cfg::kW1Rows, 0x3);
          else tma_load_2d(dst, &tmW1, &full_bar[stage], c * 64, j * 64);
          advance();
        }
        for (int h = 0; h < 2; ++h) {                                  // W2 rows [h D/2, (h+1) D/2), k-block j
          uint8_t* dst = next_slot(Cfg::kW2Bytes) + r * Cfg::kW2Rows * 128;
          if constexpr (CG == 2)
            tma_load_2d_mcast(dst, &tmW2, &full_bar[stage], j * 64, h * (D / 2) + r * Cfg::kW2Rows, 0x3);
          else tma_load_2d(dst, &tmW2, &full_bar[stage], j * 64, h * (D / 2));
          advance();
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA warpgroups =====================
    const int wg = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    const int lane = t & 31;
    const bool signal = t == 0;
    int stage = 0;
    uint32_t phase = 0;
    auto release = [&]() {
      if (signal) {
        mbar_arrive(&empty_bar[stage]);
        if constexpr (CG == 2) mbar_arrive_cluster(mapa_cluster(smem_u32(&empty_bar[stage]), rank ^ 1u));
      }
      if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
    };
    float acc[D / 4];                                                  // fc2: 64 rows x D/2 columns of this warpgroup
#pragma unroll
    for (int i = 0; i < D / 4; ++i) acc[i] = 0.0f;
    mbar_wait_mma(xs_bar, 0);
#pragma unroll 1
    for (int j = 0; j < Cfg::kChunks; ++j) {
      // ---- fc1: hidden columns [64 j + 32 wg, +32) ----
      float h1[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) h1[i] = 0.0f;
#pragma unroll 1
      for (int c = 0; c < Cfg::kKC; ++c) {
        mbar_wait_mma(&full_bar[stage], phase);
        const uint64_t da = make_desc_k_sw128(smem_u32(xs + c * 8192));
        const uint64_t db = make_desc_k_sw128(smem_u32(ring + stage * Cfg::kSlotBytes + wg * 32 * 128));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_bf16<32>(h1, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), static_cast<uint32_t>((c | k) != 0));
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(h1);
        release();
      }
      // bias + GELU + bf16 (the GEMM's EPI_GELU_BF16 epilogue) into the swizzled hidden chunk j & 1
      uint8_t* hb = hid + (j & 1) * 8192;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int col = wg * 32 + i * 8 + 2 * (lane & 3);              // column inside the chunk
        const float b0 = s_b1[j * 64 + col], b1 = s_b1[j * 64 + col + 1];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int row = (t >> 5) * 16 + (lane >> 2) + hr * 8;
          const uint32_t v = pack_bf16(gelu_erf(h1[4 * i + 2 * hr] + b0), gelu_erf(h1[4 * i + 2 * hr + 1] + b1));
          *reinterpret_cast<uint32_t*>(hb + row * 128 + ((static_cast<uint32_t>(col >> 3) ^ static_cast<uint32_t>(row & 7)) << 4) +
                                       (col & 7) * 2) = v;
        }
      }
      fence_proxy_async_smem();                                        // generic stores -> wgmma operand reads
      asm volatile("bar.sync 1, 256;" ::: "memory");                   // both halves of the chunk are in place
      // ---- fc2: k-block j, this warpgroup's W2 column half (the other half's slot is released unread) ----
      const uint64_t da = make_desc_k_sw128(smem_u32(hb));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        mbar_wait_mma(&full_bar[stage], phase);
        if (h == wg) {
          const uint64_t db = make_desc_k_sw128(smem_u32(ring + stage * Cfg::kSlotBytes));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_bf16<D / 2>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                              static_cast<uint32_t>((j | k) != 0));
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_reg_fence(acc);
        }
        release();
      }
    }
    gln_epilogue<D, D / 2>(acc, x, xn_out, p.M, p.eps, m0, wg, s_b2, s_gamma, s_beta, s_part);
  }
  // a CTA of a pair must not exit while its peer may still multicast into it or arrive on its barriers
  if constexpr (CG == 2) cluster_sync_all();
}

}  // namespace pq
