// ViT attention with its QKV projection in one persistent kernel (sm_90a, wgmma + TMA + mma.sync), T = 128 tokens,
// head_dim 64, D = 64 heads in {192, 384}:
//   att[b, :, 64h .. 64h + 64) = attention(Q_h, K_h, V_h),  [Q_h | K_h | V_h] = bf16(xn_b W_h^T + b_h)
// where xn_b is image b's 128 x D tile and W_h the 192 rows 64h.., D + 64h.., 2D + 64h.. of attn.qkv.weight.
//
// Why: as two kernels the QKV GEMM writes the 3 D-wide qkv tensor to HBM and the attention kernel reads it back (2 x 151
// MB per ViT block of PARSeq-S at bs = 512).  At T = 128 one image is one 128-row tile and one head's Q/K/V (48 KB) fits
// in shared memory, so the qkv tensor never has to leave the SM.
//
// Work items are (image, head), numbered image-major (the heads of one image run on neighbouring CTAs at the same time
// and share its xn tile through L2); a grid of at most one CTA per SM walks them with the grid's stride.
// Warpgroup 0 is the TMA producer: per item and k-block one stage of the operand ring holds the image's 128 x 64 xn box
// and the head's three 64 x 64 W boxes back to back (one 192-row K-major operand, 128B swizzle).  It runs ahead into the
// next item's k-blocks while the current item is in its epilogue and attention.  Warpgroups 1 and 2 each accumulate 64
// rows x 192 columns (wgmma m64n192k16, the k order of gemm_bf16_wgmma_kernel), add the bias, round to bf16 into the
// shared Q/K/V tiles, and then run the attention of the item as enc_attention_kernel's 8 warps (att_tile_128).
//
// Bit-identical to gemm_bf16_wgmma_kernel<EPI_BF16> followed by enc_attention_kernel: the same bf16 operands, the same
// k order, the same epilogue ((acc + bias) * 1, rounded to bf16) and the same attention code.
#pragma once
#include "gemm.cuh"
#include "kernels.cuh"

namespace pq {

constexpr int QA_THREADS = 384;   // warpgroup 0: TMA producer; warpgroups 1, 2: QKV MMAs + attention (8 warps)

struct QkvAttnCfg {
  static constexpr int kABytes = ATT_T * GEMM_BLOCK_K * 2;        // 16 KB: 128 rows of xn
  static constexpr int kWBoxBytes = ATT_DH * GEMM_BLOCK_K * 2;    // 8 KB: 64 rows of W (one of Q, K, V)
  static constexpr int kStageBytes = kABytes + 3 * kWBoxBytes;    // 40 KB
  static constexpr int kTileBytes = ATT_T * ATT_DH * 2;           // 16 KB: one of the shared Q, K, V tiles
  static constexpr int kStages = 4;                               // D = 384: 4 of the next item's 6 k-blocks in flight
  static constexpr int kSmemBytes = kStages * kStageBytes + 3 * kTileBytes + 1024 /*align slack*/ + 256 /*barriers*/;
};
static_assert(QkvAttnCfg::kSmemBytes <= 232448, "shared memory");

template <int D>
__global__ void __launch_bounds__(QA_THREADS, 1)
enc_qkv_attn_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                    const float* __restrict__ bias, __nv_bfloat16* __restrict__ out, int num_items) {
  static_assert(D == 192 || D == 384, "embed_dim");
  using Cfg = QkvAttnCfg;
  constexpr int kHeads = D / ATT_DH;
  constexpr int kNumKb = D / GEMM_BLOCK_K;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;                          // 1024-B aligned (SWIZZLE_128B requirement)
  __nv_bfloat16* sQ = reinterpret_cast<__nv_bfloat16*>(smem + Cfg::kStages * Cfg::kStageBytes);
  __nv_bfloat16* sK = sQ + ATT_T * ATT_DH;
  __nv_bfloat16* sV = sK + ATT_T * ATT_DH;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sV + ATT_T * ATT_DH);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int n_local = (num_items - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1;  // grid <= items

  grid_dep_launch();                       // PDL: the next kernel may start its own prologue
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2);         // both MMA warpgroups read every stage
    }
    fence_mbar_init();
  }
  __syncthreads();
  grid_dep_wait();                         // PDL: xn is complete and visible, att is no longer read, from here on

  if (threadIdx.x < 128) {
    // ===================== TMA producer: the CTA's items in order, running ahead across items =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_local; ++j) {
        const int item = static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x);
        const int m0 = (item / kHeads) * ATT_T, h = item % kHeads;
        for (int kb = 0; kb < kNumKb; ++kb) {
          mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmX, &full_bar[stage], kb * GEMM_BLOCK_K, m0);
#pragma unroll
          for (int m = 0; m < 3; ++m)      // the Q, K and V rows of head h
            tma_load_2d(sa + Cfg::kABytes + m * Cfg::kWBoxBytes, &tmW, &full_bar[stage], kb * GEMM_BLOCK_K,
                        m * D + h * ATT_DH);
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== MMA + attention: warpgroup wg holds rows [64 wg, 64 wg + 64) of every item =====================
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int lane = threadIdx.x & 31;
    const int warp = (threadIdx.x >> 5) - 4;                 // 0..7 over both warpgroups
    const int r0 = 64 * wg + 16 * (warp & 3) + (lane >> 2);   // accumulator rows r0, r0 + 8 of the item's tile
    int stage = 0;
    uint32_t phase = 0;
#pragma unroll 1
    for (int j = 0; j < n_local; ++j) {
      const int item = static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x);
      const int b = item / kHeads, h = item % kHeads;
      float acc[3 * ATT_DH / 2];
#pragma unroll
      for (int i = 0; i < 3 * ATT_DH / 2; ++i) acc[i] = 0.0f;
      wg_mainloop<3 * ATT_DH, false>(acc, smem, Cfg::kStageBytes, wg * (Cfg::kABytes / 2), Cfg::kABytes, full_bar,
                                     empty_bar, Cfg::kStages, kNumKb, stage, phase);
      // ---- epilogue: bf16(acc + bias) into the Q / K / V tiles.  Accumulator layout (ptx.cuh wgmma_bf16): acc[4i + {0,1}]
      // = row r0, columns 8i + 2(lane%4) + {0,1}; acc[4i + {2,3}] = row r0 + 8.  Columns [64m, 64m + 64) are matrix m.
      if (j > 0) named_bar_sync(1, 256);   // every warp has finished the previous item's attention
#pragma unroll
      for (int i = 0; i < 3 * ATT_DH / 8; ++i) {
        const int m = i / 8, c = (i % 8) * 8 + 2 * (lane & 3);
        const int col = m * D + h * ATT_DH + c;
        const float b0 = bias != nullptr ? __ldg(bias + col) : 0.0f;
        const float b1 = bias != nullptr ? __ldg(bias + col + 1) : 0.0f;
        __nv_bfloat16* dst = m == 0 ? sQ : m == 1 ? sK : sV;
        *reinterpret_cast<uint32_t*>(dst + att_swz(r0, c)) =
            pack_bf16(gemm_epi<EPI_BF16>(acc[4 * i], b0, 1.0f), gemm_epi<EPI_BF16>(acc[4 * i + 1], b1, 1.0f));
        *reinterpret_cast<uint32_t*>(dst + att_swz(r0 + 8, c)) =
            pack_bf16(gemm_epi<EPI_BF16>(acc[4 * i + 2], b0, 1.0f), gemm_epi<EPI_BF16>(acc[4 * i + 3], b1, 1.0f));
      }
      named_bar_sync(1, 256);              // every query row needs all 128 keys of both warpgroups
      att_tile_128(sQ, sK, sV, out + static_cast<long long>(b) * ATT_T * D + h * ATT_DH, D, warp, lane);
    }
  }
}

}  // namespace pq
