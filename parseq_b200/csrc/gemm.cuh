// Persistent warp-specialised bf16 GEMM on wgmma (sm_90a):
//   out[M,N] = epilogue( A[M,K] * W[N,K]^T + bias )
// A and W are bf16, K-contiguous ("K-major"); both are fetched by TMA into 128B-swizzled shared-memory stages of an
// mbarrier ring.  Warpgroup 0 is the producer (one thread issues the TMA loads); warpgroups 1 and 2 each accumulate 64
// rows of the 128 x BLOCK_N tile in registers with wgmma (m64 x BLOCK_N x k16) and store their rows straight from the
// accumulator.  A CTA (pair) walks the tiles with a stride of the grid; the ring position carries over, so the producer
// loads the next tile's operands while the MMA warpgroups run the epilogue of the current one.  Every projection of the PARSeq path goes through this kernel: patch-embed (K=96), QKV / proj / fc1 / fc2
// of the 12 ViT blocks (reference: timm Attention/Mlp via strhub/models/parseq/modules.py:145-165), the
// cross-attention K/V projection of the image memory, the decoder's q / out projections, MLP (modules.py:69-77) and
// the character head (model.py:63).
#pragma once
#include <cuda.h>
#include "ptx.cuh"

namespace pq {

enum GemmEpilogue : int {
  EPI_F32 = 0,        // out_f32 = alpha*(acc+bias) (+ resid[row or row%resid_mod])
  EPI_BF16 = 1,       // out_bf16 = bf16(alpha*(acc+bias))
  EPI_GELU_BF16 = 2,  // out_bf16 = bf16(gelu(acc+bias))
};

struct GemmParams {
  int M, N, K;
  int mode;
  float alpha;
  const float* bias;   // [N] or nullptr
  const float* resid;  // fp32 residual (may alias out: in-place accumulate) or nullptr
  long long ldr;
  int resid_mod;       // >0: residual row = row % resid_mod (broadcast tables: pos_embed, pos_queries)
  void* out;
  long long ldo;       // elements
  int vec_ok;          // 8-byte aligned column pairs: paired stores allowed
  long long blocked_rows;  // > 0: bf16 output in a column-blocked buffer [N/64][blocked_rows][64] (ldo unused)
  int num_m_tiles, num_n_tiles;  // in units of (128 * CG) x BLOCK_N
  int max_stages;                // 0: the full operand ring; n > 0: use only n slots (pipeline-depth experiments)
};

constexpr int GEMM_BLOCK_M = 128;  // rows per CTA (64 per MMA warpgroup)
constexpr int GEMM_BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int GEMM_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1, 2: MMA + epilogue

// CG = 1: one CTA computes a 128 x BLOCK_N tile.
// CG = 2: a cluster of two CTAs computes a 256 x BLOCK_N tile: each CTA loads its own 128 rows of A and HALF of the W
//         tile, multicast into both CTAs, so every W byte is fetched from L2 once per 256 (instead of 128) output rows.
template <int BLOCK_N, int CG>
struct GemmCfg {
  static constexpr int kBRows = BLOCK_N / CG;                       // W rows loaded by one CTA
  static constexpr int kABytes = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;   // 16 KB
  static constexpr int kBBytes = BLOCK_N * GEMM_BLOCK_K * 2;        // the whole W tile lands in every CTA
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStagesRaw = (232448 - 1024 - 256) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 6 ? 6 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(BLOCK_N == 64 || BLOCK_N == 128 || BLOCK_N == 192 || BLOCK_N == 256, "BLOCK_N");
  static_assert(CG == 1 || CG == 2, "CG");
  static_assert((kBRows * GEMM_BLOCK_K * 2) % 1024 == 0, "multicast halves must stay 1024-B aligned");
  static_assert(kStages >= 3, "pipeline depth");
};

// ------------------------------------------------------------------------------------------------ operand ring
// full[s]: stage s holds its A and B tiles (TMA transaction bytes).  empty[s]: every MMA warpgroup that reads stage s
// has finished with it - in both CTAs of a pair when B is multicast (2 warpgroups x CG arrivals).
//
// Consumer side of the ring for one warpgroup: accumulates a 64 x N block over num_kb k-blocks.  a_off / b_off: byte
// offsets of the warpgroup's A rows / B rows inside a stage; stage / phase: the ring position, carried over from tile to
// tile.  A stage is released once the MMAs of the NEXT k-block are queued (wgmma_wait<1>), so the tensor cores never wait
// for the release round trip; the last one once the accumulator is complete.  Hence a ring needs at least two stages.
template <int N, bool PAIR>
__device__ __forceinline__ void wg_mainloop(float (&acc)[N / 2], uint8_t* smem, int stage_bytes, int a_off, int b_off,
                                            uint64_t* full_bar, uint64_t* empty_bar, int nstages, int num_kb, int& stage,
                                            uint32_t& phase) {
  const bool signal = (threadIdx.x & 127) == 0;
  int prev = -1;
  auto release = [&](int s) {
    if (signal) {
      mbar_arrive(&empty_bar[s]);
      if constexpr (PAIR) mbar_arrive_cluster(mapa_cluster(smem_u32(&empty_bar[s]), cluster_ctarank() ^ 1u));
    }
  };
#pragma unroll 1
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait_mma(&full_bar[stage], phase);
    const uint32_t base = smem_u32(smem + stage * stage_bytes);
    const uint64_t da = make_desc_k_sw128(base + a_off);
    const uint64_t db = make_desc_k_sw128(base + b_off);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)
      wgmma_bf16<N>(acc, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k),
                    static_cast<uint32_t>((kb | k) != 0));
    wgmma_commit();
    if (prev >= 0) {
      wgmma_wait<1>();
      release(prev);
    }
    prev = stage;
    if (++stage == nstages) { stage = 0; phase ^= 1u; }
  }
  wgmma_wait<0>();
  wgmma_reg_fence(acc);
  if (prev >= 0) release(prev);
}

// ------------------------------------------------------------------------------------------------ epilogue
// Two columns of one accumulator row.  Each quad of lanes covers 8 consecutive columns of a row (32 B fp32, 16 B bf16).
__device__ __forceinline__ void gemm_store_pair(const GemmParams& p, int row, int col, float v0, float v1, float b0,
                                                float b1) {
  const bool two = col + 1 < p.N;
  float f0, f1;
  if (p.mode == EPI_GELU_BF16) {
    f0 = gelu_erf(v0 + b0);
    f1 = gelu_erf(v1 + b1);
  } else {
    f0 = (v0 + b0) * p.alpha;
    f1 = (v1 + b1) * p.alpha;
  }
  if (p.mode == EPI_F32) {
    float* o = reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ldo + col;
    if (p.resid != nullptr) {
      const long long rrow = (p.resid_mod > 0) ? (row % p.resid_mod) : row;
      const float* r = p.resid + rrow * p.ldr + col;
      if (two && p.vec_ok) {
        const float2 x = *reinterpret_cast<const float2*>(r);
        f0 += x.x;
        f1 += x.y;
      } else {
        f0 += r[0];
        if (two) f1 += r[1];
      }
    }
    if (two && p.vec_ok) *reinterpret_cast<float2*>(o) = make_float2(f0, f1);
    else {
      o[0] = f0;
      if (two) o[1] = f1;
    }
  } else {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) +
                       (p.blocked_rows > 0 ? blocked_off(p.blocked_rows, row, col) : static_cast<long long>(row) * p.ldo + col);
    if (two && p.vec_ok) *reinterpret_cast<uint32_t*>(o) = pack_bf16(f0, f1);
    else {
      o[0] = __float2bfloat16_rn(f0);
      if (two) o[1] = __float2bfloat16_rn(f1);
    }
  }
}

template <int BLOCK_N, int CG>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = GemmCfg<BLOCK_N, CG>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;                         // 1024-B aligned (SWIZZLE_128B requirement)
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const uint32_t rank = (CG == 2) ? cluster_ctarank() : 0u;
  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_clusters = gridDim.x / CG;
  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int nstages = (p.max_stages > 0 && p.max_stages < Cfg::kStages) ? p.max_stages : Cfg::kStages;

  grid_dep_launch();                       // PDL: the next kernel may start its own prologue
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 2 * CG);
    }
    fence_mbar_init();
  }
  if constexpr (CG == 2) cluster_sync_all(); else __syncthreads();
  grid_dep_wait();                         // PDL: inputs of this GEMM are complete and visible from here on

  if (threadIdx.x < 128) {
    // ===================== TMA producer =====================
    // runs ahead across tiles: the next tile's operands stream in while the MMA warpgroups store this one
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x / CG; tile < num_tiles; tile += num_clusters) {
        const int m0 = (tile / p.num_n_tiles) * (GEMM_BLOCK_M * CG) + static_cast<int>(rank) * GEMM_BLOCK_M;
        const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          uint8_t* sb = sa + Cfg::kABytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * GEMM_BLOCK_K, m0);
          if constexpr (CG == 1) {
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K, n0);
          } else {
            const int r = static_cast<int>(rank);
            tma_load_2d_mcast(sb + r * Cfg::kBRows * GEMM_BLOCK_K * 2, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K,
                              n0 + r * Cfg::kBRows, 0x3);
          }
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else {
    // ===================== MMA warpgroups: rows [64 wg, 64 wg + 64) of the tile =====================
    const int wg = (threadIdx.x >> 7) - 1;
    int stage = 0;
    uint32_t phase = 0;
#pragma unroll 1
    for (int tile = blockIdx.x / CG; tile < num_tiles; tile += num_clusters) {
      const int m0 = (tile / p.num_n_tiles) * (GEMM_BLOCK_M * CG) + static_cast<int>(rank) * GEMM_BLOCK_M;
      const int n0 = (tile % p.num_n_tiles) * BLOCK_N;
      float acc[BLOCK_N / 2];
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.0f;
      wg_mainloop<BLOCK_N, CG == 2>(acc, smem, Cfg::kStageBytes, wg * (64 * GEMM_BLOCK_K * 2), Cfg::kABytes, full_bar,
                                    empty_bar, nstages, num_kb, stage, phase);
      const int t = threadIdx.x & 127;
      const int lane = t & 31;
      const int row_a = m0 + wg * 64 + (t >> 5) * 16 + (lane >> 2);
#pragma unroll
      for (int i = 0; i < BLOCK_N / 8; ++i) {
        const int col = n0 + i * 8 + 2 * (lane & 3);
        if (col >= p.N) continue;
        float b0 = 0.0f, b1 = 0.0f;
        if (p.bias != nullptr) {
          b0 = __ldg(p.bias + col);
          if (col + 1 < p.N) b1 = __ldg(p.bias + col + 1);
        }
        if (row_a < p.M) gemm_store_pair(p, row_a, col, acc[4 * i], acc[4 * i + 1], b0, b1);
        if (row_a + 8 < p.M) gemm_store_pair(p, row_a + 8, col, acc[4 * i + 2], acc[4 * i + 3], b0, b1);
      }
    }
  }
  // a CTA of a pair must not exit while its peer may still multicast into it or arrive on its barriers
  if constexpr (CG == 2) cluster_sync_all();
}

}  // namespace pq
