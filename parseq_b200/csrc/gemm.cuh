// Persistent warp-specialised bf16 GEMM on wgmma (sm_90a):
//   out[M,N] = epilogue( A[M,K] * W[N,K]^T + bias )
// A and W are bf16, K-contiguous ("K-major"); both are fetched by TMA into 128B-swizzled shared-memory stages of an
// mbarrier ring.  Warpgroup 0 is the producer (one thread issues the TMA loads); warpgroups 1 and 2 are "ping-pong"
// consumers: each owns whole 128 x 128 output tiles (the CTA's tiles alternate between them) and accumulates one in
// registers with wgmma (two m64n128k16 per k16 step).  An ordered pair of named barriers lets only one of them issue
// its main loop at a time, so one warpgroup's epilogue (bias, GELU, rounding, store) runs under the other's MMAs.
// A CTA walks the tiles with a stride of the grid; the ring position carries over from tile to tile.  Every projection
// of the PARSeq path goes through this kernel (QKV only where the fused QKV + attention kernel of qkv_attn.cuh does not
// apply): patch-embed (K=96), QKV / proj / fc1 / fc2 of the 12 ViT blocks
// (reference: timm Attention/Mlp via strhub/models/parseq/modules.py:145-165), the cross-attention K/V projection of
// the image memory, the decoder's q / out projections, MLP (modules.py:69-77) and the character head (model.py:63).
#pragma once
#include <cuda.h>
#include "ptx.cuh"

namespace pq {

enum GemmEpilogue : int {
  EPI_F32 = 0,        // out_f32 = alpha*(acc+bias) (+ resid[row or row%resid_mod])
  EPI_BF16 = 1,       // out_bf16 = bf16(alpha*(acc+bias))
  EPI_GELU_BF16 = 2,  // out_bf16 = bf16(gelu(acc+bias))
  EPI_F32_RESID = 3,  // kernel instantiation of EPI_F32 with a residual (the API's mode stays EPI_F32)
};
// How the kernel stores its tiles.  TMA: bf16 tiles go through a 128B-swizzled shared-memory staging tile and one
// thread stores them with cp.async.bulk.tensor, 2D row-major or 3D column-blocked ([N/64][rows][64]); the tensor map's
// bounds clip ragged rows and columns.  REG: every thread stores its accumulator pairs (fp32, or a bf16 output that is
// not a valid tensor map: base or row pitch not 16-B aligned).
enum GemmStore : int { ST_REG = 0, ST_TMA_2D = 1, ST_TMA_3D = 2 };

struct GemmParams {
  int M, N, K;
  float alpha;
  const float* bias;   // [N] or nullptr
  const float* resid;  // fp32 residual (may alias out: in-place accumulate) or nullptr
  long long ldr;
  int resid_mod;       // >0: residual row = row % resid_mod (broadcast tables: pos_embed, pos_queries)
  void* out;           // register-store epilogues only (the TMA store writes through its tensor map)
  long long ldo;       // elements
  int vec_ok;          // 8-byte aligned column pairs: paired stores allowed
  int num_m_tiles, num_n_tiles;
  int max_stages;      // 0: the full operand ring; n > 0: use only n slots (pipeline-depth experiments)
};

constexpr int GEMM_BLOCK_M = 128;  // rows per tile (two m64 halves, one warpgroup)
constexpr int GEMM_BLOCK_N = 128;  // columns per tile: QKV (1152), fc1 (1536), D = 384 / 768 split without padding
constexpr int GEMM_BLOCK_K = 64;   // 64 bf16 = 128 B = one swizzle row
constexpr int GEMM_THREADS = 384;  // warpgroup 0: TMA producer, warpgroups 1, 2: MMA + epilogue (ping-pong)

struct GemmCfg {
  static constexpr int kABytes = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;   // 16 KB
  static constexpr int kBBytes = GEMM_BLOCK_N * GEMM_BLOCK_K * 2;   // 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kHalfOutBytes = GEMM_BLOCK_M * 64 * 2;       // one 128 x 64 bf16 box of the output tile
  static constexpr int kOutBytes = 2 * kHalfOutBytes;               // one staging tile per consumer warpgroup
  // Four stages run as fast as five at M = 65 536 (tests/bench_gemm_shapes.py, gemm_stages sweep) and leave shared
  // memory to spare: 193 KB with the staging tiles, 129 KB for the register-store epilogues, which need none.
  static constexpr int kStages = 4;
  template <bool STAGING>
  static constexpr int smem_bytes() {
    return kStages * kStageBytes + (STAGING ? 2 * kOutBytes : 0) + 1024 /*align slack*/ + 256 /*barriers*/;
  }
};
static_assert(GemmCfg::smem_bytes<true>() <= 232448, "shared memory");

// ------------------------------------------------------------------------------------------------ operand ring
// full[s]: stage s holds its A and B tiles (TMA transaction bytes).  empty[s]: every MMA warpgroup that reads stage s
// has finished with it - in both CTAs of a pair when B is multicast (2 warpgroups x CG arrivals).
//
// Consumer side of the ring for one warpgroup: accumulates a 64 x N block over num_kb k-blocks.  a_off / b_off: byte
// offsets of the warpgroup's A rows / B rows inside a stage; stage / phase: the ring position, carried over from tile to
// tile.  A stage is released once the MMAs of the NEXT k-block are queued (wgmma_wait<1>), so the tensor cores never wait
// for the release round trip; the last one once the accumulator is complete.  Hence a ring needs at least two stages.
// (Used by the fused GEMM + LayerNorm kernel, gemm_ln.cuh.)
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

__device__ __forceinline__ void ring_advance(int& stage, uint32_t& phase, int n, int nstages) {
  const int s = stage + n;
  phase ^= static_cast<uint32_t>((s / nstages) & 1);
  stage = s % nstages;
}

// ------------------------------------------------------------------------------------------------ epilogue
template <int EPI>
__device__ __forceinline__ float gemm_epi(float v, float b, float alpha) {
  if constexpr (EPI == EPI_GELU_BF16) return gelu_erf(v + b);
  else return (v + b) * alpha;
}

// Register-store epilogue: fp32 (EPI_F32_RESID: plus a residual or broadcast table), or bf16 where the output cannot
// be a TMA tensor.  Two columns of one accumulator row per call.
template <int EPI>
__device__ __forceinline__ void gemm_store_pair(const GemmParams& p, int row, int col, float f0, float f1) {
  const bool two = col + 1 < p.N;
  if constexpr (EPI == EPI_F32 || EPI == EPI_F32_RESID) {
    float* o = reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ldo + col;
    if constexpr (EPI == EPI_F32_RESID) {
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
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(row) * p.ldo + col;
    if (two && p.vec_ok) *reinterpret_cast<uint32_t*>(o) = pack_bf16(f0, f1);
    else {
      o[0] = __float2bfloat16_rn(f0);
      if (two) o[1] = __float2bfloat16_rn(f1);
    }
  }
}

template <int EPI, int STORE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmOut, const GemmParams p) {
  constexpr bool TMA_OUT = STORE != ST_REG;
  static_assert(!TMA_OUT || EPI == EPI_BF16 || EPI == EPI_GELU_BF16, "the TMA store carries bf16 tiles");
  using Cfg = GemmCfg;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  const uint32_t pad = ((raw_addr + 1023u) & ~1023u) - raw_addr;
  uint8_t* smem = smem_raw + pad;                         // 1024-B aligned (SWIZZLE_128B requirement)
  uint8_t* out_stage = smem + Cfg::kStages * Cfg::kStageBytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(out_stage + (TMA_OUT ? 2 * Cfg::kOutBytes : 0));
  uint64_t* empty_bar = full_bar + Cfg::kStages;

  const int num_tiles = p.num_m_tiles * p.num_n_tiles;
  const int num_kb = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
  const int nstages = (p.max_stages > 0 && p.max_stages < Cfg::kStages) ? p.max_stages : Cfg::kStages;
  const int n_local = (num_tiles - 1 - static_cast<int>(blockIdx.x)) / static_cast<int>(gridDim.x) + 1;  // grid <= tiles

  grid_dep_launch();                       // PDL: the next kernel may start its own prologue
  if (threadIdx.x == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    if constexpr (TMA_OUT) prefetch_tmap(&tmOut);
    for (int s = 0; s < Cfg::kStages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 1);         // a stage is read by one consumer warpgroup
    }
    fence_mbar_init();
  }
  __syncthreads();
  grid_dep_wait();                         // PDL: inputs of this GEMM are complete and visible from here on

  if (threadIdx.x < 128) {
    // ===================== TMA producer: the CTA's tiles in order, running ahead across tiles =====================
    setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int j = 0; j < n_local; ++j) {
        const int tile = static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x);
        const int m0 = (tile / p.num_n_tiles) * GEMM_BLOCK_M;
        const int n0 = (tile % p.num_n_tiles) * GEMM_BLOCK_N;
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait_mma(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = smem + stage * Cfg::kStageBytes;
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          tma_load_2d(sa, &tmA, &full_bar[stage], kb * GEMM_BLOCK_K, m0);
          tma_load_2d(sa + Cfg::kABytes, &tmB, &full_bar[stage], kb * GEMM_BLOCK_K, n0);
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================== MMA warpgroup wg: the CTA's local tiles wg, wg + 2, ... =====================
    setmaxnreg_inc<232>();
    const int wg = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127;
    const int lane = t & 31;
    const int warp = t >> 5;
    const bool leader = t == 0;
    uint8_t* stage_out = out_stage + wg * Cfg::kOutBytes;
    int stage = 0;
    uint32_t phase = 0;
    if (wg == 1) ring_advance(stage, phase, num_kb, nstages);     // local tile 0 belongs to warpgroup 0
#pragma unroll 1
    for (int j = wg; j < n_local; j += 2) {
      const int tile = static_cast<int>(blockIdx.x) + j * static_cast<int>(gridDim.x);
      const int m0 = (tile / p.num_n_tiles) * GEMM_BLOCK_M;
      const int n0 = (tile % p.num_n_tiles) * GEMM_BLOCK_N;
      // ordered main loops: wait until the other warpgroup has issued every MMA of local tile j - 1
      if (j > 0) named_bar_sync(1 + wg, 256);
      float acc0[64], acc1[64];            // rows [0, 64) and [64, 128) of the tile
#pragma unroll
      for (int i = 0; i < 64; ++i) { acc0[i] = 0.0f; acc1[i] = 0.0f; }
      int prev = -1;
#pragma unroll 1
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait_mma(&full_bar[stage], phase);
        const uint32_t base = smem_u32(smem + stage * Cfg::kStageBytes);
        const uint64_t da0 = make_desc_k_sw128(base);
        const uint64_t da1 = make_desc_k_sw128(base + 64 * GEMM_BLOCK_K * 2);
        const uint64_t db = make_desc_k_sw128(base + Cfg::kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < GEMM_BLOCK_K / 16; ++k) {
          const uint32_t accum = static_cast<uint32_t>((kb | k) != 0);
          wgmma_bf16<128>(acc0, da0 + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), accum);
          wgmma_bf16<128>(acc1, da1 + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), accum);
        }
        wgmma_commit();
        if (prev >= 0) {
          wgmma_wait<1>();
          if (leader) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
      if (j + 1 < n_local) named_bar_arrive(1 + (wg ^ 1), 256);   // the other warpgroup may start its main loop
      wgmma_wait<0>();
      wgmma_reg_fence(acc0);
      wgmma_reg_fence(acc1);
      if (leader) mbar_arrive(&empty_bar[prev]);
      ring_advance(stage, phase, num_kb, nstages);                 // skip the other warpgroup's tile j + 1

      // ---- epilogue.  Accumulator layout (ptx.cuh wgmma_bf16): acc_h[4i + {0,1}] = row 64h + 16 warp + lane/4,
      // columns 8i + 2(lane%4) + {0,1}; acc_h[4i + {2,3}] = the same columns 8 rows further down.
      const int r0 = 16 * warp + (lane >> 2);
      if constexpr (TMA_OUT) {
        // the previous TMA store of this warpgroup has finished reading the staging tile
        if (leader) bulk_wait_group_read<0>();
        named_bar_sync(3 + wg, 128);
      }
#pragma unroll
      for (int i = 0; i < GEMM_BLOCK_N / 8; ++i) {
        const int col = n0 + i * 8 + 2 * (lane & 3);
        float b0 = 0.0f, b1 = 0.0f;
        if (p.bias != nullptr) {
          if (col < p.N) b0 = __ldg(p.bias + col);
          if (col + 1 < p.N) b1 = __ldg(p.bias + col + 1);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {        // (half, +8 rows)
          const float* acc = (q < 2) ? acc0 : acc1;
          const int rl = 64 * (q >> 1) + r0 + 8 * (q & 1);
          const float f0 = gemm_epi<EPI>(acc[4 * i + 2 * (q & 1)], b0, p.alpha);
          const float f1 = gemm_epi<EPI>(acc[4 * i + 2 * (q & 1) + 1], b1, p.alpha);
          if constexpr (TMA_OUT) {
            // 128B swizzle: 16-B chunk c of row r sits at chunk c ^ (r % 8); r % 8 = lane / 4 here
            uint8_t* dst = stage_out + (i >> 3) * Cfg::kHalfOutBytes + rl * 128 + ((((i & 7) ^ (lane >> 2))) << 4) +
                           (lane & 3) * 4;
            *reinterpret_cast<uint32_t*>(dst) = pack_bf16(f0, f1);
          } else {
            const int row = m0 + rl;
            if (row < p.M && col < p.N) gemm_store_pair<EPI>(p, row, col, f0, f1);
          }
        }
      }
      if constexpr (TMA_OUT) {
        fence_proxy_async_smem();            // the staging writes are visible to the TMA (async proxy)
        named_bar_sync(3 + wg, 128);
        if (leader) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int c0 = n0 + 64 * h;
            if (c0 >= p.N) break;
            if constexpr (STORE == ST_TMA_3D) tma_store_3d(&tmOut, stage_out + h * Cfg::kHalfOutBytes, 0, m0, c0 / 64);
            else tma_store_2d(&tmOut, stage_out + h * Cfg::kHalfOutBytes, c0, m0);
          }
          bulk_commit_group();
        }
      }
    }
    if constexpr (TMA_OUT) {
      // the last stores have read their staging tile before the CTA's shared memory is released; their global writes
      // are part of this grid's results, visible to the next kernel once the grid completes
      if (leader) bulk_wait_group_read<0>();
    }
  }
}

}  // namespace pq
