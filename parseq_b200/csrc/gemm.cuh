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
  EPI_LSE = 4,        // no output tile: per-row log-sum-exp partials of the tile (gemm_lse_epilogue), candidate scoring
  EPI_TOPK = 5,       // EPI_LSE partials of the allowed classes plus each row's top-K classes of the tile (beam search)
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
  // EPI_LSE only: target class of each row (< 0: none) and where its logit goes; `out` holds the float2 partials
  const int* lse_tgt;
  float* lse_tlogit;
  // EPI_TOPK only: per row and tile the K best (beam_order_key) of the allowed classes, BEAM_TOPK_LD keys per (row, tile),
  // 0 past the last; allowlist rows (ceil(N / 32) words; row r reads word row r / topk_mask_div), or null
  unsigned long long* topk_keys;
  int topk_k;
  const uint32_t* topk_mask;
  int topk_mask_div;
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

// EPI_LSE: the logits of a 128 x 128 tile stay in the accumulator registers.  For each row the tile leaves (max, sum of
// exp(v - max)) over its columns < N in out[row * num_n_tiles + tile column] (float2), and the logit of the row's
// target class, if that class is one of the tile's columns, in lse_tlogit[row].  v = (acc + bias) * alpha is the value
// EPI_F32 stores, formed once per row into v[32].  Next to the 128 accumulators this costs a 48-byte stack frame (ptxas);
// forming v twice instead (max pass, sum pass) has no spill but halved the epilogue's throughput (104-110 against
// 238-250 TFLOP/s at 16384 classes, H100 80GB HBM3, 700 W), so v stays.  A tile whose max is -inf sums exp(v) instead,
// so that it contributes 0, or NaN if it holds a NaN; NaN and +inf propagate through the sum as they do through torch's
// log_softmax.  expf, not __expf: the partials carry fp32 rounding only.  The four lanes of a row (lane % 4) combine
// with a fixed xor-shuffle order.
__device__ __forceinline__ void gemm_lse_epilogue(const GemmParams& p, const float (&acc0)[64], const float (&acc1)[64],
                                                  int m0, int n0, int r0, int lane) {
  float2* part = reinterpret_cast<float2*>(p.out);
#pragma unroll
  for (int q = 0; q < 4; ++q) {        // (half, +8 rows)
    const float* acc = (q < 2) ? acc0 : acc1;
    const int row = m0 + 64 * (q >> 1) + r0 + 8 * (q & 1);
    const int tgt = (row < p.M && p.lse_tgt != nullptr) ? __ldg(p.lse_tgt + row) : -1;
    float v[32];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < GEMM_BLOCK_N / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n0 + i * 8 + 2 * (lane & 3) + e;
        const float b = (p.bias != nullptr && col < p.N) ? __ldg(p.bias + col) : 0.0f;
        const float f = gemm_epi<EPI_F32>(acc[4 * i + 2 * (q & 1) + e], b, p.alpha);
        v[2 * i + e] = col < p.N ? f : -INFINITY;
        mx = fmaxf(mx, v[2 * i + e]);
        if (col == tgt) p.lse_tlogit[row] = f;
      }
    }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float base = (mx == -INFINITY) ? 0.0f : mx;
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 32; ++k) s += expf(v[k] - base);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    if ((lane & 3) == 0 && row < p.M)
      part[static_cast<long long>(row) * p.num_n_tiles + n0 / GEMM_BLOCK_N] = make_float2(mx, s);
  }
}

// EPI_TOPK: the EPI_LSE body over the allowed classes (a masked class counts as -inf, so it adds 0 to the sum), and each
// row's K best allowed classes of the tile (-inf never listed).  The four lanes of a row hold 32 columns each: K rounds
// of a masked arg-max over a lane's 32 values (a 32-bit "taken" mask), merged over the four lanes with the xor-shuffle
// order of the LSE.  No logit reaches memory.
__device__ __forceinline__ void gemm_topk_epilogue(const GemmParams& p, const float (&acc0)[64], const float (&acc1)[64],
                                                   int m0, int n0, int r0, int lane) {
  float2* part = reinterpret_cast<float2*>(p.out);
  const int words = (p.N + 31) >> 5;
#pragma unroll
  for (int q = 0; q < 4; ++q) {        // (half, +8 rows)
    const float* acc = (q < 2) ? acc0 : acc1;
    const int row = m0 + 64 * (q >> 1) + r0 + 8 * (q & 1);
    const uint32_t* mrow = (p.topk_mask != nullptr && row < p.M)
                               ? p.topk_mask + static_cast<long long>(row / p.topk_mask_div) * words : nullptr;
    float v[32];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < GEMM_BLOCK_N / 8; ++i) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = n0 + i * 8 + 2 * (lane & 3) + e;
        const float b = (p.bias != nullptr && col < p.N) ? __ldg(p.bias + col) : 0.0f;
        const float f = gemm_epi<EPI_F32>(acc[4 * i + 2 * (q & 1) + e], b, p.alpha);
        const bool ok = col < p.N && (mrow == nullptr || class_allowed(mrow, col));
        v[2 * i + e] = ok ? f : -INFINITY;
        mx = fmaxf(mx, v[2 * i + e]);
      }
    }
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float base = (mx == -INFINITY) ? 0.0f : mx;
    float s = 0.0f;
#pragma unroll
    for (int k = 0; k < 32; ++k) s += expf(v[k] - base);
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    const int tile = n0 / GEMM_BLOCK_N;
    if ((lane & 3) == 0 && row < p.M) part[static_cast<long long>(row) * p.num_n_tiles + tile] = make_float2(mx, s);
    unsigned long long* keys = p.topk_keys + (static_cast<long long>(row) * p.num_n_tiles + tile) * BEAM_TOPK_LD;
    uint32_t taken = 0u;
#pragma unroll 1
    for (int r = 0; r < p.topk_k; ++r) {
      unsigned long long best = 0ull;
      int bk = -1;
#pragma unroll
      for (int k = 0; k < 32; ++k) {
        const int col = n0 + (k >> 1) * 8 + 2 * (lane & 3) + (k & 1);
        const unsigned long long key =
            (((taken >> k) & 1u) || v[k] == -INFINITY) ? 0ull : beam_order_key(v[k], col);
        if (key > best) { best = key; bk = k; }
      }
      unsigned long long w = best;
      w = max(w, __shfl_xor_sync(0xffffffffu, w, 1));
      w = max(w, __shfl_xor_sync(0xffffffffu, w, 2));
      if (w != 0ull && w == best) taken |= 1u << bk;   // keys are unique within a row: one lane takes it
      if ((lane & 3) == 0 && row < p.M) keys[r] = w;
    }
  }
}

// The kernel body lives in gemm_body.inc, included by each kernel below with EPI and STORE in scope.
template <int EPI, int STORE>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_wgmma_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmOut, const GemmParams p) {
#include "gemm_body.inc"
}

// The head GEMM of candidate scoring: the same body with the log-sum-exp epilogue (EPI_LSE, register path).  A kernel of
// its own name rather than one more gemm_bf16_wgmma_kernel instantiation, which keeps that kernel's set unchanged.
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_lse_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                     const __grid_constant__ CUtensorMap tmOut, const GemmParams p) {
  constexpr int EPI = EPI_LSE, STORE = ST_REG;
#include "gemm_body.inc"
}

// The head GEMM of beam search above 128 classes: the same body with the top-K epilogue (EPI_TOPK, register path).
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_bf16_topk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                      const __grid_constant__ CUtensorMap tmOut, const GemmParams p) {
  constexpr int EPI = EPI_TOPK, STORE = ST_REG;
#include "gemm_body.inc"
}

}  // namespace pq
