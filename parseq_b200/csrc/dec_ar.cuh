// Persistent autoregressive-decode kernel: the whole `decode_ar` loop of PARSeq.forward (model.py:119-147) for one
// super-chunk of images in ONE launch.  The AR loop is a chain of tiny, strictly dependent operations (M = batch rows
// per step); as separate kernels each link costs a kernel boundary (a launch gap each, 10 links per step, 26
// steps).  Here every step is 8 phases separated by a software grid barrier (~2 us):
//   P1 self-attention over the (position, token) K/V table            (warp per (image, head))
//   P2 y  = pos_queries[i] + out_proj(sa)                              (64x64 mma.sync tiles)
//   P3 qc = scale * q_proj(LN1(y))                                     (LayerNorm fused as the A-operand prologue)
//   P4 cross-attention over the image K/V cache                        (warp per (image, head))
//   P5 y += out_proj(ca)
//   P6 hd = GELU(linear1(LN2(y)))
//   P7 part[s] = linear2(hd) over K-slice s (3-way split-K, deterministic: no atomics)
//   P8 logits[:, i] = head(LN3(y + part0 + part1 + part2)); ids[:, i+1] = argmax   (64x96 tiles, argmax in the epilogue)
// The projections of one step are 1.7 GFLOP over M <= 512 rows: latency-, not throughput-bound, so they run on
// warp-level mma.sync tiles fed by cp.async (no TMA / mbarrier set-up cost per phase); the large-M refine / NAR passes and the
// encoder stay on the wgmma GEMM.  Numerics: identical rounding points to the multi-kernel path (bf16 operands,
// fp32 accumulation, fp32 residual stream y, fp32 LayerNorm / softmax statistics).
#pragma once
#include <type_traits>

#include "ptx.cuh"

namespace pq {

struct DecArParams {
  int B, L, Md, V, C, T, heads;
  float qscale;
  const float* qs;                // [L, D] pre-scaled self-attention queries of pos_queries
  const __nv_bfloat16* kvtab;     // [(pos*V + tok), 2D]
  const float* posq;              // [L, D]
  const __nv_bfloat16 *Wo_s, *Wq_c, *Wo_c, *W1, *W2, *Wh;
  const float *bo_s, *bq_c, *bo_c, *b1, *b2, *bh;
  const float *g1, *be1, *g2, *be2, *g3, *be3;
  const __nv_bfloat16* ckv;       // column-blocked [2D/64][kv_rows][64], row = image * T + key (ptx.cuh: blocked_off)
  long long kv_rows;
  int* ids;                       // [B, ids_ld]: ids[:,0] = BOS on entry
  int ids_ld;
  __nv_bfloat16 *sa, *ca, *hd;    // [B, D], [B, D], [B, Md]
  float *y, *qc;                  // [B, D]
  float* part;                    // [3][B, D] split-K partial sums of linear2 (summed in fixed order by the head phase)
  float* logits;                  // [B, L, C]
  const int* forced;              // optional teacher forcing [B, forced_ld]
  int forced_ld;
  unsigned int* bar;              // grid-barrier counter, zero on entry
  unsigned long long* prof;       // optional [L][16] globaltimer stamps of block 0 (phase boundaries), or nullptr
};

constexpr int DEC_THREADS = 256;

__device__ __forceinline__ uint32_t swz64(int r, int c) {  // element offset of (row r, col c) in a [rows][64] bf16 tile
  return static_cast<uint32_t>(r * 64 + ((((c >> 3) ^ (r & 7)) << 3) | (c & 7)));
}

__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define DEC_PROF(slot)                                                                     \
  do {                                                                                     \
    if (p.prof != nullptr && blockIdx.x == 0 && threadIdx.x == 0) p.prof[step * 16 + (slot)] = global_timer_ns(); \
  } while (0)

__device__ __forceinline__ void grid_barrier(unsigned int* bar, unsigned int& target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    target += gridDim.x;
    __threadfence();
    atomicAdd(bar, 1u);
    unsigned int v;
    long long t0 = clock64();
    do {
      asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(bar) : "memory");
      if (v < target && (clock64() - t0) > PQ_SPIN_LIMIT_CYCLES) {
        printf("[parseq_b200] grid barrier timeout: block %d count %u target %u\n", blockIdx.x, v, target);
        __trap();
      }
    } while (v < target);
    __threadfence();
  }
  __syncthreads();
}

enum DecEpi : int { DE_POSQ = 0, DE_SCALE = 1, DE_RMW = 2, DE_GELU = 3, DE_HEAD = 4, DE_PART = 5 };
constexpr int DEC_KSPLIT = 3;      // linear2 (K = 4D) is split 3-way over otherwise idle CTAs

struct DecSmem {   // byte offsets into dynamic shared memory
  // a_res: [D/64][64*64] bf16 (LN'ed rows, resident), a_st / w_st: double-buffered streamed k-blocks
};

// One output tile: rows [row0, row0+64) x cols [n0, n0 + 16*NT) of  A[M,K] * W[N,K]^T.
//   LN_A: A = bf16(LayerNorm(ysrc rows; gamma, beta, eps=1e-5)) computed here (K == D), else A bf16 [M, lda] streamed.
// 8 warps: warp w -> 16-row slab (w & 3), column half (w >> 2) of NT n8-tiles.  W (and A) k-blocks of 64 are streamed
// through a 3-stage cp.async ring (each stage costs one L2 round trip, so depth matters more than width here).
constexpr int DEC_STAGES = 4;
constexpr int DEC_MAX_BN = 128;
template <int D, int NT, bool LN_A, int EPI, int MS = 4>
__device__ void dec_tile(const DecArParams& p, unsigned char* smem, const __nv_bfloat16* __restrict__ A, int lda,
                         const float* __restrict__ ysrc, const float* __restrict__ gamma, const float* __restrict__ beta,
                         const __nv_bfloat16* __restrict__ W, int K, int N, const float* __restrict__ bias, int row0, int n0,
                         int step, int ldw = 0, int split = 0, const float* __restrict__ addp = nullptr) {
  // ldw: row pitch of W (elements) when only a K-slice of it is multiplied (split-K), 0 -> K.
  // addp: LN_A only - DEC_KSPLIT extra fp32 [M, D] arrays added (in fixed order) to ysrc before normalising.
  // MS = 4: 64-row tile, warp w -> slab (w & 3), column half (w >> 2);  MS = 1: 16-row tile, warp w -> columns only
  constexpr int NWN = 8 / MS;                 // warps along N
  constexpr int BN = 8 * NT * NWN;
  constexpr int TM = 16 * MS;                 // rows per tile
  const int wld = ldw ? ldw : K;
  static_assert(BN <= DEC_MAX_BN, "tile width");
  __nv_bfloat16* a_res = reinterpret_cast<__nv_bfloat16*>(smem);                        // [D/64][4096]
  __nv_bfloat16* a_st = a_res + (D / 64) * 4096;                                         // [STAGES][4096]
  __nv_bfloat16* w_st = a_st + DEC_STAGES * 4096;                                        // [STAGES][BN*64]
  float* s_log = reinterpret_cast<float*>(w_st + DEC_STAGES * DEC_MAX_BN * 64);          // [64][128] (head only)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int M = p.B;
  const int nkb = K / 64;

  auto load_stage = [&](int kb, int stage) {
    for (int i = tid; i < BN * 8; i += DEC_THREADS) {
      const int r = i >> 3, ck = i & 7;
      int n = n0 + r;
      if (n >= N) n = N - 1;
      cp_async_16(smem_u32(w_st + stage * (BN * 64) + swz64(r, ck * 8)), W + static_cast<long long>(n) * wld + kb * 64 + ck * 8);
    }
    if (!LN_A) {
      for (int i = tid; i < TM * 8; i += DEC_THREADS) {
        const int r = i >> 3, ck = i & 7;
        int m = row0 + r;
        if (m >= M) m = M - 1;
        cp_async_16(smem_u32(a_st + stage * 4096 + swz64(r, ck * 8)), A + static_cast<long long>(m) * lda + kb * 64 + ck * 8);
      }
    }
  };

  // prologue: fill STAGES-1 stages (one commit group per k-block, empty groups keep the accounting uniform)
#pragma unroll
  for (int s0 = 0; s0 < DEC_STAGES - 1; ++s0) {
    if (s0 < nkb) load_stage(s0, s0);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  if (LN_A) {
    // LayerNorm of this tile's 64 rows while the first W stages are in flight; 4 rows per warp at a time with all
    // loads issued before the first reduction (one L2 round trip per batch instead of one per row)
    constexpr int NV = D / 64;
    auto ln_rows = [&](auto RBtag, int first) {   // RB rows of this warp starting at its `first`-th row
      constexpr int RB = decltype(RBtag)::value;
      float2 v[RB][NV];
#pragma unroll
      for (int j = 0; j < RB; ++j) {
        int m = row0 + warp + 8 * (first + j);
        if (m >= M) m = M - 1;
        const float2* xr = reinterpret_cast<const float2*>(ysrc + static_cast<long long>(m) * D);
#pragma unroll
        for (int i = 0; i < NV; ++i) v[j][i] = xr[i * 32 + lane];
        if (addp != nullptr) {
          float2 a[DEC_KSPLIT][NV];
#pragma unroll
          for (int sp = 0; sp < DEC_KSPLIT; ++sp) {
            const float2* ar = reinterpret_cast<const float2*>(addp + (static_cast<long long>(sp) * M + m) * D);
#pragma unroll
            for (int i = 0; i < NV; ++i) a[sp][i] = ar[i * 32 + lane];
          }
#pragma unroll
          for (int sp = 0; sp < DEC_KSPLIT; ++sp)
#pragma unroll
            for (int i = 0; i < NV; ++i) { v[j][i].x += a[sp][i].x; v[j][i].y += a[sp][i].y; }
        }
      }
#pragma unroll
      for (int j = 0; j < RB; ++j) {
        const int r = warp + 8 * (first + j);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) s += v[j][i].x + v[j][i].y;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = s * (1.0f / D);
        float q = 0.f;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const float a = v[j][i].x - mean, b = v[j][i].y - mean;
          q += a * a + b * b;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
        const float rstd = 1.0f / sqrtf(q * (1.0f / D) + 1e-5f);
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int c = (i * 32 + lane) * 2;          // column of v[.][i].x
          const float2 g = __ldg(reinterpret_cast<const float2*>(gamma) + i * 32 + lane);
          const float2 b = __ldg(reinterpret_cast<const float2*>(beta) + i * 32 + lane);
          const float o0 = (v[j][i].x - mean) * rstd * g.x + b.x;
          const float o1 = (v[j][i].y - mean) * rstd * g.y + b.y;
          *reinterpret_cast<uint32_t*>(a_res + (c >> 6) * 4096 + swz64(r, c & 63)) = pack_bf16(o0, o1);
        }
      }
    };
    constexpr int RPW = TM / 8;               // rows per warp
    if (RPW == 2) {
      ln_rows(std::integral_constant<int, 2>{}, 0);
    } else if (addp != nullptr) {
#pragma unroll 1
      for (int f = 0; f < RPW; f += 2) ln_rows(std::integral_constant<int, 2>{}, f);
    } else {
#pragma unroll 1
      for (int f = 0; f < RPW; f += 4) ln_rows(std::integral_constant<int, 4>{}, f);
    }
  }

  const int ms = (MS == 4) ? (warp & 3) : 0, nh = (MS == 4) ? (warp >> 2) : warp;
  float acc[NT][4];
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) { acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f; }

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb % DEC_STAGES;
    asm volatile("cp.async.wait_group %0;" ::"n"(DEC_STAGES - 2) : "memory");   // k-block kb has landed
    __syncthreads();                                                             // ... for every thread; stage (kb-1) is free
    if (kb + DEC_STAGES - 1 < nkb) load_stage(kb + DEC_STAGES - 1, (kb + DEC_STAGES - 1) % DEC_STAGES);
    asm volatile("cp.async.commit_group;" ::: "memory");
    const __nv_bfloat16* at = LN_A ? (a_res + kb * 4096) : (a_st + st * 4096);
    const __nv_bfloat16* wt = w_st + st * (BN * 64);
#pragma unroll
    for (int kt = 0; kt < 4; ++kt) {
      uint32_t a0, a1, a2, a3;
      {
        const int row = ms * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int col = kt * 16 + (lane >> 4) * 8;
        ldmatrix_x4(smem_u32(at + swz64(row, col)), a0, a1, a2, a3);
      }
#pragma unroll
      for (int np = 0; np < NT / 2; ++np) {
        const int n = (nh * NT + np * 2) * 8 + (lane & 7) + (lane >> 4) * 8;
        const int col = kt * 16 + ((lane >> 3) & 1) * 8;
        uint32_t b0, b1, b2, b3;
        ldmatrix_x4(smem_u32(wt + swz64(n, col)), b0, b1, b2, b3);
        mma_bf16_16816(acc[np * 2], a0, a1, a2, a3, b0, b1);
        mma_bf16_16816(acc[np * 2 + 1], a0, a1, a2, a3, b2, b3);
      }
    }
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();                                   // all warps done with smem before the next tile / phase reuses it

  // ---------------- epilogue ----------------
  const int g = lane >> 2, t = lane & 3;
  const int r_lo = row0 + ms * 16 + g, r_hi = r_lo + 8;
  if (EPI == DE_HEAD) {
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int c = (nh * NT + nt) * 8 + 2 * t;     // column inside the 96-wide tile
      const float b0 = (c < N) ? __ldg(bias + c) : 0.f, b1 = (c + 1 < N) ? __ldg(bias + c + 1) : 0.f;
      s_log[(ms * 16 + g) * 128 + c] = acc[nt][0] + b0;
      s_log[(ms * 16 + g) * 128 + c + 1] = acc[nt][1] + b1;
      s_log[(ms * 16 + g + 8) * 128 + c] = acc[nt][2] + b0;
      s_log[(ms * 16 + g + 8) * 128 + c + 1] = acc[nt][3] + b1;
    }
    __syncthreads();
    for (int r = warp; r < TM; r += 8) {
      const int m = row0 + r;
      if (m >= M) continue;                          // warp-uniform
      float* lrow = p.logits + (static_cast<long long>(m) * p.L + step) * p.C;
      float best = -INFINITY;
      int bi = 0x7fffffff;
      for (int j = lane; j < N; j += 32) {
        const float v = s_log[r * 128 + j];
        lrow[j] = v;
        if (v > best) { best = v; bi = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
      }
      if (lane == 0 && step + 1 < p.L) {
        int v = bi;
        if (p.forced != nullptr) v = p.forced[static_cast<long long>(m) * p.forced_ld + step + 1];
        p.ids[static_cast<long long>(m) * p.ids_ld + step + 1] = v;
      }
    }
    __syncthreads();
    return;
  }
#pragma unroll
  for (int nt = 0; nt < NT; ++nt) {
    const int c = n0 + (nh * NT + nt) * 8 + 2 * t;
    if (c >= N) continue;                            // ragged last column tile (D = 192 with 128-wide tiles); N is even
    const float2 bb = __ldg(reinterpret_cast<const float2*>(bias + c));
    float v00 = acc[nt][0] + bb.x, v01 = acc[nt][1] + bb.y, v10 = acc[nt][2] + bb.x, v11 = acc[nt][3] + bb.y;
    if (EPI == DE_POSQ) {
      const float2 pq2 = __ldg(reinterpret_cast<const float2*>(p.posq + static_cast<long long>(step) * D + c));
      if (r_lo < M) *reinterpret_cast<float2*>(p.y + static_cast<long long>(r_lo) * D + c) = make_float2(v00 + pq2.x, v01 + pq2.y);
      if (r_hi < M) *reinterpret_cast<float2*>(p.y + static_cast<long long>(r_hi) * D + c) = make_float2(v10 + pq2.x, v11 + pq2.y);
    } else if (EPI == DE_SCALE) {
      if (r_lo < M) *reinterpret_cast<float2*>(p.qc + static_cast<long long>(r_lo) * D + c) = make_float2(v00 * p.qscale, v01 * p.qscale);
      if (r_hi < M) *reinterpret_cast<float2*>(p.qc + static_cast<long long>(r_hi) * D + c) = make_float2(v10 * p.qscale, v11 * p.qscale);
    } else if (EPI == DE_RMW) {
      if (r_lo < M) {
        float2* d = reinterpret_cast<float2*>(p.y + static_cast<long long>(r_lo) * D + c);
        const float2 o = *d;
        *d = make_float2(o.x + v00, o.y + v01);
      }
      if (r_hi < M) {
        float2* d = reinterpret_cast<float2*>(p.y + static_cast<long long>(r_hi) * D + c);
        const float2 o = *d;
        *d = make_float2(o.x + v10, o.y + v11);
      }
    } else if (EPI == DE_PART) {   // split-K partial (bias only in split 0), no read-modify-write
      const float kb0 = (split == 0) ? 1.0f : 0.0f;
      float* dst = p.part + static_cast<long long>(split) * M * D;
      if (r_lo < M) *reinterpret_cast<float2*>(dst + static_cast<long long>(r_lo) * D + c) = make_float2(acc[nt][0] + kb0 * bb.x, acc[nt][1] + kb0 * bb.y);
      if (r_hi < M) *reinterpret_cast<float2*>(dst + static_cast<long long>(r_hi) * D + c) = make_float2(acc[nt][2] + kb0 * bb.x, acc[nt][3] + kb0 * bb.y);
    } else {  // DE_GELU -> hd bf16 [M, Md]
      if (r_lo < M) *reinterpret_cast<uint32_t*>(p.hd + static_cast<long long>(r_lo) * p.Md + c) = pack_bf16(gelu_erf(v00), gelu_erf(v01));
      if (r_hi < M) *reinterpret_cast<uint32_t*>(p.hd + static_cast<long long>(r_hi) * p.Md + c) = pack_bf16(gelu_erf(v10), gelu_erf(v11));
    }
  }
}

template <int D, int TB>   // TB = number of 128-key blocks of the image memory (T <= 128*TB)
__global__ void __launch_bounds__(DEC_THREADS, 1) dec_ar_kernel(const DecArParams p) {
  extern __shared__ __align__(128) unsigned char dec_smem[];
  grid_dep_launch();
  grid_dep_wait();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int gwarp = blockIdx.x * (DEC_THREADS / 32) + warp;
  const int nwarps = gridDim.x * (DEC_THREADS / 32);
  const int mt = (p.B + 63) / 64;
  unsigned int target = 0;

  for (int step = 0; step < p.L; ++step) {
    const int nkeys = step + 1;
    DEC_PROF(0);
    // ---------------- P1: self-attention, warp per (image, head); query position = step ----------------
    // context ids of all items of this warp -> shared memory first (independent loads, one L2 round trip)
    int* s_ids = reinterpret_cast<int*>(dec_smem) + warp * (8 * 32);
    {
      int j = 0;
      for (int item = gwarp; item < p.B * p.heads && j < 8; item += nwarps, ++j)
        s_ids[j * 32 + lane] = (lane < nkeys) ? p.ids[static_cast<long long>(item / p.heads) * p.ids_ld + lane] : 0;
      __syncwarp();
    }
    int jitem = 0;
#pragma unroll 1
    for (int item = gwarp; item < p.B * p.heads; item += nwarps, ++jitem) {
      const int b = item / p.heads, h = item % p.heads;
      const int myid = (jitem < 8) ? s_ids[jitem * 32 + lane]
                                   : ((lane < nkeys) ? p.ids[static_cast<long long>(b) * p.ids_ld + lane] : 0);
      float kreg[32];
      if (lane < nkeys) {
        const uint4* kr = reinterpret_cast<const uint4*>(p.kvtab + (static_cast<long long>(lane) * p.V + myid) * 2 * D + h * 32);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint4 u = __ldg(kr + j);
          const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&u);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(p2[e]);
            kreg[j * 8 + e * 2] = f.x;
            kreg[j * 8 + e * 2 + 1] = f.y;
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 32; ++j) kreg[j] = 0.f;
      }
      const float qv = __ldg(p.qs + static_cast<long long>(step) * D + h * 32 + lane);
      float vreg[32];
      // element offset of key `lane`'s V row segment for this head (one multiply per lane instead of one per key)
      const int voff = (lane * p.V + myid) * (2 * D) + D + h * 32;
#pragma unroll
      for (int k = 0; k < 32; ++k) {      // V gathers issued together with the K loads: one L2 round trip per item
        const int ok = __shfl_sync(0xffffffffu, voff, k);
        vreg[k] = (k < nkeys) ? __bfloat162float(p.kvtab[ok + lane]) : 0.f;
      }
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) s = fmaf(__shfl_sync(0xffffffffu, qv, j), kreg[j], s);
      if (lane >= nkeys) s = -INFINITY;
      float mx = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float e = (lane < nkeys) ? expf(s - mx) : 0.f;
      float sum = e;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float pme = e / sum;
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 32; ++k) acc = fmaf(__shfl_sync(0xffffffffu, pme, k), vreg[k], acc);
      p.sa[static_cast<long long>(b) * D + h * 32 + lane] = __float2bfloat16_rn(acc);
    }
    DEC_PROF(1);
    grid_barrier(p.bar, target);
    DEC_PROF(2);
    // ---------------- P2: y = pos_queries[step] + out_proj(sa) ----------------
    for (int tile = blockIdx.x; tile < mt * (D / 64); tile += gridDim.x)
      dec_tile<D, 4, false, DE_POSQ>(p, dec_smem, p.sa, D, nullptr, nullptr, nullptr, p.Wo_s, D, D, p.bo_s, (tile / (D / 64)) * 64,
                                     (tile % (D / 64)) * 64, step);
    DEC_PROF(3);
    grid_barrier(p.bar, target);
    DEC_PROF(4);
    // ---------------- P3: qc = scale * q_proj(LN1(y)) ----------------
    {
      const int mt16 = (p.B + 15) / 16, ntq = (D + 127) / 128;   // D = 192: second tile is half empty
      for (int tile = blockIdx.x; tile < mt16 * ntq; tile += gridDim.x)
        dec_tile<D, 2, true, DE_SCALE, 1>(p, dec_smem, nullptr, 0, p.y, p.g1, p.be1, p.Wq_c, D, D, p.bq_c, (tile / ntq) * 16,
                                          (tile % ntq) * 128, step);
    }
    DEC_PROF(5);
    grid_barrier(p.bar, target);
    DEC_PROF(6);
    // ---------------- P4: cross-attention, warp per (image, head), T <= 128*TB keys ----------------
    for (int item = gwarp; item < p.B * p.heads; item += nwarps) {
      const int b = item / p.heads, h = item % p.heads;
      const long long row_b = static_cast<long long>(b) * p.T;
      // lane = (key group kg = lane>>2, 8-channel chunk cc = lane&3) for the 16-byte V loads
      const int kg = lane >> 2, cc = lane & 3;
      const __nv_bfloat16* kb0 = p.ckv + blocked_off(p.kv_rows, row_b, h * 32);                 // + key * 64
      const __nv_bfloat16* vb = p.ckv + blocked_off(p.kv_rows, row_b, D + h * 32 + cc * 8);     // + key * 64
      const float qv = p.qc[static_cast<long long>(b) * D + h * 32 + lane];
      float sc[4 * TB];
      uint4 vv[16];
#pragma unroll
      for (int blk = 0; blk < TB; ++blk) {
        uint32_t kw[4][16];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int key = blk * 128 + r * 32 + lane;
          if (key < p.T) {
            const uint4* kr = reinterpret_cast<const uint4*>(kb0 + static_cast<long long>(key) * 64);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const uint4 u = __ldg(kr + j);
              kw[r][j * 4] = u.x; kw[r][j * 4 + 1] = u.y; kw[r][j * 4 + 2] = u.z; kw[r][j * 4 + 3] = u.w;
            }
          } else {
#pragma unroll
            for (int j = 0; j < 16; ++j) kw[r][j] = 0u;
          }
        }
        if (TB == 1) {   // single block: request V together with K (one L2 round trip per item)
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int key = i * 8 + kg;
            vv[i] = (key < p.T) ? __ldg(reinterpret_cast<const uint4*>(vb + static_cast<long long>(key) * 64)) : make_uint4(0u, 0u, 0u, 0u);
          }
        }
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
        for (int w = 0; w < 16; ++w) {
          const float qa = __shfl_sync(0xffffffffu, qv, 2 * w), qb = __shfl_sync(0xffffffffu, qv, 2 * w + 1);
          s0 = fmaf(qb, __uint_as_float(kw[0][w] & 0xffff0000u), fmaf(qa, __uint_as_float(kw[0][w] << 16), s0));
          s1 = fmaf(qb, __uint_as_float(kw[1][w] & 0xffff0000u), fmaf(qa, __uint_as_float(kw[1][w] << 16), s1));
          s2 = fmaf(qb, __uint_as_float(kw[2][w] & 0xffff0000u), fmaf(qa, __uint_as_float(kw[2][w] << 16), s2));
          s3 = fmaf(qb, __uint_as_float(kw[3][w] & 0xffff0000u), fmaf(qa, __uint_as_float(kw[3][w] << 16), s3));
        }
        sc[blk * 4 + 0] = (blk * 128 + lane < p.T) ? s0 : -INFINITY;
        sc[blk * 4 + 1] = (blk * 128 + 32 + lane < p.T) ? s1 : -INFINITY;
        sc[blk * 4 + 2] = (blk * 128 + 64 + lane < p.T) ? s2 : -INFINITY;
        sc[blk * 4 + 3] = (blk * 128 + 96 + lane < p.T) ? s3 : -INFINITY;
      }
      float mx = sc[0];
#pragma unroll
      for (int r = 1; r < 4 * TB; ++r) mx = fmaxf(mx, sc[r]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float sum = 0.f;
#pragma unroll
      for (int r = 0; r < 4 * TB; ++r) {
        sc[r] = expf(sc[r] - mx);
        sum += sc[r];
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      float o[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
      for (int blk = 0; blk < TB; ++blk) {
        if (TB != 1) {
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const int key = blk * 128 + i * 8 + kg;
            vv[i] = (key < p.T) ? __ldg(reinterpret_cast<const uint4*>(vb + static_cast<long long>(key) * 64)) : make_uint4(0u, 0u, 0u, 0u);
          }
        }
#pragma unroll
        for (int it = 0; it < 16; ++it) {              // key = blk*128 + it*8 + kg -> sc[blk*4 + (it>>2)], lane (it&3)*8 + kg
          const float pk = __shfl_sync(0xffffffffu, sc[blk * 4 + (it >> 2)], (it & 3) * 8 + kg);
          const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&vv[it]);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const float2 f = __bfloat1622float2(p2[e]);
            o[e * 2] = fmaf(pk, f.x, o[e * 2]);
            o[e * 2 + 1] = fmaf(pk, f.y, o[e * 2 + 1]);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        o[j] += __shfl_xor_sync(0xffffffffu, o[j], 4);
        o[j] += __shfl_xor_sync(0xffffffffu, o[j], 8);
        o[j] += __shfl_xor_sync(0xffffffffu, o[j], 16);
      }
      if (kg == 0) {
        const float inv = 1.0f / sum;
        uint4 q;
        q.x = pack_bf16(o[0] * inv, o[1] * inv); q.y = pack_bf16(o[2] * inv, o[3] * inv);
        q.z = pack_bf16(o[4] * inv, o[5] * inv); q.w = pack_bf16(o[6] * inv, o[7] * inv);
        *reinterpret_cast<uint4*>(p.ca + static_cast<long long>(b) * D + h * 32 + cc * 8) = q;
      }
    }
    DEC_PROF(7);
    grid_barrier(p.bar, target);
    DEC_PROF(8);
    // ---------------- P5: y += out_proj(ca) ----------------
    for (int tile = blockIdx.x; tile < mt * (D / 64); tile += gridDim.x)
      dec_tile<D, 4, false, DE_RMW>(p, dec_smem, p.ca, D, nullptr, nullptr, nullptr, p.Wo_c, D, D, p.bo_c, (tile / (D / 64)) * 64,
                                    (tile % (D / 64)) * 64, step);
    DEC_PROF(9);
    grid_barrier(p.bar, target);
    DEC_PROF(10);
    // ---------------- P6: hd = GELU(linear1(LN2(y))) ----------------
    {
      const int ntl = p.Md / 128;
      for (int tile = blockIdx.x; tile < mt * ntl; tile += gridDim.x)
        dec_tile<D, 8, true, DE_GELU>(p, dec_smem, nullptr, 0, p.y, p.g2, p.be2, p.W1, D, p.Md, p.b1, (tile / ntl) * 64,
                                      (tile % ntl) * 128, step);
    }
    DEC_PROF(11);
    grid_barrier(p.bar, target);
    DEC_PROF(12);
    // ---------------- P7: y += linear2(hd) ----------------
    {
      const int nt2 = D / 64, ks = p.Md / DEC_KSPLIT;       // K slice per split (multiple of 64)
      for (int tile = blockIdx.x; tile < mt * nt2 * DEC_KSPLIT; tile += gridDim.x) {
        const int sp = tile % DEC_KSPLIT, tn = (tile / DEC_KSPLIT) % nt2, tm = tile / (DEC_KSPLIT * nt2);
        dec_tile<D, 4, false, DE_PART>(p, dec_smem, p.hd + sp * ks, p.Md, nullptr, nullptr, nullptr, p.W2 + sp * ks, ks, D, p.b2,
                                       tm * 64, tn * 64, step, p.Md, sp);
      }
    }
    DEC_PROF(13);
    grid_barrier(p.bar, target);
    DEC_PROF(14);
    // ---------------- P8: logits[:, step] = head(LN3(y)); ids[:, step+1] = argmax ----------------
    {
      const int mt16 = (p.B + 15) / 16;
      for (int tile = blockIdx.x; tile < mt16; tile += gridDim.x)
        dec_tile<D, 2, true, DE_HEAD, 1>(p, dec_smem, nullptr, 0, p.y, p.g3, p.be3, p.Wh, D, p.C, p.bh, tile * 16, 0, step, 0, 0,
                                         p.part);
    }
    DEC_PROF(15);
    grid_barrier(p.bar, target);
  }
}

template <int D>
constexpr size_t dec_ar_smem_bytes() {
  return static_cast<size_t>((D / 64) * 4096 + DEC_STAGES * 4096 + DEC_STAGES * DEC_MAX_BN * 64) * 2 + 64 * 128 * 4;
}

}  // namespace pq
