// Non-GEMM kernels of the PARSeq path: patch gather (im2col), LayerNorm, ViT attention core,
// decoder two-stream self-attention over the (position, token) K/V table, cross-attention over the
// cached image K/V, greedy argmax / refine-context construction, early-exit step count.
#pragma once
#include "ptx.cuh"

namespace pq {

// ---------------------------------------------------------------------------------------------
// Patch gather: images fp32 NCHW [B,3,H,W] -> A_pe bf16 [B*T, Kp] with token t = r*gw + c and
// k = ch*ph*pw + dy*pw + dx  (Conv2d(3,D,k=s=patch) as a GEMM; timm PatchEmbed via modules.py:145-161).
// One thread per (token, ch, dy): reads pw contiguous floats, writes pw contiguous bf16.
__global__ void im2col_patch_kernel(const float* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H,
                                    int W, int ph, int pw, int gh, int gw) {
  grid_dep_launch();
  grid_dep_wait();
  const long long total = static_cast<long long>(B) * gh * gw * 3 * ph;
  const int Kp = 3 * ph * pw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    // order: b, r, dy, ch, c  -> consecutive threads walk along an image row (coalesced reads)
    long long t = i;
    const int c = static_cast<int>(t % gw); t /= gw;
    const int ch = static_cast<int>(t % 3); t /= 3;
    const int dy = static_cast<int>(t % ph); t /= ph;
    const int r = static_cast<int>(t % gh); t /= gh;
    const int b = static_cast<int>(t);
    const float* src = img + ((static_cast<long long>(b) * 3 + ch) * H + (r * ph + dy)) * W + c * pw;
    __nv_bfloat16* dst = out + (static_cast<long long>(b) * gh * gw + r * gw + c) * Kp + ch * ph * pw + dy * pw;
    if (pw == 8 && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0)) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(src));
      const float4 d = __ldg(reinterpret_cast<const float4*>(src) + 1);
      uint4 q;
      q.x = pack_bf16(a.x, a.y); q.y = pack_bf16(a.z, a.w);
      q.z = pack_bf16(d.x, d.y); q.w = pack_bf16(d.z, d.w);
      *reinterpret_cast<uint4*>(dst) = q;
    } else {
      for (int dx = 0; dx < pw; ++dx) dst[dx] = __float2bfloat16_rn(src[dx]);
    }
  }
}

// Same gather for raw uint8 HWC crops [B, H, W, 3] with the reference's input transform folded in:
// T.ToTensor() (u / 255) followed by T.Normalize(0.5, 0.5) ((x - 0.5) / 0.5)  (strhub/data/module.py:68-82), evaluated in
// fp32 with IEEE division exactly like torchvision, then rounded to bf16 like the float path.
__global__ void im2col_patch_u8_kernel(const uint8_t* __restrict__ img, __nv_bfloat16* __restrict__ out, int B, int H,
                                       int W, int ph, int pw, int gh, int gw) {
  grid_dep_launch();
  grid_dep_wait();
  const long long total = static_cast<long long>(B) * gh * gw * ph;     // one thread per (token, dy): pw*3 bytes
  const int Kp = 3 * ph * pw;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    long long t = i;
    const int c = static_cast<int>(t % gw); t /= gw;
    const int dy = static_cast<int>(t % ph); t /= ph;
    const int r = static_cast<int>(t % gh); t /= gh;
    const int b = static_cast<int>(t);
    const uint8_t* src = img + ((static_cast<long long>(b) * H + (r * ph + dy)) * W + c * pw) * 3;
    __nv_bfloat16* dst = out + (static_cast<long long>(b) * gh * gw + r * gw + c) * Kp + dy * pw;
    for (int dx = 0; dx < pw; ++dx) {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float x = __fdiv_rn(static_cast<float>(src[dx * 3 + ch]), 255.0f);
        dst[ch * ph * pw + dx] = __float2bfloat16_rn(__fdiv_rn(x - 0.5f, 0.5f));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// LayerNorm over the last dim (biased variance, two-pass in registers), one warp per row.
// y_bf16 = bf16(LN(x)); optional fp32 copy (encoder output `memory`).
// Optional pre-add: x_row += add[(row % add_mod)] (broadcast table, e.g. pos_queries) and the sum is written back
// to xw (the residual stream) before normalising - lets the producing GEMM use its plain TMA-store epilogue.
template <int D>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float eps, int M,
                                                        __nv_bfloat16* __restrict__ y, float* __restrict__ y32,
                                                        const float* __restrict__ add, int add_mod,
                                                        float* __restrict__ xw) {
  grid_dep_launch();
  grid_dep_wait();
  static_assert(D % 64 == 0, "D must be a multiple of 64");
  constexpr int NV = D / 64;  // float2 per lane
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= M) return;
  const int lane = threadIdx.x & 31;
  const float2* xr = reinterpret_cast<const float2*>(x + static_cast<long long>(row) * D);
  float2 v[NV];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) v[i] = xr[i * 32 + lane];
  if (add != nullptr) {
    const float2* ar = reinterpret_cast<const float2*>(add + static_cast<long long>(row % add_mod) * D);
    float2* wr = reinterpret_cast<float2*>(xw + static_cast<long long>(row) * D);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float2 a = __ldg(ar + i * 32 + lane);
      v[i].x += a.x;
      v[i].y += a.y;
      wr[i * 32 + lane] = v[i];
    }
  }
#pragma unroll
  for (int i = 0; i < NV; ++i) s += v[i].x + v[i].y;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.0f / D);
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float a = v[i].x - mean, b = v[i].y - mean;
    q += a * a + b * b;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = 1.0f / sqrtf(q * (1.0f / D) + eps);
  const float2* g2 = reinterpret_cast<const float2*>(gamma);
  const float2* b2 = reinterpret_cast<const float2*>(beta);
  uint32_t* yr = reinterpret_cast<uint32_t*>(y + static_cast<long long>(row) * D);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float2 g = __ldg(g2 + i * 32 + lane), b = __ldg(b2 + i * 32 + lane);
    const float o0 = (v[i].x - mean) * rstd * g.x + b.x;
    const float o1 = (v[i].y - mean) * rstd * g.y + b.y;
    yr[i * 32 + lane] = pack_bf16(o0, o1);
    if (y32 != nullptr) reinterpret_cast<float2*>(y32 + static_cast<long long>(row) * D)[i * 32 + lane] = make_float2(o0, o1);
  }
}

// ---------------------------------------------------------------------------------------------
// ViT attention core for T = 128 tokens, head dim 64 (timm Attention: softmax(QK^T / 8) V, no mask).
// One CTA per (image, head), 8 warps x 16 query rows.  Q/K/V tiles (128x64 bf16) are staged in
// XOR-swizzled shared memory with cp.async; S = QK^T and O = PV run on mma.sync m16n8k16 with the
// probabilities kept in registers (bf16 A fragments), fp32 row statistics, O/rowsum -> bf16.
constexpr int ATT_T = 128;
constexpr int ATT_DH = 64;
__device__ __forceinline__ uint32_t att_swz(int r, int c) {  // element offset of (row r, col c), c%8==0 chunks
  return static_cast<uint32_t>(r * ATT_DH + ((((c >> 3) ^ (r & 7)) << 3) | (c & 7)));
}
// The arithmetic of one (image, head) once its Q/K/V tiles (att_swz layout) are in shared memory: warp `warp` (0..7) of
// the 8 that run it computes query rows [16 warp, 16 warp + 16) and stores them to obase (row pitch D elements).  The
// warp's rows of sQ are overwritten (output staging); sK / sV are only read.  Shared by enc_attention_kernel and the
// fused QKV + attention kernel (qkv_attn.cuh), so both compute the same bits.
__device__ __forceinline__ void att_tile_128(__nv_bfloat16* sQ, const __nv_bfloat16* sK, const __nv_bfloat16* sV,
                                             __nv_bfloat16* __restrict__ obase, int D, int warp, int lane) {
  const int r0 = warp * 16;
  // ---- Q fragments for the 4 k-steps over d ----
  uint32_t qf[4][4];
#pragma unroll
  for (int kt = 0; kt < 4; ++kt) {
    const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int col = kt * 16 + (lane >> 4) * 8;
    ldmatrix_x4(smem_u32(sQ + att_swz(row, col)), qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3]);
  }
  // ---- S = Q K^T : 16 n-tiles of 8 keys ----
  float sacc[16][4];
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) { sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.f; }
#pragma unroll
  for (int kt = 0; kt < 4; ++kt) {
#pragma unroll
    for (int np = 0; np < 8; ++np) {
      const int key = np * 16 + (lane & 7) + (lane >> 4) * 8;
      const int col = kt * 16 + ((lane >> 3) & 1) * 8;
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4(smem_u32(sK + att_swz(key, col)), b0, b1, b2, b3);
      mma_bf16_16816(sacc[2 * np], qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3], b0, b1);
      mma_bf16_16816(sacc[2 * np + 1], qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3], b2, b3);
    }
  }
  // ---- softmax over 128 keys; rows g (c0,c1) and g+8 (c2,c3) ----
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    mx0 = fmaxf(mx0, fmaxf(sacc[nt][0], sacc[nt][1]));
    mx1 = fmaxf(mx1, fmaxf(sacc[nt][2], sacc[nt][3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;  // d^-0.5 * log2(e)
  float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
  for (int nt = 0; nt < 16; ++nt) {
    sacc[nt][0] = exp2f((sacc[nt][0] - mx0) * kScaleLog2);
    sacc[nt][1] = exp2f((sacc[nt][1] - mx0) * kScaleLog2);
    sacc[nt][2] = exp2f((sacc[nt][2] - mx1) * kScaleLog2);
    sacc[nt][3] = exp2f((sacc[nt][3] - mx1) * kScaleLog2);
    sum0 += sacc[nt][0] + sacc[nt][1];
    sum1 += sacc[nt][2] + sacc[nt][3];
  }
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
  // ---- O = P V : 8 k-steps over keys, 8 n-tiles over d ----
  float oacc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) { oacc[nt][0] = oacc[nt][1] = oacc[nt][2] = oacc[nt][3] = 0.f; }
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) {
    const uint32_t a0 = pack_bf16(sacc[2 * kk][0], sacc[2 * kk][1]);
    const uint32_t a1 = pack_bf16(sacc[2 * kk][2], sacc[2 * kk][3]);
    const uint32_t a2 = pack_bf16(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1]);
    const uint32_t a3 = pack_bf16(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3]);
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      const int key = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
      const int col = np * 16 + (lane >> 4) * 8;
      uint32_t b0, b1, b2, b3;
      ldmatrix_x4_trans(smem_u32(sV + att_swz(key, col)), b0, b1, b2, b3);
      mma_bf16_16816(oacc[2 * np], a0, a1, a2, a3, b0, b1);
      mma_bf16_16816(oacc[2 * np + 1], a0, a1, a2, a3, b2, b3);
    }
  }
  // ---- normalise, stage through this warp's (now dead) Q rows, coalesced 16-B stores ----
  const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
  const int g = lane >> 2, t = lane & 3;
  __syncwarp();
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int col = nt * 8 + 2 * t;
    *reinterpret_cast<uint32_t*>(sQ + att_swz(r0 + g, col)) = pack_bf16(oacc[nt][0] * inv0, oacc[nt][1] * inv0);
    *reinterpret_cast<uint32_t*>(sQ + att_swz(r0 + g + 8, col)) = pack_bf16(oacc[nt][2] * inv1, oacc[nt][3] * inv1);
  }
  __syncwarp();
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = i * 32 + lane;       // 16 rows x 8 chunks
    const int r = r0 + (idx >> 3), ck = idx & 7;
    const uint4 val = *reinterpret_cast<const uint4*>(sQ + att_swz(r, ck * 8));
    *reinterpret_cast<uint4*>(obase + static_cast<long long>(r) * D + ck * 8) = val;
  }
}

__global__ void __launch_bounds__(256, 2) enc_attention_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                            __nv_bfloat16* __restrict__ out, int D, int heads) {
  grid_dep_launch();
  grid_dep_wait();
  __shared__ __align__(128) __nv_bfloat16 sQ[ATT_T * ATT_DH];
  __shared__ __align__(128) __nv_bfloat16 sK[ATT_T * ATT_DH];
  __shared__ __align__(128) __nv_bfloat16 sV[ATT_T * ATT_DH];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ld = 3ll * D;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * ATT_T * ld + h * ATT_DH;
  // 3 matrices x 128 rows x 8 chunks of 16 B
  for (int i = tid; i < 3 * ATT_T * 8; i += 256) {
    const int m = i / (ATT_T * 8);
    const int r = (i / 8) % ATT_T;
    const int ck = i % 8;
    const __nv_bfloat16* src = base + static_cast<long long>(r) * ld + m * D + ck * 8;
    __nv_bfloat16* dstm = (m == 0) ? sQ : (m == 1) ? sK : sV;
    cp_async_16(smem_u32(dstm + att_swz(r, ck * 8)), src);
  }
  cp_async_wait_all();
  __syncthreads();
  att_tile_128(sQ, sK, sV, out + static_cast<long long>(b) * ATT_T * D + h * ATT_DH, D, warp, lane);
}

// ---------------------------------------------------------------------------------------------
// ViT attention core for ANY token count T (e.g. 196 = 224x224/16x16, 240 = 48x160/4x8), head dim 64: correctness
// path for the geometries that do not fill one 128-row tile per image (the T = 128 fast path is attn_tc.cuh).
// grid = (B*heads, ceil(T/128)): one CTA per 128-query tile; keys are visited in blocks of 128 in two passes
// (pass 1: row maxima, pass 2: P = exp(S - max), O += P V) so the rounding points equal the single-tile kernel's.
// Rows / keys >= T are masked; same mma.sync fragment scheme as enc_attention_kernel.
__global__ void __launch_bounds__(256, 2) enc_attention_any_kernel(const __nv_bfloat16* __restrict__ qkv,
                                                                   __nv_bfloat16* __restrict__ out, int T, int D,
                                                                   int heads) {
  grid_dep_launch();
  grid_dep_wait();
  __shared__ __align__(128) __nv_bfloat16 sQ[ATT_T * ATT_DH];
  __shared__ __align__(128) __nv_bfloat16 sK[ATT_T * ATT_DH];
  __shared__ __align__(128) __nv_bfloat16 sV[ATT_T * ATT_DH];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * ATT_T;                         // first query row of this tile
  const int nkb = (T + ATT_T - 1) / ATT_T;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long ld = 3ll * D;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * T * ld + h * ATT_DH;
  auto load_tile = [&](__nv_bfloat16* dst, int mat, int row0, int nrows) {   // rows clamped to T-1 (masked later)
    for (int i = tid; i < nrows * 8; i += 256) {
      const int r = i >> 3, ck = i & 7;
      int row = row0 + r;
      if (row >= T) row = T - 1;
      cp_async_16(smem_u32(dst + att_swz(r, ck * 8)), base + static_cast<long long>(row) * ld + mat * D + ck * 8);
    }
  };
  load_tile(sQ, 0, q0, ATT_T);
  cp_async_wait_all();
  __syncthreads();
  const int r0 = warp * 16;
  const bool active = (q0 + r0) < T;     // warp-uniform: a warp whose 16 query rows are all padding only helps loading
  uint32_t qf[4][4];
#pragma unroll
  for (int kt = 0; kt < 4; ++kt) {
    const int row = r0 + (lane & 7) + ((lane >> 3) & 1) * 8;
    const int col = kt * 16 + (lane >> 4) * 8;
    ldmatrix_x4(smem_u32(sQ + att_swz(row, col)), qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3]);
  }
  const int t4 = lane & 3;
  constexpr float kScaleLog2 = 0.125f * 1.4426950408889634f;
  float mx0 = -INFINITY, mx1 = -INFINITY, sum0 = 0.f, sum1 = 0.f;
  float oacc[8][4];
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) { oacc[nt][0] = oacc[nt][1] = oacc[nt][2] = oacc[nt][3] = 0.f; }
  for (int pass = 0; pass < 2; ++pass) {
    for (int kb = 0; kb < nkb; ++kb) {
      __syncthreads();                                       // previous tile fully consumed
      // only the 16-key groups that hold at least one real key are loaded and multiplied (T = 129: 1 of 8 in block 1)
      const int nvalid = (T - kb * ATT_T < ATT_T) ? (T - kb * ATT_T) : ATT_T;
      const int np_max = (nvalid + 15) >> 4;
      load_tile(sK, 1, kb * ATT_T, np_max * 16);
      if (pass == 1) load_tile(sV, 2, kb * ATT_T, np_max * 16);
      cp_async_wait_all();
      __syncthreads();
      if (!active) continue;
      float sacc[16][4];
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) { sacc[nt][0] = sacc[nt][1] = sacc[nt][2] = sacc[nt][3] = 0.f; }
#pragma unroll
      for (int kt = 0; kt < 4; ++kt) {
#pragma unroll
        for (int np = 0; np < 8; ++np) {
          if (np >= np_max) break;
          const int key = np * 16 + (lane & 7) + (lane >> 4) * 8;
          const int col = kt * 16 + ((lane >> 3) & 1) * 8;
          uint32_t b0, b1, b2, b3;
          ldmatrix_x4(smem_u32(sK + att_swz(key, col)), b0, b1, b2, b3);
          mma_bf16_16816(sacc[2 * np], qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3], b0, b1);
          mma_bf16_16816(sacc[2 * np + 1], qf[kt][0], qf[kt][1], qf[kt][2], qf[kt][3], b2, b3);
        }
      }
      // mask keys >= T (columns 8*nt + 2*t4, +1 of this key block)
#pragma unroll
      for (int nt = 0; nt < 16; ++nt) {
        const int k0 = kb * ATT_T + nt * 8 + 2 * t4;
        if (k0 >= T) { sacc[nt][0] = -INFINITY; sacc[nt][2] = -INFINITY; }
        if (k0 + 1 >= T) { sacc[nt][1] = -INFINITY; sacc[nt][3] = -INFINITY; }
      }
      if (pass == 0) {
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
          mx0 = fmaxf(mx0, fmaxf(sacc[nt][0], sacc[nt][1]));
          mx1 = fmaxf(mx1, fmaxf(sacc[nt][2], sacc[nt][3]));
        }
      } else {
#pragma unroll
        for (int nt = 0; nt < 16; ++nt) {
          sacc[nt][0] = exp2f((sacc[nt][0] - mx0) * kScaleLog2);
          sacc[nt][1] = exp2f((sacc[nt][1] - mx0) * kScaleLog2);
          sacc[nt][2] = exp2f((sacc[nt][2] - mx1) * kScaleLog2);
          sacc[nt][3] = exp2f((sacc[nt][3] - mx1) * kScaleLog2);
          sum0 += sacc[nt][0] + sacc[nt][1];
          sum1 += sacc[nt][2] + sacc[nt][3];
        }
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          if (kk >= np_max) break;           // P is exactly 0 on the padded keys
          const uint32_t a0 = pack_bf16(sacc[2 * kk][0], sacc[2 * kk][1]);
          const uint32_t a1 = pack_bf16(sacc[2 * kk][2], sacc[2 * kk][3]);
          const uint32_t a2 = pack_bf16(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1]);
          const uint32_t a3 = pack_bf16(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3]);
#pragma unroll
          for (int np = 0; np < 4; ++np) {
            const int key = kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
            const int col = np * 16 + (lane >> 4) * 8;
            uint32_t b0, b1, b2, b3;
            ldmatrix_x4_trans(smem_u32(sV + att_swz(key, col)), b0, b1, b2, b3);
            mma_bf16_16816(oacc[2 * np], a0, a1, a2, a3, b0, b1);
            mma_bf16_16816(oacc[2 * np + 1], a0, a1, a2, a3, b2, b3);
          }
        }
      }
    }
    if (pass == 0) {
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
      mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
      mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    }
  }
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1);
  sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1);
  sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
  const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
  const int g = lane >> 2;
  __nv_bfloat16* obase = out + static_cast<long long>(b) * T * D + h * ATT_DH;
  const int row_lo = q0 + r0 + g, row_hi = row_lo + 8;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt) {
    const int col = nt * 8 + 2 * t4;
    if (row_lo < T) *reinterpret_cast<uint32_t*>(obase + static_cast<long long>(row_lo) * D + col) = pack_bf16(oacc[nt][0] * inv0, oacc[nt][1] * inv0);
    if (row_hi < T) *reinterpret_cast<uint32_t*>(obase + static_cast<long long>(row_hi) * D + col) = pack_bf16(oacc[nt][2] * inv1, oacc[nt][3] * inv1);
  }
}

// ---------------------------------------------------------------------------------------------
// Decoder context rows for the (position, token) K/V table:
//   ctx[pos*V + tok] = sqrt(D)*E[tok] + (pos >= 1 ? pos_queries[pos-1] : 0)     (model.py:94-99, modules.py:175-176)
__global__ void build_ctx_rows_kernel(const float* __restrict__ emb, const float* __restrict__ posq, float* __restrict__ ctx,
                                      int L, int V, int D, float sqrtD) {
  const long long total = static_cast<long long>(L) * V * D;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % D);
    const int tok = static_cast<int>((i / D) % V);
    const int pos = static_cast<int>(i / (static_cast<long long>(D) * V));
    float v = sqrtD * emb[static_cast<long long>(tok) * D + c];
    if (pos >= 1) v = posq[static_cast<long long>(pos - 1) * D + c] + v;
    ctx[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Greedy argmax (torch.argmax semantics: first NaN, else first maximum; ptx.cuh) of logits rows -> token ids.
// One warp per row.  Row r = (b, s): reads logits[b, src_pos0 + s, :C], writes ids[b*ids_ld + dst_pos0 + s].
// If `forced` != nullptr the written id is forced[b*forced_ld + dst_pos0 + s] (teacher forcing).
// If `mask` != nullptr (class allowlist rows of the B images, ptx.cuh class_allowed) the disallowed logits of the row are
// set to -inf in place before the argmax; `ids` may then be nullptr (masking only).
__global__ void argmax_rows_kernel(float* __restrict__ logits, int L, int C, int B, int nrows_per_b, int src_pos0,
                                   int* __restrict__ ids, int ids_ld, int dst_pos0, const int* __restrict__ forced,
                                   int forced_ld, const uint32_t* __restrict__ mask) {
  grid_dep_launch();
  grid_dep_wait();
  const int w = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (w >= B * nrows_per_b) return;
  const int lane = threadIdx.x & 31;
  const int b = w / nrows_per_b, s = w % nrows_per_b;
  float* row = logits + (static_cast<long long>(b) * L + src_pos0 + s) * C;
  float best = -INFINITY;
  int bi = ARGMAX_NONE;
  if (mask != nullptr) {
    const uint32_t* mrow = mask + static_cast<long long>(b) * class_mask_words(C);
    for (int j = lane; j < C; j += 32) {
      float v = row[j];
      if (!class_allowed(mrow, j)) { v = -INFINITY; row[j] = v; }   // argmax_finish below re-reads this lane's columns
      argmax_scan(best, bi, v, j);
    }
  } else {
    for (int j = lane; j < C; j += 32) argmax_scan(best, bi, row[j], j);
  }
  bi = argmax_finish(best, bi, row, C, lane);
  if (lane == 0 && ids != nullptr) {
    int v = bi;
    if (forced != nullptr) v = forced[static_cast<long long>(b) * forced_ld + dst_pos0 + s];
    ids[static_cast<long long>(b) * ids_ld + dst_pos0 + s] = v;
  }
}

__global__ void fill_ids_kernel(int* __restrict__ ids, int B, int ld, int bos, int pad) {
  grid_dep_launch();
  grid_dep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * ld) ids[i] = ((i % ld) == 0) ? bos : pad;
}

// S = number of AR steps the reference returns under its batch-wide early exit (model.py:144):
// smallest j>=1 such that every row has an EOS among ids[b,1..j]  == max_b first_eos_pos(b); L if any row has none.
__global__ void ar_steps_kernel(const int* __restrict__ ids, int ids_ld, int B, int L, int eos_id, int* __restrict__ steps) {
  grid_dep_launch();
  grid_dep_wait();
  int worst = 0;
  for (int b = threadIdx.x; b < B; b += blockDim.x) {
    int first = L;
    for (int j = 1; j < L; ++j)
      if (ids[static_cast<long long>(b) * ids_ld + j] == eos_id) { first = j; break; }
    worst = max(worst, first);
  }
  atomicMax(steps, worst);
}
__global__ void set_int_kernel(int* p, int v) {
  grid_dep_launch();
  grid_dep_wait(); if (threadIdx.x == 0 && blockIdx.x == 0) *p = v; }

// ---------------------------------------------------------------------------------------------
// Decoder self-attention, one CTA per image, one warp per head (head dim 32), ALL nq queries of the pass:
// the context K rows (lane = key, KPL keys per lane: key lane + 32 u) and V columns (lane = channel) of the head are
// gathered once from the (position, token) table into registers, then every query costs ~130 warp instructions per
// 32 keys.  KPL = 1 holds up to 32 keys (L <= 32), KPL = 2 up to 64 (labels of up to 63 characters).
// (DecoderLayer.forward_stream step 1, modules.py:69-72)
//   q      : Qs[qpos] fp32 (W_q LN_q(pos_queries[qpos]) + b, pre-scaled by 1/sqrt(32); input independent)
//   K/V    : kvtab[(k*V + ids[b,k]) * 2D + {0, D} + c] bf16   (the content stream is a function of
//            (position, token) only at decoder depth 1)
//   mask   : mode 0 (AR step / NAR): keys 0..nkeys-1 all visible (model.py:130-136: the sliced causal row is
//            all-False);  mode 1 (cloze refine): key k masked iff k == q+1 or an EOS occurs in ids[b, 0..k]
//            (model.py:157,163)
// out bf16 [B*nq, D] (A operand of the out-projection GEMM).
//            mode 2 (PARSeq.decode with caller-supplied masks, model.py:86-103): Qs holds one query row per (image,
//            query) [B*nq, D]; key k of query qi is masked iff qmask[qi*nkeys + k] or pmask[b*nkeys + k] (either may be
//            null); a row with every key masked yields NaN, as torch's softmax over -inf does
//            QROW (decoders of depth >= 2): Qs holds one query row per (image, query) [B*nq, D] in every mode
//            CACHE (decoders of depth >= 2): K/V rows come from a per-image cache [B, V, 2D] (V = key rows per image),
//            row b * V + k, instead of the (position, token) table
template <int KPL, bool QROW = false, bool CACHE = false>
__device__ __forceinline__ void dec_self_attn2_body(const float* __restrict__ Qs, const __nv_bfloat16* __restrict__ kvtab,
                                                    const int* __restrict__ ids, int ids_ld, int V, int D, int nq, int q0,
                                                    int nkeys, int mode, int eos_id, __nv_bfloat16* __restrict__ out,
                                                    int qsplit, const unsigned char* __restrict__ qmask,
                                                    const unsigned char* __restrict__ pmask) {
  constexpr int NK = 32 * KPL;                          // keys held by one warp
  // grid = B * qsplit: CTA (b, part) handles queries [part*nq/qsplit, (part+1)*nq/qsplit) of image b
  __shared__ int s_ids[NK];
  __shared__ unsigned s_eos[KPL];                       // EOS ballot of each 32-key group (KPL > 1)
  __shared__ int s_first_eos;
  grid_dep_launch();
  grid_dep_wait();
  const int b = blockIdx.x / qsplit, part = blockIdx.x % qsplit;
  const int q_begin = (part * nq) / qsplit, q_end = ((part + 1) * nq) / qsplit;
  const int lane = threadIdx.x & 31;
  const int heads = D >> 5, nwarps = blockDim.x >> 5;   // blockDim.x = min(D, 384): heads are looped when D > 384
  if (threadIdx.x < NK) {
    const int id = (threadIdx.x < nkeys) ? ids[static_cast<long long>(b) * ids_ld + threadIdx.x] : -1;
    s_ids[threadIdx.x] = id;
    const unsigned m = __ballot_sync(0xffffffffu, id == eos_id);
    if constexpr (KPL == 1) {
      if (threadIdx.x == 0) s_first_eos = (m != 0u) ? (__ffs(m) - 1) : (1 << 30);
    } else {
      if (lane == 0) s_eos[threadIdx.x >> 5] = m;
    }
  }
  __syncthreads();
  if constexpr (KPL > 1) {                              // the first EOS is in the first group whose ballot is not empty
    if (threadIdx.x == 0) {
      int f = 1 << 30;
#pragma unroll
      for (int u = KPL - 1; u >= 0; --u)
        if (s_eos[u] != 0u) f = 32 * u + __ffs(s_eos[u]) - 1;
      s_first_eos = f;
    }
    __syncthreads();
  }
  const int first_eos = s_first_eos;
  for (int h = threadIdx.x >> 5; h < heads; h += nwarps) {
  float kreg[KPL][32], vreg[NK];
#pragma unroll
  for (int u = 0; u < KPL; ++u) {
    const int key = lane + 32 * u;
    if (key < nkeys) {
      const long long kvrow = CACHE ? static_cast<long long>(b) * V + key : static_cast<long long>(key) * V + s_ids[key];
      const uint4* kr = reinterpret_cast<const uint4*>(kvtab + kvrow * 2 * D + h * 32);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 w = __ldg(kr + j);
        const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&w);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 f = __bfloat1622float2(p2[e]);
          kreg[u][j * 8 + e * 2] = f.x;
          kreg[u][j * 8 + e * 2 + 1] = f.y;
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) kreg[u][j] = 0.f;
    }
  }
#pragma unroll
  for (int k = 0; k < NK; ++k)
    vreg[k] = (k < nkeys) ? __bfloat162float(kvtab[(CACHE ? static_cast<long long>(b) * V + k : static_cast<long long>(k) * V + s_ids[k]) * 2 * D + D + h * 32 + lane]) : 0.f;
  for (int qi = q_begin; qi < q_end; ++qi) {
    const int qpos = q0 + qi;
    const long long qrow = (QROW || mode == 2) ? (static_cast<long long>(b) * nq + qi) : qpos;
    const float qv = __ldg(Qs + qrow * D + h * 32 + lane);   // lane j holds q_j
    float acc = 0.f;
    if constexpr (KPL == 1) {
      float s = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) s = fmaf(__shfl_sync(0xffffffffu, qv, j), kreg[0][j], s);
      bool masked = (lane >= nkeys) || ((mode == 1) && (lane == qpos + 1 || lane >= first_eos));
      if (mode == 2 && lane < nkeys) {
        if (qmask != nullptr && qmask[qi * nkeys + lane] != 0) masked = true;
        if (pmask != nullptr && pmask[static_cast<long long>(b) * nkeys + lane] != 0) masked = true;
      }
      if (masked) s = -INFINITY;
      float mx = s;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float e = masked ? 0.f : expf(s - mx);
      float sum = e;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float pme = e / sum;
#pragma unroll
      for (int k = 0; k < 32; ++k) acc = fmaf(__shfl_sync(0xffffffffu, pme, k), vreg[k], acc);
    } else {
      // scores of keys lane and lane + 32 (and so on), one shared max / sum over all of them
      float s[KPL];
#pragma unroll
      for (int u = 0; u < KPL; ++u) s[u] = 0.f;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const float qj = __shfl_sync(0xffffffffu, qv, j);
#pragma unroll
        for (int u = 0; u < KPL; ++u) s[u] = fmaf(qj, kreg[u][j], s[u]);
      }
      bool masked[KPL];
#pragma unroll
      for (int u = 0; u < KPL; ++u) {
        const int key = lane + 32 * u;
        masked[u] = (key >= nkeys) || ((mode == 1) && (key == qpos + 1 || key >= first_eos));
        if (mode == 2 && key < nkeys) {
          if (qmask != nullptr && qmask[qi * nkeys + key] != 0) masked[u] = true;
          if (pmask != nullptr && pmask[static_cast<long long>(b) * nkeys + key] != 0) masked[u] = true;
        }
        if (masked[u]) s[u] = -INFINITY;
      }
      float mx = s[0];
#pragma unroll
      for (int u = 1; u < KPL; ++u) mx = fmaxf(mx, s[u]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      float e[KPL];
#pragma unroll
      for (int u = 0; u < KPL; ++u) e[u] = masked[u] ? 0.f : expf(s[u] - mx);
      float sum = e[0];
#pragma unroll
      for (int u = 1; u < KPL; ++u) sum += e[u];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
#pragma unroll
      for (int u = 0; u < KPL; ++u) {
        const float pme = e[u] / sum;
#pragma unroll
        for (int k = 0; k < 32; ++k) acc = fmaf(__shfl_sync(0xffffffffu, pme, k), vreg[u * 32 + k], acc);
      }
    }
    out[(static_cast<long long>(b) * nq + qi) * D + h * 32 + lane] = __float2bfloat16_rn(acc);
  }
  }
}
// up to 32 keys (L <= 32)
__global__ void dec_self_attn2_kernel(const float* __restrict__ Qs, const __nv_bfloat16* __restrict__ kvtab,
                                      const int* __restrict__ ids, int ids_ld, int V, int D, int nq, int q0, int nkeys,
                                      int mode, int eos_id, __nv_bfloat16* __restrict__ out, int qsplit,
                                      const unsigned char* __restrict__ qmask = nullptr,
                                      const unsigned char* __restrict__ pmask = nullptr) {
  dec_self_attn2_body<1>(Qs, kvtab, ids, ids_ld, V, D, nq, q0, nkeys, mode, eos_id, out, qsplit, qmask, pmask);
}
// up to 64 keys (labels of up to 63 characters); 384 threads at most, so that K and V of 64 keys stay in registers
__global__ void __launch_bounds__(384) dec_self_attn2_long_kernel(
    const float* __restrict__ Qs, const __nv_bfloat16* __restrict__ kvtab, const int* __restrict__ ids, int ids_ld, int V,
    int D, int nq, int q0, int nkeys, int mode, int eos_id, __nv_bfloat16* __restrict__ out, int qsplit,
    const unsigned char* __restrict__ qmask = nullptr, const unsigned char* __restrict__ pmask = nullptr) {
  dec_self_attn2_body<2>(Qs, kvtab, ids, ids_ld, V, D, nq, q0, nkeys, mode, eos_id, out, qsplit, qmask, pmask);
}

// Decoders of depth >= 2: one query row per (image, query) - the content stream's own rows, or the query stream of a
// layer >= 1 - over the (position, token) table (CACHE = false: layer 0) or a per-image K/V cache (CACHE = true)
template <bool CACHE>
__global__ void dec_self_attn2_rows_kernel(const float* __restrict__ Qs, const __nv_bfloat16* __restrict__ kv,
                                           const int* __restrict__ ids, int ids_ld, int V, int D, int nq, int q0, int nkeys,
                                           int mode, int eos_id, __nv_bfloat16* __restrict__ out, int qsplit,
                                           const unsigned char* __restrict__ qmask, const unsigned char* __restrict__ pmask) {
  dec_self_attn2_body<1, true, CACHE>(Qs, kv, ids, ids_ld, V, D, nq, q0, nkeys, mode, eos_id, out, qsplit, qmask, pmask);
}
template <bool CACHE>
__global__ void __launch_bounds__(384) dec_self_attn2_rows_long_kernel(
    const float* __restrict__ Qs, const __nv_bfloat16* __restrict__ kv, const int* __restrict__ ids, int ids_ld, int V,
    int D, int nq, int q0, int nkeys, int mode, int eos_id, __nv_bfloat16* __restrict__ out, int qsplit,
    const unsigned char* __restrict__ qmask, const unsigned char* __restrict__ pmask) {
  dec_self_attn2_body<2, true, CACHE>(Qs, kv, ids, ids_ld, V, D, nq, q0, nkeys, mode, eos_id, out, qsplit, qmask, pmask);
}
// Layer-0 content rows of context positions [k0, k0 + nc) of B images (the rows build_ctx_rows_kernel puts into the
// K/V table, same arithmetic): x[b * nc + c] = sqrt(D) E[ids[b, k]] + (k >= 1 ? pos_queries[k - 1] : 0), k = k0 + c
__global__ void gather_ctx_rows_kernel(const float* __restrict__ emb, const float* __restrict__ posq, const int* __restrict__ ids,
                                       int ids_ld, int B, int k0, int nc, int D, float sqrtD, float* __restrict__ x) {
  grid_dep_launch();
  grid_dep_wait();
  const long long total = static_cast<long long>(B) * nc * D;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % D);
    const long long row = i / D;
    const int k = k0 + static_cast<int>(row % nc);
    const int tok = ids[(row / nc) * ids_ld + k];
    float v = sqrtD * emb[static_cast<long long>(tok) * D + c];
    if (k >= 1) v = posq[static_cast<long long>(k - 1) * D + c] + v;
    x[i] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// Decoder cross-attention over the cached image K/V, head dim 32.  The pieces below are shared by the three kernels
// that compute a cross-attention row's probabilities, so that they are computed one way: dec_cross_attn3_kernel (the
// decoder's passes), dec_cross_attn3_grouped_kernel (candidate scoring) and dec_cross_attn_maps_kernel (the maps, which
// must be bitwise the probabilities the P.V of the other two uses).
// kv: column-blocked cross K/V cache [2D/64][kv_rows][64] (ptx.cuh: blocked_off), row = image * T + key.

// Stages head h's K of keys [0, 32 * NR) of the image whose first cache row is row_b into sK (bf16x2 words, pitch 17:
// odd, so that lane = key reads are conflict-free), and with V its V into sV [32 * NR][32]; keys >= T are zero.
template <int NR, int NT, bool V>
__device__ __forceinline__ void cross_stage_kv(uint32_t* sK, __nv_bfloat16* sV, const __nv_bfloat16* __restrict__ kv,
                                               long long kv_rows, long long row_b, int T, int D, int h, int tid) {
  for (int t = tid; t < 32 * NR; t += NT) {
    if (t < T) {
      const uint4* kr = reinterpret_cast<const uint4*>(kv + blocked_off(kv_rows, row_b + t, h * 32));
      const uint4* vr = reinterpret_cast<const uint4*>(kv + blocked_off(kv_rows, row_b + t, D + h * 32));
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint4 u = __ldg(kr + j);
        sK[t * 17 + j * 4 + 0] = u.x; sK[t * 17 + j * 4 + 1] = u.y;
        sK[t * 17 + j * 4 + 2] = u.z; sK[t * 17 + j * 4 + 3] = u.w;
        if (V) reinterpret_cast<uint4*>(sV + t * 32)[j] = __ldg(vr + j);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j) sK[t * 17 + j] = 0u;
      if (V) {
#pragma unroll
        for (int j = 0; j < 4; ++j) reinterpret_cast<uint4*>(sV + t * 32)[j] = make_uint4(0u, 0u, 0u, 0u);
      }
    }
  }
}

// One query row against the staged keys (qv: lane j holds q_j): sc[r] = exp(s - max) of key r * 32 + lane (0 for keys
// >= T), in a fixed fmaf order over the 16 bf16x2 words; returns the xor-shuffle sum of the exponentials.
template <int NR>
__device__ __forceinline__ float cross_row_exp(const uint32_t* sK, float qv, int T, int lane, float (&sc)[NR]) {
#pragma unroll
  for (int r = 0; r < NR; ++r) sc[r] = 0.f;
#pragma unroll
  for (int w = 0; w < 16; ++w) {
    const float qa = __shfl_sync(0xffffffffu, qv, 2 * w), qb = __shfl_sync(0xffffffffu, qv, 2 * w + 1);
#pragma unroll
    for (int r = 0; r < NR; ++r) {
      const uint32_t kw = sK[(r * 32 + lane) * 17 + w];
      sc[r] = fmaf(qb, __uint_as_float(kw & 0xffff0000u), fmaf(qa, __uint_as_float(kw << 16), sc[r]));
    }
  }
  float mx = -INFINITY;
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    if (r * 32 + lane >= T) sc[r] = -INFINITY;
    mx = fmaxf(mx, sc[r]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int r = 0; r < NR; ++r) {
    sc[r] = expf(sc[r] - mx);
    sum += sc[r];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  return sum;
}

// out[0, 32) = bf16(sum_k sc_k v_k / sum) of one row.  P.V with 16-byte smem reads: lane = (key group kg = lane>>2,
// 8-channel chunk cc = lane&3); 4*NR iterations cover the keys; the 8 key groups are then summed with xor-shuffles and
// lanes 0..3 hold the 32 output channels.
template <int NR>
__device__ __forceinline__ void cross_row_pv(const __nv_bfloat16* sV, const float (&sc)[NR], float sum, int lane,
                                             __nv_bfloat16* __restrict__ out) {
  const int kg = lane >> 2, cc = lane & 3;
  float o[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = 0.f;
#pragma unroll
  for (int it = 0; it < 4 * NR; ++it) {              // key = it*8 + kg -> register sc[it>>2], source lane (it&3)*8 + kg
    const int key = it * 8 + kg;
    const uint4 vvv = *reinterpret_cast<const uint4*>(sV + key * 32 + cc * 8);
    const float pk = __shfl_sync(0xffffffffu, sc[it >> 2], (it & 3) * 8 + kg);
    const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&vvv);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float2 f = __bfloat1622float2(p2[e]);
      o[e * 2] = fmaf(pk, f.x, o[e * 2]);
      o[e * 2 + 1] = fmaf(pk, f.y, o[e * 2 + 1]);
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
    uint4 q4;
    q4.x = pack_bf16(o[0] * inv, o[1] * inv); q4.y = pack_bf16(o[2] * inv, o[3] * inv);
    q4.z = pack_bf16(o[4] * inv, o[5] * inv); q4.w = pack_bf16(o[6] * inv, o[7] * inv);
    *reinterpret_cast<uint4*>(out + cc * 8) = q4;
  }
}

// One CTA per (image, head), 4 warps.  The head's K and V tiles are staged once in shared memory, so the per-image K/V
// cache is read once per decode pass; the query rows are distributed over the warps and each row is handled entirely
// inside one warp (scores for NR keys per lane, shuffle softmax, P.V): no block-level synchronisation after the load.
// q fp32 [rows, D] pre-scaled by 1/sqrt(32); out bf16 [rows, D]; the rows of this launch belong to images b_first,
// b_first + 1, ...
// GROUPED (candidate scoring): the query rows of image b_first + j are rows [cand_off[j] * nq, cand_off[j + 1] * nq)
// (candidates are image-major, nq rows each); CTA (j * heads + h, y) serves rows [y * rows_per_cta, (y + 1) *
// rows_per_cta) of the image, grid.y covering the image with the most rows.  Otherwise image j's rows are
// [j * nq, (j + 1) * nq).  Every row is computed the same way in both, so its bits do not depend on how many candidates
// share its image.
template <int NR, bool GROUPED>
__device__ __forceinline__ void dec_cross_attn3_body(const float* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                                                     long long kv_rows, int b_first, int T, int D, int heads, int nq,
                                                     const int* __restrict__ cand_off, int rows_per_cta,
                                                     __nv_bfloat16* __restrict__ out) {
  constexpr int TK = 32 * NR;
  __shared__ uint32_t sK[TK * 17];
  __shared__ __align__(16) __nv_bfloat16 sV[TK * 32];
  grid_dep_launch();
  grid_dep_wait();
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  long long row0 = static_cast<long long>(b) * nq;
  int q_begin = 0, q_end = nq;
  if (GROUPED) {
    row0 = static_cast<long long>(cand_off[b]) * nq;
    const int rows = (cand_off[b + 1] - cand_off[b]) * nq;
    q_begin = static_cast<int>(blockIdx.y) * rows_per_cta;
    if (q_begin >= rows) return;
    q_end = q_begin + rows_per_cta < rows ? q_begin + rows_per_cta : rows;
  }
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  cross_stage_kv<NR, 128, true>(sK, sV, kv, kv_rows, static_cast<long long>(b_first + b) * T, T, D, h, tid);
  __syncthreads();
  for (int qi = q_begin + warp; qi < q_end; qi += 4) {
    const long long row = row0 + qi;
    float sc[NR];
    const float sum = cross_row_exp<NR>(sK, q[row * D + h * 32 + lane], T, lane, sc);
    cross_row_pv<NR>(sV, sc, sum, lane, out + row * D + h * 32);
  }
}

template <int NR>   // keys per lane: T <= 32 * NR (NR = 4: T <= 128, NR = 8: T <= 256)
__global__ void __launch_bounds__(128) dec_cross_attn3_kernel(const float* __restrict__ q,
                                                              const __nv_bfloat16* __restrict__ kv, long long kv_rows,
                                                              int b_first, int T, int D, int heads, int nq,
                                                              __nv_bfloat16* __restrict__ out) {
  dec_cross_attn3_body<NR, false>(q, kv, kv_rows, b_first, T, D, heads, nq, nullptr, 0, out);
}

template <int NR>
__global__ void __launch_bounds__(128) dec_cross_attn3_grouped_kernel(const float* __restrict__ q,
                                                                      const __nv_bfloat16* __restrict__ kv, long long kv_rows,
                                                                      int b_first, int T, int D, int heads, int nq,
                                                                      const int* __restrict__ cand_off, int rows_per_cta,
                                                                      __nv_bfloat16* __restrict__ out) {
  dec_cross_attn3_body<NR, true>(q, kv, kv_rows, b_first, T, D, heads, nq, cand_off, rows_per_cta, out);
}

// ---------------------------------------------------------------------------------------------
// Cross-attention maps (parseq_forward_args.attn_maps): maps[row, t] = (1 / heads) * sum_h softmax_t(q_h . k_h,t) of
// the query rows of one decoder pass, the head-averaged weights nn.MultiheadAttention returns.  One CTA of 8 warps per
// (image, block of AMAP_ROWS query rows); the heads are visited in order, each head's K staged and each row's
// exponentials and their sum computed by the pieces dec_cross_attn3_kernel uses (cross_stage_kv, cross_row_exp): they are
// bitwise those of its P.V, which scales sum(e * v) by 1 / sum where this kernel stores p = e * (1 / sum) per key.
// Each warp keeps its AMAP_ROWS / 8 rows' running sums in registers; the heads are summed in fixed order, so the maps
// are bitwise reproducible and independent of the batch.  q fp32 [B*nq, D] pre-scaled; maps fp32 [B*nq, T].
// GROUPED (candidate scoring, parseq_score_args.attn_maps): the maps have out_ld rows per candidate, candidate c's
// query rows are q rows [c * nq, c * nq + nq) (nq <= out_ld), and image j owns the map rows [cand_off[j] * out_ld,
// cand_off[j + 1] * out_ld); CTA (j, y) writes AMAP_ROWS of them, grid.y covering the image with the most.  Row i of
// candidate c is computed for i <= lengths[c] and written as 0 past it (its sums stay 0), so rows past a label's EOS
// cost no exponentials.  A computed row's bits are those of the non-grouped kernel for the same q row.
constexpr int AMAP_ROWS = 32;
constexpr int AMAP_THREADS = 256;
template <int NR, bool GROUPED>
__device__ __forceinline__ void dec_cross_attn_maps_body(const float* __restrict__ q, const __nv_bfloat16* __restrict__ kv,
                                                         long long kv_rows, int b_first, int T, int D, int heads, int nq,
                                                         const int* __restrict__ cand_off, const int* __restrict__ lengths,
                                                         int out_ld, float* __restrict__ maps) {
  constexpr int TK = 32 * NR, WARPS = AMAP_THREADS / 32, RPW = AMAP_ROWS / WARPS;
  __shared__ uint32_t sK[TK * 17];
  grid_dep_launch();
  grid_dep_wait();
  const int b = blockIdx.x, q_begin = static_cast<int>(blockIdx.y) * AMAP_ROWS;
  int rows = nq, out0 = 0;
  if (GROUPED) {
    out0 = cand_off[b] * out_ld;
    rows = cand_off[b + 1] * out_ld - out0;
    if (q_begin >= rows) return;                       // CTA-uniform, before any barrier
  }
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const long long row_b = static_cast<long long>(b_first + b) * T;
  float acc[RPW][NR];
#pragma unroll
  for (int j = 0; j < RPW; ++j)
#pragma unroll
    for (int r = 0; r < NR; ++r) acc[j][r] = 0.f;
  for (int h = 0; h < heads; ++h) {
    if (h > 0) __syncthreads();                          // every warp is done with the previous head's K
    cross_stage_kv<NR, AMAP_THREADS, false>(sK, nullptr, kv, kv_rows, row_b, T, D, h, tid);
    __syncthreads();
#pragma unroll
    for (int j = 0; j < RPW; ++j) {
      const int qi = q_begin + warp + j * WARPS;
      if (qi >= (GROUPED ? rows : nq)) continue;         // warp-uniform
      long long row = static_cast<long long>(b) * nq + qi;
      if (GROUPED) {
        const int c = (out0 + qi) / out_ld, i = out0 + qi - c * out_ld;
        if (i > lengths[c]) continue;                    // warp-uniform: past the label's EOS
        row = static_cast<long long>(c) * nq + i;
      }
      float sc[NR];
      const float sum = cross_row_exp<NR>(sK, q[row * D + h * 32 + lane], T, lane, sc);
      const float inv = 1.0f / sum;
#pragma unroll
      for (int r = 0; r < NR; ++r) acc[j][r] += sc[r] * inv;
    }
  }
  const float rh = static_cast<float>(heads);
#pragma unroll
  for (int j = 0; j < RPW; ++j) {
    const int qi = q_begin + warp + j * WARPS;
    if (qi >= (GROUPED ? rows : nq)) continue;
    float* out = maps + ((GROUPED ? static_cast<long long>(out0) : static_cast<long long>(b) * nq) + qi) * T;
#pragma unroll
    for (int r = 0; r < NR; ++r)
      if (r * 32 + lane < T) out[r * 32 + lane] = acc[j][r] / rh;
  }
}

template <int NR>   // keys per lane: T <= 32 * NR
__global__ void __launch_bounds__(AMAP_THREADS, 1) dec_cross_attn_maps_kernel(const float* __restrict__ q,
                                                                         const __nv_bfloat16* __restrict__ kv,
                                                                         long long kv_rows, int b_first, int T, int D,
                                                                         int heads, int nq, float* __restrict__ maps) {
  dec_cross_attn_maps_body<NR, false>(q, kv, kv_rows, b_first, T, D, heads, nq, nullptr, nullptr, 0, maps);
}

template <int NR>
__global__ void __launch_bounds__(AMAP_THREADS, 1) dec_cross_attn_maps_grouped_kernel(
    const float* __restrict__ q, const __nv_bfloat16* __restrict__ kv, long long kv_rows, int b_first, int T, int D,
    int heads, int nq, const int* __restrict__ cand_off, const int* __restrict__ lengths, int out_ld,
    float* __restrict__ maps) {
  dec_cross_attn_maps_body<NR, true>(q, kv, kv_rows, b_first, T, D, heads, nq, cand_off, lengths, out_ld, maps);
}

// Rows past each hypothesis's length of the beam maps (parseq_beam_args.attn_maps) to 0: one CTA per hypothesis h of
// rows_per map rows, rows i > lengths[h] (every row of a missing hypothesis, length -1).
__global__ void maps_zero_tail_kernel(float* __restrict__ maps, const int* __restrict__ lengths, int rows_per, int T) {
  grid_dep_wait();
  const int h = blockIdx.x;
  const int first = lengths[h] + 1 > 0 ? lengths[h] + 1 : 0;
  float* m = maps + (static_cast<long long>(h) * rows_per + first) * T;
  const int n = (rows_per - first) * T;
  for (int i = threadIdx.x; i < n; i += blockDim.x) m[i] = 0.f;
}

// ---------------------------------------------------------------------------------------------
// Candidate scoring, last step: one CTA per candidate m, thread i = position i <= n_m (n_m = lengths[m]).  The term of
// position i is log_softmax(logits row)[t_i] = (t - M) - log(S), with M, S the merge of the row's per-tile partials
// (gemm_lse_epilogue) in column order: M = max of the tile maxima, S = sum of s_j exp(m_j - M).  The candidate's score is
// the sum of its terms in position order (thread 0).  Rows: the partial row of (m, i) is prow_m * P + i with prow_m =
// m - m0 (PARSeq: rows are (candidate, position)) or cand_img[m] - img0 (ViTSTR: rows are (image, position), shared by
// the image's candidates); the target logit is tlogit[(m - m0) * P + i], or, with xn != null (ViTSTR), the dot product
// of the bf16 row xn[prow] with the bf16 head row W[t] plus bias[t]: warp w takes positions w, w + 2, ..., its lanes
// read both rows as bf16 pairs (coalesced) and sum in fp32 with a fixed xor-shuffle order.  token_lp (may be null):
// [M][L] terms, 0 past n_m.
// No early griddepcontrol.launch_dependents: the next kernel on the stream (the next group of candidates, which
// rewrites the chain's LayerNorm, partial and target-logit buffers) may start only once this grid has exited, and this
// grid's wait orders it after the head GEMM that wrote what it reads.
// The merge of a row's per-tile (max, sum exp) partials (gemm_lse_epilogue, gemm_topk_epilogue) in column order:
// M = max of the tile maxima, S = sum of s_j exp(m_j - M); the row's log-sum-exp is M + log(S).
__device__ __forceinline__ void lse_merge(const float2* pr, int ntiles, float& M, float& S) {
  M = -INFINITY;
  for (int j = 0; j < ntiles; ++j) M = fmaxf(M, pr[j].x);
  S = 0.0f;
  for (int j = 0; j < ntiles; ++j) S += pr[j].y * expf(pr[j].x - M);
}
__global__ void __launch_bounds__(64) score_reduce_kernel(const float2* __restrict__ part, int ntiles,
                                                          const float* __restrict__ tlogit, const int* __restrict__ tgt,
                                                          const int* __restrict__ lengths, const int* __restrict__ cand_img,
                                                          int m0, int img0, int P, const __nv_bfloat16* __restrict__ xn,
                                                          const __nv_bfloat16* __restrict__ W, const float* __restrict__ bias,
                                                          int D, float* __restrict__ scores, float* __restrict__ token_lp,
                                                          int L) {
  __shared__ float s_term[64];
  __shared__ float s_tl[64];
  grid_dep_wait();
  const int m = m0 + static_cast<int>(blockIdx.x), i = threadIdx.x;
  const int n = lengths[m];
  const long long prow0 = static_cast<long long>(cand_img != nullptr ? cand_img[m] - img0 : m - m0) * P;
  const long long trow0 = static_cast<long long>(m - m0) * P;
  if (xn != nullptr) {
    const int warp = i >> 5, lane = i & 31;
    for (int k = warp; k <= n; k += 2) {
      const int c = tgt[trow0 + k];
      const __nv_bfloat162* x = reinterpret_cast<const __nv_bfloat162*>(xn + (prow0 + k) * D);
      const __nv_bfloat162* w = reinterpret_cast<const __nv_bfloat162*>(W + static_cast<long long>(c) * D);
      float t = 0.0f;
      for (int j = lane; j < D / 2; j += 32) {
        const float2 a = __bfloat1622float2(x[j]), b = __bfloat1622float2(w[j]);
        t = fmaf(a.y, b.y, fmaf(a.x, b.x, t));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if (lane == 0) s_tl[k] = t + bias[c];
    }
    __syncthreads();
  }
  float term = 0.0f;
  if (i <= n) {
    float M, S;
    lse_merge(part + (prow0 + i) * ntiles, ntiles, M, S);
    const float t = xn != nullptr ? s_tl[i] : tlogit[trow0 + i];
    term = (t - M) - logf(S);
  }
  if (token_lp != nullptr && i < L) token_lp[static_cast<long long>(m) * L + i] = term;
  s_term[i] = term;
  __syncthreads();
  if (i == 0) {
    float s = 0.0f;
    for (int k = 0; k <= n; ++k) s += s_term[k];
    scores[m] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// Beam search (parseq_beam_search).  A group's state has one row r = b * K + k per (image b, slot k): ids[r][ids_ld]
// (BOS, c_1.., then PAD; the EOS of a finished label stays in its row), score[r], len[r] (characters so far, -1 empty)
// and st[r] (BEAM_ACTIVE / BEAM_DONE / BEAM_EMPTY).  Every beam row of every step reads a valid token id, so the decoder
// runs on all rows without a branch; only the selection looks at the state.
constexpr int BEAM_MAX = 16;
constexpr int BEAM_ACTIVE = 0, BEAM_DONE = 1, BEAM_EMPTY = 2;
constexpr int BEAM_THREADS = 32 * BEAM_MAX;

// slot 0 of every image active with [BOS] and score 0, the other slots empty
__global__ void beam_init_kernel(int* __restrict__ ids, float* __restrict__ score, int* __restrict__ len, int* __restrict__ st,
                                 int rows, int K, int ids_ld, int bos, int pad) {
  grid_dep_launch();
  grid_dep_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < rows * ids_ld) ids[i] = ((i % ids_ld) == 0) ? bos : pad;
  if (i < rows) {
    const bool first = (i % K) == 0;
    score[i] = first ? 0.0f : -INFINITY;
    len[i] = first ? 0 : -1;
    st[i] = first ? BEAM_ACTIVE : BEAM_EMPTY;
  }
}

// One beam step of a group: one CTA per image, warp k < K expands slot k.  The row of (b, k) is row0 + b * img_stride +
// k * slot_stride (PARSeq: the step's b * K + k; ViTSTR: the image's position-`step` row for every slot).
//   1. Each active slot takes its row's log-sum-exp over the allowed classes and its K best classes in row order
//      (beam_order_key; masked and -inf classes never expand):
//      - at <= 128 classes (topk null) the lanes scan the logits row [C] for the max m and the sum s of exp(x - m) (m = -inf:
//        exp(x)), LSE = m + log(s), and keep their K best keys in registers;
//      - above 128 classes the head GEMM's top-K epilogue left per 128-column tile the (max, sum) partial `part` [ntiles]
//        and the tile's K best keys `topk` [ntiles][BEAM_TOPK_LD] of the allowed classes: lane 0 merges the partials in
//        column order (lse_merge, as score_reduce_kernel), the lanes keep the K best of the tiles' keys.
//      A NaN or +inf allowed logit makes the LSE NaN.  K rounds of a warp arg-max over the lanes' list heads
//      (xor-shuffle butterfly) give the slot's K expansions in row order.
//   2. Thread 0 builds the pool in slot order: a finished slot contributes itself, an active slot its expansions, each
//      with score parent + (logit - LSE) in fp32 (the logit is read back from its key).
//   3. Every entry counts the entries that rank before it (higher score, or equal and earlier; NaN after every number;
//      -inf never kept): the K first are the new slots.
//   4. The new state goes to the *_out buffers, parent[r] = the state row each new slot came from (the K/V cache rows
//      follow it at depth >= 2), and after the last step the results: out_ids [K][num_steps] per image (c_1..c_n, then
//      0 = EOS / padding), out_len (-1 empty), out_score (-inf empty).
// LEX (parseq_beam_search_lexicon): each slot also walks a lexicon DAG (BeamLex).  Its LSE is taken exactly as above
// from the whole logits row (the lexicon step always has the row: topk is null at every C), but only the node's
// expandable classes enter the lanes' lists: the lanes stride over the node's edges (class allowed, logit != -inf, and
// step + 1 < num_steps so that a character leaves room for its EOS), lane 0 adds EOS when the node is terminal.  Lanes
// k < K then find the child of the slot's k-th expansion by binary search over the node's sorted edge classes; the child
// travels with the pool entry into node_out (-1 for a finished or empty slot).  Step 0 takes slot 0's node from roots.
// No early griddepcontrol.launch_dependents: what comes next reads the state this grid writes.
struct BeamLex {
  const int* first_edge;            // [V + 1]
  const int* edge_class;            // [E], strictly increasing within a node
  const int* edge_child;            // [E]
  const unsigned char* terminal;    // [V]
  const int* roots;                 // [images of the group] or null (node 0)
  const int* node_in;               // [rows]
  int* node_out;                    // [rows]
};
template <bool LEX>
__global__ void __launch_bounds__(BEAM_THREADS) beam_select_kernel(
    const float* __restrict__ logits, const float2* __restrict__ part, const unsigned long long* __restrict__ topk,
    int ntiles, long long row0, long long img_stride, long long slot_stride, int C, int K, int step, int num_steps,
    const uint32_t* __restrict__ mask, int mask_ld, const int* __restrict__ ids_in, const float* __restrict__ score_in,
    const int* __restrict__ len_in, const int* __restrict__ st_in, int* __restrict__ ids_out, float* __restrict__ score_out,
    int* __restrict__ len_out, int* __restrict__ st_out, int* __restrict__ parent, int ids_ld, int* __restrict__ out_ids,
    int* __restrict__ out_len, float* __restrict__ out_score, BeamLex lex) {
  __shared__ unsigned long long s_key[BEAM_MAX][BEAM_MAX];
  __shared__ float s_lse[BEAM_MAX];
  __shared__ float p_score[BEAM_MAX * BEAM_MAX];
  __shared__ int p_slot[BEAM_MAX * BEAM_MAX], p_cls[BEAM_MAX * BEAM_MAX];
  __shared__ int s_sel[BEAM_MAX];
  __shared__ int s_n;
  __shared__ int s_child[LEX ? BEAM_MAX : 1][BEAM_MAX];
  __shared__ int p_child[LEX ? BEAM_MAX * BEAM_MAX : 1];
  grid_dep_wait();
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int r0 = b * K;
  const uint32_t* mrow = mask != nullptr ? mask + static_cast<long long>(b) * mask_ld : nullptr;
  if (tid < BEAM_MAX) s_sel[tid] = -1;
  if (warp < K && st_in[r0 + warp] == BEAM_ACTIVE) {
    const long long row = row0 + b * img_stride + warp * slot_stride;
    unsigned long long top[BEAM_MAX];
#pragma unroll
    for (int j = 0; j < BEAM_MAX; ++j) top[j] = 0ull;
    unsigned long long thr = 0ull;
    auto insert = [&](unsigned long long v) {
      if (v <= thr) return;
#pragma unroll
      for (int j = 0; j < BEAM_MAX; ++j) {        // insertion into the lane's descending list
        const unsigned long long t = top[j];
        const bool sw = v > t;
        top[j] = sw ? v : t;
        v = sw ? t : v;
      }
#pragma unroll
      for (int j = 0; j < BEAM_MAX; ++j)
        if (j == K - 1) thr = top[j];
    };
    float lse;
    if (LEX || topk == nullptr) {
      const float* lr = logits + row * C;
      float m = -INFINITY;
      for (int c = lane; c < C; c += 32) {
        if (mrow != nullptr && !class_allowed(mrow, c)) continue;
        const float x = lr[c];
        m = fmaxf(m, x);
        if (!LEX && x != -INFINITY) insert(beam_order_key(x, c));
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float base = (m == -INFINITY) ? 0.0f : m;
      float s = 0.0f;
      for (int c = lane; c < C; c += 32)
        if (mrow == nullptr || class_allowed(mrow, c)) s += expf(lr[c] - base);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      lse = m + logf(s);
    } else {
      const unsigned long long* kr = topk + row * ntiles * BEAM_TOPK_LD;
      for (int i = lane; i < ntiles * K; i += 32) {
        const int t = i / K, j = i - t * K;
        const unsigned long long v = kr[t * BEAM_TOPK_LD + j];
        if (v != 0ull) insert(v);
      }
      float M = 0.0f, S = 0.0f;
      if (lane == 0) lse_merge(part + row * ntiles, ntiles, M, S);
      lse = __shfl_sync(0xffffffffu, M + logf(S), 0);
    }
    int e0 = 0, e1 = 0;
    if constexpr (LEX) {
      const int v = step == 0 ? (lex.roots != nullptr ? lex.roots[b] : 0) : lex.node_in[r0 + warp];
      const float* lr = logits + row * C;
      e0 = lex.first_edge[v];
      e1 = lex.first_edge[v + 1];
      if (step + 1 < num_steps) {
        for (int ei = e0 + lane; ei < e1; ei += 32) {
          const int c = lex.edge_class[ei];
          if (mrow != nullptr && !class_allowed(mrow, c)) continue;
          const float x = lr[c];
          if (x != -INFINITY) insert(beam_order_key(x, c));
        }
      }
      if (lane == 0 && lex.terminal[v] != 0 && lr[0] != -INFINITY) insert(beam_order_key(lr[0], 0));
    }
    int h = 0;
    for (int r = 0; r < K; ++r) {
      unsigned long long cand = 0ull;
#pragma unroll
      for (int j = 0; j < BEAM_MAX; ++j)
        if (j == h && j < K) cand = top[j];
      unsigned long long best = cand;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, best, o);
        best = u > best ? u : best;
      }
      if (best != 0ull && cand == best) ++h;     // keys are unique within a row: one lane advances
      if (lane == 0) s_key[warp][r] = best;
    }
    if (lane == 0) s_lse[warp] = lse;
    if constexpr (LEX) {
      __syncwarp();
      if (lane < K) {
        const unsigned long long key = s_key[warp][lane];
        const int c = key != 0ull ? beam_key_class(key) : 0;
        int child = -1;
        if (c != 0) {
          int lo = e0, hi = e1 - 1;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (lex.edge_class[mid] < c) lo = mid + 1; else hi = mid;
          }
          child = lex.edge_child[lo];
        }
        s_child[warp][lane] = child;
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    int n = 0;
    for (int k = 0; k < K; ++k) {
      const int sk = st_in[r0 + k];
      const float ps = score_in[r0 + k];
      if (sk == BEAM_DONE) {
        p_score[n] = ps; p_slot[n] = k; p_cls[n] = -1;
        if constexpr (LEX) p_child[n] = -1;
        ++n;
      } else if (sk == BEAM_ACTIVE) {
        for (int j = 0; j < K && s_key[k][j] != 0ull; ++j) {
          const int c = beam_key_class(s_key[k][j]);
          p_score[n] = ps + (beam_key_value(s_key[k][j]) - s_lse[k]); p_slot[n] = k; p_cls[n] = c;
          if constexpr (LEX) p_child[n] = s_child[k][j];
          ++n;
        }
      }
    }
    s_n = n;
  }
  __syncthreads();
  const int n = s_n;
  if (tid < n) {
    const float v = p_score[tid];
    if (v != -INFINITY) {
      const bool vn = isnan(v);
      int rank = 0;
      for (int j = 0; j < n && rank < K; ++j) {
        const float u = p_score[j];
        if (j == tid || u == -INFINITY) continue;
        const bool un = isnan(u);
        rank += (un != vn) ? vn : ((!un && u > v) || ((un || u == v) && j < tid));
      }
      if (rank < K) s_sel[rank] = tid;
    }
  }
  __syncthreads();
  for (int idx = tid; idx < K * ids_ld; idx += blockDim.x) {
    const int k = idx / ids_ld, t = idx - k * ids_ld;
    const int e = s_sel[k];
    int v = ids_in[static_cast<long long>(r0 + k) * ids_ld + t];      // an empty slot keeps a row of valid ids
    if (e >= 0) {
      const int c = p_cls[e];
      v = (c >= 0 && t == step + 1) ? c : ids_in[static_cast<long long>(r0 + p_slot[e]) * ids_ld + t];
    }
    ids_out[static_cast<long long>(r0 + k) * ids_ld + t] = v;
  }
  const bool last = step + 1 == num_steps;
  if (tid < K) {
    const int k = tid, e = s_sel[k];
    float sc = -INFINITY;
    int ln = -1, sn = BEAM_EMPTY, par = k;
    if (e >= 0) {
      const int c = p_cls[e];
      par = p_slot[e];
      sc = p_score[e];
      if (c < 0) { ln = len_in[r0 + par]; sn = BEAM_DONE; }
      else if (c == 0) { ln = step; sn = BEAM_DONE; }
      else { ln = step + 1; sn = last ? BEAM_DONE : BEAM_ACTIVE; }
    }
    score_out[r0 + k] = sc;
    len_out[r0 + k] = ln;
    st_out[r0 + k] = sn;
    parent[r0 + k] = r0 + par;
    if constexpr (LEX) lex.node_out[r0 + k] = e >= 0 ? p_child[e] : -1;
    if (last) {
      out_len[r0 + k] = ln;
      out_score[r0 + k] = sc;
    }
  }
  if (last) {
    for (int idx = tid; idx < K * num_steps; idx += blockDim.x) {
      const int k = idx / num_steps, t = idx - k * num_steps;
      const int e = s_sel[k];
      int v = 0;
      if (e >= 0) {
        const int c = p_cls[e], p = p_slot[e];
        const int ln = c < 0 ? len_in[r0 + p] : (c == 0 ? step : step + 1);
        if (t < ln) v = t < step ? ids_in[static_cast<long long>(r0 + p) * ids_ld + t + 1] : c;
      }
      out_ids[static_cast<long long>(r0 + k) * num_steps + t] = v;
    }
  }
}

// Depth >= 2: the content K/V cache rows 0..n-1 of every new beam row come from its parent's row (cache [rows][pitch][2D]
// bf16, in 16-byte units: pitch4 per row, n4 valid)
__global__ void beam_kv_gather_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst, const int* __restrict__ parent,
                                      int rows, long long pitch4, int n4) {
  grid_dep_launch();
  grid_dep_wait();
  const long long total = static_cast<long long>(rows) * n4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int r = static_cast<int>(i / n4), j = static_cast<int>(i % n4);
    dst[r * pitch4 + j] = src[parent[r] * pitch4 + j];
  }
}

// ---------------------------------------------------------------------------------------------
// ViTSTR (vitstr/model.py:14-28 over timm VisionTransformer._pos_embed): token 0 of every image is
// cls_token + pos_embed[0]; tokens 1..Tp are the patch embeddings (pos_embed[1..Tp] already added by the patch GEMM).
__global__ void cls_assemble_kernel(const float4* __restrict__ patches, const float4* __restrict__ cls,
                                    const float4* __restrict__ pos0, float4* __restrict__ x, int B, int Tp, int D4) {
  grid_dep_launch();
  grid_dep_wait();                 // launched with the PDL attribute: the patch GEMM's output is complete from here on
  const long long total = static_cast<long long>(B) * (Tp + 1) * D4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % D4);
    const long long row = i / D4;
    const int t = static_cast<int>(row % (Tp + 1));
    const long long b = row / (Tp + 1);
    float4 v;
    if (t == 0) {
      const float4 a = cls[c], p = pos0[c];
      v = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
    } else {
      v = patches[(b * Tp + (t - 1)) * D4 + c];
    }
    x[i] = v;
  }
}
// out[b, j, :] = x[b, first + j, :], j < n (the `x[:, :seqlen]` / `logits[:, 1:]` slices of vitstr/model.py:21,
// vitstr/system.py:70 applied BEFORE norm + head: both are row-wise, so only the kept rows are computed).
__global__ void gather_token_rows_kernel(const float4* __restrict__ x, float4* __restrict__ out, int B, int T, int first,
                                         int n, int D4) {
  grid_dep_launch();
  grid_dep_wait();
  const long long total = static_cast<long long>(B) * n * D4;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int c = static_cast<int>(i % D4);
    const long long row = i / D4;
    const int j = static_cast<int>(row % n);
    const long long b = row / n;
    out[i] = x[(b * T + first + j) * D4 + c];
  }
}

// ---------------------------------------------------------------------------------------------
// Fused tail of a decoder pass: out = LayerNorm(y; decoder.norm) -> logits = head(out) -> greedy argmax
// (modules.py:124 `Decoder.norm`, model.py:138 `self.head`, model.py:142 argmax).  4 rows per CTA; the head weight
// (C x D bf16, 73 KB for 95 x 384) is staged in shared memory with an odd word pitch (lane = class reads are
// conflict-free); each warp computes a (32 classes x 4 rows) partial over a quarter of K; the normalised rows are
// rounded to bf16 exactly like a tensor-core A operand.
// logits fp32: row r -> logits[r * logits_ld .. + C); ids (optional): row r = (b, qi) -> ids[b*ids_ld + dst_off + qi].
// mask (optional): class allowlist rows of the images, row r = (b, qi) reads image b's (ptx.cuh class_allowed).
constexpr int HEAD_ROWS = 4;
template <int D>
__global__ void __launch_bounds__(384) dec_ln_head_argmax_kernel(
    const float* __restrict__ y, const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
    const __nv_bfloat16* __restrict__ Wh, const float* __restrict__ bh, int M, int C, float* __restrict__ logits,
    long long logits_ld, int* __restrict__ ids, int ids_ld, int nq, int dst_off, const int* __restrict__ forced,
    int forced_ld, const uint32_t* __restrict__ mask) {
  extern __shared__ __align__(16) unsigned char head_smem[];
  constexpr int WP = D / 2 + 1;                         // weight row pitch in 32-bit words (odd -> conflict-free)
  uint32_t* sW = reinterpret_cast<uint32_t*>(head_smem);            // [C][WP] bf16x2
  float* sy = reinterpret_cast<float*>(head_smem + ((static_cast<size_t>(C) * WP * 4 + 15) / 16) * 16);   // [4][D]
  float* spart = sy + HEAD_ROWS * D;                                // [4 k-quarters][4 rows][128]
  float* sl = spart + 4 * HEAD_ROWS * 128;                          // [4][128] logits
  grid_dep_launch();
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int nwarps = blockDim.x >> 5;
  // (weights do not depend on the previous kernel: stage them before the dependency wait)
  const uint32_t* Wg = reinterpret_cast<const uint32_t*>(Wh);
  for (int i = tid; i < C * (D / 2); i += blockDim.x) {
    const int c = i / (D / 2), k = i % (D / 2);
    sW[c * WP + k] = __ldg(Wg + i);
  }
  grid_dep_wait();
  const int row0 = blockIdx.x * HEAD_ROWS;
  // ---- LayerNorm of up to 4 rows (warp per row), rounded to bf16 ----
  constexpr int NV = D / 64;
  if (warp < HEAD_ROWS) {
    const int r = warp;
    const int row = row0 + r;
    float2 v[NV];
    if (row < M) {
      const float2* xr = reinterpret_cast<const float2*>(y + static_cast<long long>(row) * D);
#pragma unroll
      for (int i = 0; i < NV; ++i) v[i] = xr[i * 32 + lane];
    } else {
#pragma unroll
      for (int i = 0; i < NV; ++i) v[i] = make_float2(0.f, 0.f);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) s += v[i].x + v[i].y;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.0f / D);
    float qv = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float a = v[i].x - mean, b2 = v[i].y - mean;
      qv += a * a + b2 * b2;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) qv += __shfl_xor_sync(0xffffffffu, qv, o);
    const float rstd = 1.0f / sqrtf(qv * (1.0f / D) + eps);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const float2 g = __ldg(reinterpret_cast<const float2*>(gamma) + i * 32 + lane);
      const float2 bb = __ldg(reinterpret_cast<const float2*>(beta) + i * 32 + lane);
      const float o0 = (v[i].x - mean) * rstd * g.x + bb.x;
      const float o1 = (v[i].y - mean) * rstd * g.y + bb.y;
      reinterpret_cast<float2*>(sy + r * D)[i * 32 + lane] =
          make_float2(__bfloat162float(__float2bfloat16_rn(o0)), __bfloat162float(__float2bfloat16_rn(o1)));
    }
  }
  __syncthreads();
  // ---- head partials: unit = (class pass of 32, quarter of K); lane = class; 4 rows at once ----
  const int passes = (C + 31) / 32;
  constexpr int KQ = D / 8;                               // words per K quarter
  for (int u = warp; u < passes * 4; u += nwarps) {
    const int c = (u >> 2) * 32 + lane;
    const int kq = u & 3;
    const int cc = (c < C) ? c : (C - 1);
    const uint32_t* wr = sW + cc * WP + kq * KQ;
    const float* y0 = sy + kq * KQ * 2;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
#pragma unroll 4
    for (int k = 0; k < KQ; ++k) {
      const uint32_t w2 = wr[k];
      const float wx = __uint_as_float(w2 << 16), wy = __uint_as_float(w2 & 0xffff0000u);
      const float2 p0 = *reinterpret_cast<const float2*>(y0 + 2 * k);
      const float2 p1 = *reinterpret_cast<const float2*>(y0 + D + 2 * k);
      const float2 p2 = *reinterpret_cast<const float2*>(y0 + 2 * D + 2 * k);
      const float2 p3 = *reinterpret_cast<const float2*>(y0 + 3 * D + 2 * k);
      a0 = fmaf(wy, p0.y, fmaf(wx, p0.x, a0));
      a1 = fmaf(wy, p1.y, fmaf(wx, p1.x, a1));
      a2 = fmaf(wy, p2.y, fmaf(wx, p2.x, a2));
      a3 = fmaf(wy, p3.y, fmaf(wx, p3.x, a3));
    }
    float* sp = spart + (kq * HEAD_ROWS) * 128 + (c & 127);
    sp[0] = a0; sp[128] = a1; sp[256] = a2; sp[384] = a3;
  }
  __syncthreads();
  for (int i = tid; i < HEAD_ROWS * C; i += blockDim.x) {
    const int r = i / C, c = i % C;
    float l = ((spart[(0 * HEAD_ROWS + r) * 128 + c] + spart[(1 * HEAD_ROWS + r) * 128 + c]) +
               (spart[(2 * HEAD_ROWS + r) * 128 + c] + spart[(3 * HEAD_ROWS + r) * 128 + c])) + __ldg(bh + c);
    const int row = row0 + r;
    if (mask != nullptr && row < M &&
        !class_allowed(mask + static_cast<long long>(row / nq) * class_mask_words(C), c))
      l = -INFINITY;
    sl[r * 128 + c] = l;
    if (row < M) logits[static_cast<long long>(row) * logits_ld + c] = l;
  }
  if (ids == nullptr) return;
  __syncthreads();
  // ---- greedy argmax (torch.argmax order), warp per row ----
  if (warp < HEAD_ROWS) {
    const int r = warp;
    const int row = row0 + r;
    if (row < M) {
      float best = -INFINITY;
      int bi = ARGMAX_NONE;
      for (int j = lane; j < C; j += 32) argmax_scan(best, bi, sl[r * 128 + j], j);
      bi = argmax_finish(best, bi, sl + r * 128, C, lane);
      if (lane == 0) {
        const int b = row / nq, qi = row % nq;
        int v = bi;
        if (forced != nullptr) v = forced[static_cast<long long>(b) * forced_ld + dst_off + qi];
        ids[static_cast<long long>(b) * ids_ld + dst_off + qi] = v;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// row_max_prob_warp: the max softmax probability of one row (NaN where its maximum is not finite) and its id, the same
// bits in every lane of the warp (the butterfly sums are commutative).  The confidence is the product of these factors in
// row order through the first EOS; orient.cuh computes the rows of one image on several warps and multiplies the same
// factors in the same order.
__device__ __forceinline__ float row_max_prob_warp(const float* __restrict__ row, int C, int* id) {
  const int lane = threadIdx.x & 31;
  float best = -INFINITY;
  int bi = ARGMAX_NONE;
  for (int j = lane; j < C; j += 32) argmax_scan(best, bi, row[j], j);
  bi = argmax_finish(best, bi, row, C, lane);
  best = row[bi];
  // torch's softmax of a row whose maximum is not finite (it holds a NaN or a +inf, or is all -inf) is all NaN, and
  // max() over it gives index 0 with probability NaN
  const bool finite = isfinite(best);
  float se = 0.f;
  if (finite)
    for (int j = lane; j < C; j += 32) se += expf(row[j] - best);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
  *id = finite ? bi : 0;
  return finite ? 1.0f / se : __int_as_float(0x7fc00000);
}

// Fused post-processing of the reference's test path (strhub/models/base.py:132-142 + Tokenizer._filter,
// strhub/data/utils.py:120-129): per image  ids[i] = argmax_c logits[i, c]  (first maximum),  length = index of the
// first EOS (L if none),  confidence = prod_{i <= min(length, L-1)} max_c softmax(logits[i])_c  (the EOS probability is
// included).  A row whose maximum is NaN or +-inf has an all-NaN softmax in torch: id 0 (EOS) with probability NaN.
// One warp per image; only (length, confidence, ids) cross PCIe instead of the [B, L, C] probabilities.
__global__ void postprocess_kernel(const float* __restrict__ logits, int B, int L, int C, int eos_id, int* __restrict__ ids,
                                   int* __restrict__ lengths, float* __restrict__ confidence) {
  const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (b >= B) return;
  const int lane = threadIdx.x & 31;
  float conf = 1.0f;
  int len = L;
  bool done = false;
  for (int i = 0; i < L; ++i) {
    int id;
    const float p = row_max_prob_warp(logits + (static_cast<long long>(b) * L + i) * C, C, &id);
    if (lane == 0) ids[static_cast<long long>(b) * L + i] = id;
    if (!done) {
      conf *= p;                    // max softmax probability of position i
      if (id == eos_id) { len = i; done = true; }
    }
  }
  if (lane == 0) {
    lengths[b] = len;
    confidence[b] = conf;
  }
}

// ---------------------------------------------------------------------------------------------
// Boundary helpers of the module API (PARSeq.decode / head / text_embed called on their own).
__global__ void f32_to_bf16_kernel(const float4* __restrict__ x, uint2* __restrict__ y, long long n4) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 v = x[i];
    y[i] = make_uint2(pack_bf16(v.x, v.y), pack_bf16(v.z, v.w));
  }
}
// dst[b, :] = src[:] for b < B (n floats, n % 4 == 0)
__global__ void bcast_rows_kernel(const float4* __restrict__ src, float4* __restrict__ dst, int n4, int B) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < static_cast<long long>(B) * n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = src[i % n4];
}
// ids [B, J] (row pitch J) -> context buffer [B, ld]
__global__ void copy_ids_kernel(const int* __restrict__ src, int J, int* __restrict__ dst, int B, int ld) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B * ld) dst[i] = ((i % ld) < J) ? src[(i / ld) * J + (i % ld)] : 0;
}
// TokenEmbedding.forward (modules.py:175-176): out[i, :] = sqrt(D) * E[ids[i], :]
__global__ void text_embed_kernel(const int* __restrict__ ids, const float* __restrict__ E, float* __restrict__ out, int n,
                                  int D, int V, float scale) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < static_cast<long long>(n) * D;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    int tok = ids[i / D];
    tok = tok < 0 ? 0 : (tok >= V ? V - 1 : tok);
    out[i] = scale * E[static_cast<long long>(tok) * D + (i % D)];
  }
}

}  // namespace pq
