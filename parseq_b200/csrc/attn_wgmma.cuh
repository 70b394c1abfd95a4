// ViT attention core on wgmma (sm_90a): out = softmax(Q K^T / sqrt(64)) V per (image, head, 128-query tile), from the
// packed qkv rows [B*T, 3D] (bf16) of the QKV GEMM.
//
// One CTA of two warpgroups; warpgroup w owns queries [64 w, 64 w + 64) of the tile.  Q, K (K-major: the 64 channels
// of a row are contiguous) and V^T (channels as rows, keys contiguous) are staged in shared memory in the 128B-swizzled
// layout wgmma reads; keys past T are zero rows and masked.  S = Q K^T (m64 x NK x k16, fp32 in registers), row max and
// exp in registers (a row lives in a quad of lanes), P = bf16(exp) back to shared memory as the A operand of
// O = P V (m64 x 64 x k16); O is divided by the fp32 row sum of exp.  NK (keys per tile) = 128 or 256.
#pragma once
#include "ptx.cuh"

namespace pq {

constexpr int ATW_THREADS = 256;

template <int NK>
constexpr int atw_smem_bytes() {
  return 1024 /*align*/ + 128 * 128 /*Q*/ + NK * 128 /*K*/ + NK * 128 /*V^T*/ + NK * 256 /*P*/;
}

// byte offset of element (row, k) in a K-major, 128B-swizzled operand made of 64-column chunks of `rows` rows each
__device__ __forceinline__ uint32_t sw128_off(int rows, int row, int k) {
  return static_cast<uint32_t>((k >> 6) * rows * 128 + row * 128) +
         ((static_cast<uint32_t>((k & 63) >> 3) ^ static_cast<uint32_t>(row & 7)) << 4) + static_cast<uint32_t>(k & 7) * 2;
}

template <int NK>
__global__ void __launch_bounds__(ATW_THREADS, 1)
enc_attention_wgmma_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int D, int heads) {
  static_assert(NK == 128 || NK == 256, "keys per tile");
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* qs = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* ks = qs + 128 * 128;
  uint8_t* vt = ks + NK * 128;
  uint8_t* ps = vt + NK * 128;

  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int q0 = blockIdx.y * 128;
  const long long ld = 3ll * D;
  const __nv_bfloat16* base = qkv + static_cast<long long>(b) * T * ld + h * 64;

  grid_dep_launch();
  grid_dep_wait();
  // ---- stage Q, K, V^T (16 B = 8 channels per load) ----
  for (int idx = threadIdx.x; idx < 128 * 8; idx += ATW_THREADS) {
    const int r = idx >> 3, u = idx & 7;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (q0 + r < T) v = *reinterpret_cast<const uint4*>(base + (q0 + r) * ld + u * 8);
    *reinterpret_cast<uint4*>(qs + sw128_off(128, r, u * 8)) = v;
  }
  for (int idx = threadIdx.x; idx < NK * 8; idx += ATW_THREADS) {
    const int r = idx >> 3, u = idx & 7;
    uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
    if (r < T) {
      kv = *reinterpret_cast<const uint4*>(base + r * ld + D + u * 8);
      vv = *reinterpret_cast<const uint4*>(base + r * ld + 2 * D + u * 8);
    }
    *reinterpret_cast<uint4*>(ks + sw128_off(NK, r, u * 8)) = kv;
    const __nv_bfloat16* ve = reinterpret_cast<const __nv_bfloat16*>(&vv);
#pragma unroll
    for (int e = 0; e < 8; ++e)     // V^T: channel u*8+e is a row, key r a column
      *reinterpret_cast<__nv_bfloat16*>(vt + sw128_off(64, u * 8 + e, r)) = ve[e];
  }
  fence_proxy_async_smem();
  __syncthreads();

  const int wg = threadIdx.x >> 7;
  const int t = threadIdx.x & 127;
  const int lane = t & 31;
  const int ra = (t >> 5) * 16 + (lane >> 2);          // rows ra, ra + 8 of this warpgroup's 64

  // ---- S = Q K^T ----
  float s[NK / 2];
#pragma unroll
  for (int i = 0; i < NK / 2; ++i) s[i] = 0.0f;
  {
    const uint64_t da = make_desc_k_sw128(smem_u32(qs + wg * 64 * 128));
    const uint64_t db = make_desc_k_sw128(smem_u32(ks));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k)
      wgmma_bf16<NK>(s, da + static_cast<uint64_t>(2 * k), db + static_cast<uint64_t>(2 * k), static_cast<uint32_t>(k != 0));
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_reg_fence(s);
  }
  // ---- softmax numerator in registers; P = bf16(exp) ----
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < NK / 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int key = i * 8 + 2 * (lane & 3) + (e & 1);
      if (key >= T) s[4 * i + e] = -INFINITY;
      mx[e >> 1] = fmaxf(mx[e >> 1], s[4 * i + e]);
    }
  float sum[2] = {0.f, 0.f};
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
    mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
  }
#pragma unroll
  for (int i = 0; i < NK / 8; ++i)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const float e0 = expf((s[4 * i + 2 * hr] - mx[hr]) * 0.125f);
      const float e1 = expf((s[4 * i + 2 * hr + 1] - mx[hr]) * 0.125f);
      sum[hr] += e0 + e1;
      const int row = wg * 64 + ra + 8 * hr;
      *reinterpret_cast<uint32_t*>(ps + sw128_off(128, row, i * 8 + 2 * (lane & 3))) = pack_bf16(e0, e1);
    }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 1);
    sum[hr] += __shfl_xor_sync(0xffffffffu, sum[hr], 2);
  }
  fence_proxy_async_smem();
  asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory");   // this warpgroup's P rows are in place

  // ---- O = P V ----
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.0f;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < NK / 16; ++kk) {
    const int c = kk >> 2;
    const uint64_t da = make_desc_k_sw128(smem_u32(ps + c * 128 * 128 + wg * 64 * 128)) + static_cast<uint64_t>(2 * (kk & 3));
    const uint64_t db = make_desc_k_sw128(smem_u32(vt + c * 64 * 128)) + static_cast<uint64_t>(2 * (kk & 3));
    wgmma_bf16<64>(o, da, db, static_cast<uint32_t>(kk != 0));
  }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_reg_fence(o);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int q = q0 + wg * 64 + ra + 8 * hr;
    if (q >= T) continue;
    const float inv = 1.0f / sum[hr];
    __nv_bfloat16* orow = out + (static_cast<long long>(b) * T + q) * D + h * 64;
#pragma unroll
    for (int i = 0; i < 8; ++i)
      *reinterpret_cast<uint32_t*>(orow + i * 8 + 2 * (lane & 3)) = pack_bf16(o[4 * i + 2 * hr] * inv, o[4 * i + 2 * hr + 1] * inv);
  }
}

}  // namespace pq
