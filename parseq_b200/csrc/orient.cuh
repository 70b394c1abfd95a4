// Orientation search (parseq_forward_crops_oriented, include/parseq_b200.h): the confidence of each pass-1 reading and
// the select kernel that keeps, per crop, the most confident of its readings.  One CTA per reading for the confidences,
// one per crop for the selection and copy; no atomics.  A reading's
// confidence is postprocess_kernel's: the same per-row factors (row_max_prob_warp, kernels.cuh), here one warp per row,
// multiplied in row order through the first EOS by one thread.
#pragma once

#include <cstdint>

#include "kernels.cuh"

namespace pq {

constexpr int ORIENT_THREADS = 256;
struct OrientList { int o[4]; };   // the orientations of readings 1..R-1 of a crop: o[r] for its reading r + 1

// The confidence of one image's rows [L][C] (L <= 64), the same value in every thread of the CTA
__device__ __forceinline__ float seq_confidence_cta(const float* __restrict__ logits, int L, int C) {
  __shared__ float s_p[64];
  __shared__ int s_id[64];
  __shared__ float s_conf;
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x >> 5; i < L; i += blockDim.x >> 5) {
    int id;
    const float p = row_max_prob_warp(logits + static_cast<long long>(i) * C, C, &id);
    if (lane == 0) {
      s_p[i] = p;
      s_id[i] = id;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float conf = 1.0f;
    for (int i = 0; i < L; ++i) {
      conf *= s_p[i];
      if (s_id[i] == 0) break;     // EOS
    }
    s_conf = conf;
  }
  __syncthreads();
  const float c = s_conf;
  __syncthreads();                 // the shared rows are reused by the next reading
  return c;
}

// n floats src -> dst by the CTA, in the widest vector both pointers allow
template <typename V>
__device__ __forceinline__ void cta_copy_vec(float* __restrict__ dst, const float* __restrict__ src, long long n) {
  constexpr int W = sizeof(V) / sizeof(float);
  long long head = static_cast<long long>((sizeof(V) - (reinterpret_cast<uintptr_t>(dst) & (sizeof(V) - 1))) & (sizeof(V) - 1)) /
                   sizeof(float);
  head = head < n ? head : n;
  if (threadIdx.x < head) dst[threadIdx.x] = src[threadIdx.x];
  dst += head;
  src += head;
  n -= head;
  const long long nv = n / W;
  for (long long i = threadIdx.x; i < nv; i += blockDim.x) reinterpret_cast<V*>(dst)[i] = reinterpret_cast<const V*>(src)[i];
  for (long long i = nv * W + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}
__device__ __forceinline__ void cta_copy(float* dst, const float* src, long long n) {
  const uintptr_t d = reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src);
  if ((d & 15) == 0) cta_copy_vec<float4>(dst, src, n);
  else if ((d & 7) == 0) cta_copy_vec<float2>(dst, src, n);
  else cta_copy_vec<float>(dst, src, n);
}
__device__ __forceinline__ void cta_zero(float* dst, long long n) {
  long long head = static_cast<long long>((16 - (reinterpret_cast<uintptr_t>(dst) & 15)) & 15) / 4;
  head = head < n ? head : n;
  if (threadIdx.x < head) dst[threadIdx.x] = 0.f;
  dst += head;
  n -= head;
  const long long n4 = n / 4;
  for (long long i = threadIdx.x; i < n4; i += blockDim.x) reinterpret_cast<float4*>(dst)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) dst[i] = 0.f;
}

// Rows [S, L) of image b's outputs (logits [L][C], ids [L], maps [L][T]; ids / maps may be null) -> 0
__device__ __forceinline__ void zero_rows(float* logits, int* ids, float* maps, long long b, int S, int L, int C, int T) {
  if (S >= L) return;
  cta_zero(logits + (b * L + S) * C, 1ll * (L - S) * C);
  if (ids != nullptr) cta_zero(reinterpret_cast<float*>(ids) + b * L + S, L - S);
  if (maps != nullptr) cta_zero(maps + (b * L + S) * T, 1ll * (L - S) * T);
}

// After pass 1 (every crop read at o0, into the caller's outputs), CTA b: rotation[b] = o0, confidence[b] = the
// reading's confidence; steps_acc = the pass's step count *steps.  zero_tail: rows from *steps on are zeroed.
__global__ void __launch_bounds__(ORIENT_THREADS) orient_init_kernel(
    float* __restrict__ logits, int* __restrict__ ids, float* __restrict__ maps, int L, int C, int T, int o0,
    const int* __restrict__ steps, bool zero_tail, int* __restrict__ steps_acc, int* __restrict__ rotation,
    float* __restrict__ confidence) {
  const long long b = blockIdx.x;
  if (b == 0 && threadIdx.x == 0) *steps_acc = *steps;
  const float conf = seq_confidence_cta(logits + b * L * C, L, C);
  if (threadIdx.x == 0) {
    rotation[b] = o0;
    confidence[b] = conf;
  }
  if (zero_tail) zero_rows(logits, ids, maps, b, *steps, L, C, T);
}

// After one pass-2 super-chunk, CTA j: rd_conf[j] = the confidence of reading j of the static outputs.
__global__ void __launch_bounds__(ORIENT_THREADS) orient_conf_kernel(const float* __restrict__ rd_logits, int L, int C,
                                                                     float* __restrict__ rd_conf) {
  const long long j = blockIdx.x;
  const float c = seq_confidence_cta(rd_logits + j * L * C, L, C);
  if (threadIdx.x == 0) rd_conf[j] = c;
}

// Then CTA k: the static outputs hold readings k * R1 + r (r < R1) of listed crop k, crop rd_crop[k * R1], with their
// confidences in rd_conf.  In order, a reading wins when its confidence is greater than the best so far (initially the
// crop's pass-1 confidence), or is a number where the best is NaN.  The winner's logits, ids and maps go to the crop's
// rows of the caller's outputs (rows from *steps on zeroed when zero_tail), with its orientation and confidence.
// steps_acc = max(steps_acc, *steps).
__global__ void __launch_bounds__(ORIENT_THREADS) orient_select_kernel(
    const float* __restrict__ rd_logits, const int* __restrict__ rd_ids, const float* __restrict__ rd_maps,
    const float* __restrict__ rd_conf, const int* __restrict__ rd_crop, int R1, OrientList orient, int L, int C, int T,
    const int* __restrict__ steps, bool zero_tail, int* __restrict__ steps_acc, float* __restrict__ logits,
    int* __restrict__ ids, float* __restrict__ maps, int* __restrict__ rotation, float* __restrict__ confidence) {
  const long long k = blockIdx.x;
  if (k == 0 && threadIdx.x == 0) *steps_acc = max(*steps_acc, *steps);
  const long long b = rd_crop[k * R1];
  float best = confidence[b];
  int win = -1;
  for (int r = 0; r < R1; ++r) {
    const float c = rd_conf[k * R1 + r];
    if (c > best || (isnan(best) && !isnan(c))) {
      best = c;
      win = r;
    }
  }
  if (win < 0) return;
  const long long j = k * R1 + win;
  const int S = zero_tail ? *steps : L;
  cta_copy(logits + b * L * C, rd_logits + j * L * C, 1ll * S * C);
  if (ids != nullptr) cta_copy(reinterpret_cast<float*>(ids) + b * L, reinterpret_cast<const float*>(rd_ids) + j * L, S);
  if (maps != nullptr) cta_copy(maps + b * L * T, rd_maps + j * L * T, 1ll * S * T);
  zero_rows(logits, ids, maps, b, S, L, C, T);
  if (threadIdx.x == 0) {
    rotation[b] = orient.o[win];
    confidence[b] = best;
  }
}

// dst[i][:] = src[rows[i]][:] for i < n rows of ld words (the allowlist rows of pass-2 readings)
__global__ void gather_rows_kernel(const uint32_t* __restrict__ src, const int* __restrict__ rows, int n, int ld,
                                   uint32_t* __restrict__ dst) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < static_cast<long long>(n) * ld;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    dst[i] = src[static_cast<long long>(rows[i / ld]) * ld + i % ld];
}

}  // namespace pq
