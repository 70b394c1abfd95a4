// Raw crops of any size -> the engine's uint8 [N, H, W, 3] input: PIL's uint8 bicubic Image.resize (Resample.c,
// 8 bpc), with the rotation of Image.rotate(r, expand=True) as an index remap of the source read.  The reference runs
// this on every crop (strhub/data/module.py:69-82: rotate, T.Resize(img_size, BICUBIC)); the result is byte-identical.
//
// Exactness (DESIGN.md section 3.7): PIL resamples in two separable passes with uint8 between them; each output value of
// a pass is clip8((2^21 + sum in * k) >> 22) in int32, k the 22-bit fixed-point bicubic (a = -0.5) weights of
// precompute_coeffs / normalize_coeffs_8bpc.  Integer sums are exact in any order (wrapping adds are associative), so
// only the coefficients must be reproduced to the bit: they are computed here in double with explicit round-to-nearest
// intrinsics, because nvcc would otherwise contract a * b + c into a DFMA that PIL's host build does not use.
#pragma once
#include <cstdint>

namespace pq {

constexpr int CROP_BAND = 8;          // output lines of the second pass per CTA
constexpr int CROP_THREADS = 128;
constexpr int CROP_MAX_SIDE = 8192;

// One crop as the resize kernel reads it: pixel (y, x) of the ROTATED crop is at data + origin + y * sy + x * sx
// (byte strides +-3, +-3 w0).
struct CropDesc {
  long long origin;
  int sy, sx;
  int h, w;                           // rotated size
};

// Image.resize runs the vertical pass first for tall crops it shrinks vertically (Image.py: size[1] > size[0] * 100).
__host__ __device__ inline bool crop_vertical_first(int h, int w, int out_h) { return h > 100 * w && out_h < h; }

// Upper bound of the taps of one output coordinate: ksize of precompute_coeffs, (int)ceil(support) * 2 + 1.
__host__ __device__ inline int crop_ksize(int in, int out) {
  const double scale = static_cast<double>(in) / out;
  const double fs = scale < 1.0 ? 1.0 : scale;
  return static_cast<int>(ceil(2.0 * fs)) * 2 + 1;
}

// Dynamic shared memory of one CTA for a crop: first-pass table [out_f][ksize + 2], second-pass table [BAND][ksize + 2].
__host__ __device__ inline int crop_smem_ints(int h, int w, int out_h, int out_w) {
  const bool vf = crop_vertical_first(h, w, out_h);
  const int nf_in = vf ? h : w, nf_out = vf ? out_h : out_w, ns_in = vf ? w : h, ns_out = vf ? out_w : out_h;
  return nf_out * (crop_ksize(nf_in, nf_out) + 2) + CROP_BAND * (crop_ksize(ns_in, ns_out) + 2);
}

// Resample.c bicubic_filter, a = -0.5, in its evaluation order.
__device__ __forceinline__ double crop_cubic(double x) {
  if (x < 0.0) x = -x;
  if (x < 1.0) return __dadd_rn(__dmul_rn(__dmul_rn(__dsub_rn(__dmul_rn(1.5, x), 2.5), x), x), 1.0);
  if (x < 2.0) return __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(__dsub_rn(x, 5.0), x), 8.0), x), 4.0), -0.5);
  return 0.0;
}

// precompute_coeffs + normalize_coeffs_8bpc for output coordinate xx of an in -> out pass: writes the fixed-point taps
// to k[0, n) and returns xmin; *n = number of taps.
__device__ __noinline__ int crop_coeffs(int in, int out, int xx, int* k, int* n) {
  const double scale = __ddiv_rn(static_cast<double>(in), static_cast<double>(out));
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = __dmul_rn(2.0, fs);
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn(static_cast<double>(xx), 0.5), scale);
  int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, support), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, support), 0.5));
  if (xmax > in) xmax = in;
  xmax -= xmin;
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x)
    ww = __dadd_rn(ww, crop_cubic(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss)));
  for (int x = 0; x < xmax; ++x) {
    double w = crop_cubic(__dmul_rn(__dadd_rn(__dsub_rn(static_cast<double>(x + xmin), center), 0.5), ss));
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    k[x] = __double2int_rz(__dadd_rn(__dmul_rn(w, 4194304.0), w < 0.0 ? -0.5 : 0.5));
  }
  *n = xmax;
  return xmin;
}

__device__ __forceinline__ int crop_clip8(int v) {
  v >>= 22;
  return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// grid (bands, crops), CROP_THREADS threads.  The CTA of band b writes output lines [8b, 8b + 8) of the second pass (rows
// for the usual horizontal-then-vertical order, columns for tall crops).  Each thread owns (first-pass output
// coordinate, channel) items: it streams the input lines the band's windows cover, resamples each along the first axis
// once (rounded to uint8 as PIL does), and adds it into the int32 accumulators of the band lines whose window holds it.
// Nothing outside shared memory grows with the crop: the tables are bounded by the 8192-pixel side limit.
__global__ void __launch_bounds__(CROP_THREADS) crop_resize_bicubic_kernel(const uint8_t* __restrict__ data,
                                                                           const CropDesc* __restrict__ tab, int out_h,
                                                                           int out_w, uint8_t* __restrict__ out) {
  extern __shared__ int crop_smem[];
  const CropDesc d = tab[blockIdx.y];
  const bool vf = crop_vertical_first(d.h, d.w, out_h);
  const int nf_in = vf ? d.h : d.w, nf_out = vf ? out_h : out_w;
  const int ns_in = vf ? d.w : d.h, ns_out = vf ? out_w : out_h;
  const long long fstride = vf ? d.sy : d.sx, sstride = vf ? d.sx : d.sy;
  const int s0 = blockIdx.x * CROP_BAND;
  if (s0 >= ns_out) return;
  const int kf = crop_ksize(nf_in, nf_out), ks = crop_ksize(ns_in, ns_out);
  int* f_min = crop_smem;                            // [nf_out]
  int* f_n = f_min + nf_out;                         // [nf_out]
  int* f_k = f_n + nf_out;                           // [nf_out][kf]
  int* s_min = f_k + nf_out * kf;                    // [BAND]
  int* s_n = s_min + CROP_BAND;                      // [BAND]
  int* s_k = s_n + CROP_BAND;                        // [BAND][ks]
  for (int f = threadIdx.x; f < nf_out; f += blockDim.x) {
    f_min[f] = crop_coeffs(nf_in, nf_out, f, f_k + f * kf, f_n + f);
  }
  if (threadIdx.x < CROP_BAND) {
    const int r = threadIdx.x;
    int n = 0, m = 0;
    if (s0 + r < ns_out) m = crop_coeffs(ns_in, ns_out, s0 + r, s_k + r * ks, &n);
    s_min[r] = m;
    s_n[r] = n;
  }
  __syncthreads();
  // input lines of the band: from the first line's window start to the furthest window end
  const int jlo = s_min[0];
  int jhi = 0;
#pragma unroll
  for (int r = 0; r < CROP_BAND; ++r) jhi = max(jhi, s_min[r] + s_n[r]);
  const uint8_t* src = data + d.origin;
  uint8_t* dst = out + 3ll * out_h * out_w * blockIdx.y;
  for (int it = threadIdx.x; it < nf_out * 3; it += blockDim.x) {
    const int f = it / 3, c = it - 3 * f;
    const int fmin = f_min[f], nf = f_n[f];
    const int* k = f_k + f * kf;
    int acc[CROP_BAND];
#pragma unroll
    for (int r = 0; r < CROP_BAND; ++r) acc[r] = 1 << 21;
    for (int j = jlo; j < jhi; ++j) {
      const uint8_t* p = src + j * sstride + fmin * fstride + c;
      int sum = 1 << 21;
      for (int i = 0; i < nf; ++i) sum += static_cast<int>(__ldg(p + i * fstride)) * k[i];
      const int m = crop_clip8(sum);
#pragma unroll
      for (int r = 0; r < CROP_BAND; ++r) {
        const int q = j - s_min[r];
        if (q >= 0 && q < s_n[r]) acc[r] += m * s_k[r * ks + q];
      }
    }
#pragma unroll
    for (int r = 0; r < CROP_BAND; ++r) {
      const int s = s0 + r;
      if (s < ns_out) {
        const int pix = vf ? f * out_w + s : s * out_w + f;
        dst[3 * pix + c] = static_cast<uint8_t>(crop_clip8(acc[r]));
      }
    }
  }
}

}  // namespace pq
