// Text regions of full frames -> rectified crops: PIL's Image.transform(size, PERSPECTIVE, coeffs, BICUBIC) of an RGB
// frame (Geometry.c: ImagingGenericTransform with perspective_transform and bicubic_filter32RGB), byte for byte.
//
// Per output pixel (x, y): (xin, yin) = (x + 0.5, y + 0.5) goes through the map, numerator a0 xin + a1 yin + a2 in that
// order, divided by a6 xin + a7 yin + 1.  A source point outside [0, W) x [0, H) gives 0.  Otherwise 0.5 is subtracted,
// the floor taken, and the 4 x 4 BICUBIC macro of Geometry.c runs along the rows, then down the column of the four row
// values, with taps clamped to the frame; the value is clipped to [0, 255] and truncated.
//
// Exactness (DESIGN.md section 3.14): every fp64 operation is written with a round-to-nearest intrinsic in PIL's
// evaluation order, because nvcc would otherwise contract a * b + c into a DFMA that PIL's host build does not use.  The
// row pass takes uint8 taps, so its p2..p4 are integer sums as in C (exact in any order).  A pixel's bytes depend only on
// its region's frame, size and coefficients: no atomics, no shared memory, nothing that grows with the frame.
//
// Curved regions (polygons of 2k points, DESIGN.md section 3.15) take region_tps_kernel: the thin-plate spline of TRBA's
// GridGenerator maps the pixel onto the frame, and the same sampler tail (region_sample) gives its bytes.
#pragma once
#include <cstdint>

namespace pq {

constexpr int REGION_THREADS = 256;
constexpr int REGION_MAX_SIDE = 8192;       // output sides, the raw-crop path's limit
constexpr int REGION_MAX_FRAME_SIDE = 32768;
constexpr int TPS_MIN_K = 3, TPS_MAX_K = 32;  // points per polygon edge: 2k = F fiducials, 6..64
constexpr int TPS_MAX_COEFFS = 2 * TPS_MAX_K + 3;

// One region as the warp kernel reads it
struct RegionDesc {
  double a[8];                              // PIL PERSPECTIVE coefficients: output (x + .5, y + .5) -> frame
  long long src;                            // byte offset of the region's frame in `frames` (HWC RGB)
  long long dst;                            // byte offset of the region's crop in `out` (HWC RGB, packed)
  int fh, fw;                               // frame size
  int h, w;                                 // crop size
};

// One polygon region as the thin-plate-spline kernel reads it (DESIGN.md section 3.15)
struct TpsDesc {
  long long src;                            // byte offset of the region's frame in `frames` (HWC RGB)
  long long dst;                            // byte offset of the region's crop in `out` (HWC RGB, packed)
  int fh, fw;                               // frame size
  int h, w;                                 // crop size
  int k;                                    // points per edge: F = 2k fiducials
  double t[2 * TPS_MAX_COEFFS];             // T [F + 3][2]: frame (x, y) coefficients of 1, xn, yn, phi_0..phi_{F-1}
  double cx[TPS_MAX_K];                     // C_x = numpy.linspace(-1, 1, k); C_y is -1 (top) and +1 (bottom)
};

// Geometry.c BICUBIC of four uint8 taps: p2..p4 are int expressions in C, exact in double
__device__ __forceinline__ double region_cubic_u8(int v1, int v2, int v3, int v4, double d) {
  const double p1 = static_cast<double>(v2);
  const double p2 = static_cast<double>(-v1 + v3);
  const double p3 = static_cast<double>(2 * (v1 - v2) + v3 - v4);
  const double p4 = static_cast<double>(-v1 + v2 - v3 + v4);
  return __dadd_rn(p1, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

// Geometry.c BICUBIC of four double row values, in C's left-to-right order
__device__ __forceinline__ double region_cubic_f64(double v1, double v2, double v3, double v4, double d) {
  const double p1 = v2;
  const double p2 = __dadd_rn(-v1, v3);
  const double p3 = __dsub_rn(__dadd_rn(__dmul_rn(2.0, __dsub_rn(v1, v2)), v3), v4);
  const double p4 = __dadd_rn(__dsub_rn(__dadd_rn(-v1, v2), v3), v4);
  return __dadd_rn(p1, __dmul_rn(d, __dadd_rn(p2, __dmul_rn(d, __dadd_rn(p3, __dmul_rn(d, p4))))));
}

// The sampler tail both kernels share: frame point (sx, sy) of an RGB frame fh x fw -> the 3 bytes at dst.  Outside
// [0, W) x [0, H) gives 0 (written so that a NaN, which the host checks rule out, also gives 0); otherwise 0.5 is
// subtracted, the floor taken, and Geometry.c's 4 x 4 BICUBIC runs rows first with clamped taps, clipped and truncated.
__device__ __forceinline__ void region_sample(const uint8_t* __restrict__ frames, const long long* __restrict__ src_offset,
                                              int fh, int fw, double sx, double sy, uint8_t* __restrict__ dst) {
  if (!(sx >= 0.0 && sx < static_cast<double>(fw) && sy >= 0.0 && sy < static_cast<double>(fh))) {
    dst[0] = dst[1] = dst[2] = 0;
    return;
  }
  const double xs = __dsub_rn(sx, 0.5), ys = __dsub_rn(sy, 0.5);
  const int ix = __double2int_rd(xs), iy = __double2int_rd(ys);   // FLOOR: xs, ys >= -0.5
  const double dx = __dsub_rn(xs, static_cast<double>(ix));       // exact
  const double dy = __dsub_rn(ys, static_cast<double>(iy));
  long long col[4], row[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int cx = min(max(ix - 1 + k, 0), fw - 1), cy = min(max(iy - 1 + k, 0), fh - 1);
    col[k] = 3ll * cx;
    row[k] = 3ll * fw * cy;
  }
  const uint8_t* src = frames + __ldg(src_offset);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    double v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const uint8_t* r = src + row[k] + c;
      v[k] = region_cubic_u8(__ldg(r + col[0]), __ldg(r + col[1]), __ldg(r + col[2]), __ldg(r + col[3]), dx);
    }
    const double o = region_cubic_f64(v[0], v[1], v[2], v[3], dy);
    dst[c] = o <= 0.0 ? 0 : (o >= 255.0 ? 255 : static_cast<uint8_t>(__double2int_rz(o)));
  }
}

// grid (pixel tiles, regions), REGION_THREADS threads: one thread per output pixel, all three channels.  Tiles past a
// region's h * w pixels return at once (the grid covers the largest region of the launch).
__global__ void __launch_bounds__(REGION_THREADS) region_warp_kernel(const uint8_t* __restrict__ frames,
                                                                     const RegionDesc* __restrict__ tab,
                                                                     uint8_t* __restrict__ out) {
  const RegionDesc* d = tab + blockIdx.y;
  const int h = __ldg(&d->h), w = __ldg(&d->w);
  const long long p = static_cast<long long>(blockIdx.x) * REGION_THREADS + threadIdx.x;
  if (p >= static_cast<long long>(h) * w) return;
  const int y = static_cast<int>(p / w), x = static_cast<int>(p - static_cast<long long>(y) * w);
  const double a0 = __ldg(&d->a[0]), a1 = __ldg(&d->a[1]), a2 = __ldg(&d->a[2]), a3 = __ldg(&d->a[3]);
  const double a4 = __ldg(&d->a[4]), a5 = __ldg(&d->a[5]), a6 = __ldg(&d->a[6]), a7 = __ldg(&d->a[7]);
  const int fh = __ldg(&d->fh), fw = __ldg(&d->fw);
  uint8_t* dst = out + __ldg(&d->dst) + 3 * p;

  const double xin = __dadd_rn(static_cast<double>(x), 0.5), yin = __dadd_rn(static_cast<double>(y), 0.5);
  const double den = __dadd_rn(__dadd_rn(__dmul_rn(a6, xin), __dmul_rn(a7, yin)), 1.0);
  const double sx = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a0, xin), __dmul_rn(a1, yin)), a2), den);
  const double sy = __ddiv_rn(__dadd_rn(__dadd_rn(__dmul_rn(a3, xin), __dmul_rn(a4, yin)), a5), den);
  region_sample(frames, &d->src, fh, fw, sx, sy, dst);
}

// grid (pixel tiles, regions), REGION_THREADS threads: the thin-plate spline of TRBA's GridGenerator with the
// region's coefficients, then region_sample.  Per output pixel (x, y): xn = (2x + 1 - w) / w, yn = (2y + 1 - h) / h;
// for fiducial m, r_m = sqrt((xn - C_x[m])^2 + (yn - C_y[m])^2) and phi_m = (r_m r_m) ln(r_m + 1e-6); then
// X = T0 + T1 xn + T2 yn + sum_m T_{3+m} phi_m in that order, each product and sum rounded on its own (no DFMA), likewise
// Y.  Only ln is not correctly rounded.  The CTA stages its region's T and C_x in shared memory.
__global__ void __launch_bounds__(REGION_THREADS) region_tps_kernel(const uint8_t* __restrict__ frames,
                                                                    const TpsDesc* __restrict__ tab,
                                                                    uint8_t* __restrict__ out) {
  __shared__ double s_t[2 * TPS_MAX_COEFFS];
  __shared__ double s_cx[TPS_MAX_K];
  const TpsDesc* d = tab + blockIdx.y;
  const int h = __ldg(&d->h), w = __ldg(&d->w), k = __ldg(&d->k);
  const long long p0 = static_cast<long long>(blockIdx.x) * REGION_THREADS;
  if (p0 >= static_cast<long long>(h) * w) return;                  // the whole CTA, before the barrier
  for (int i = threadIdx.x; i < 2 * (2 * k + 3); i += REGION_THREADS) s_t[i] = __ldg(&d->t[i]);
  for (int i = threadIdx.x; i < k; i += REGION_THREADS) s_cx[i] = __ldg(&d->cx[i]);
  __syncthreads();
  const long long p = p0 + threadIdx.x;
  if (p >= static_cast<long long>(h) * w) return;
  const int y = static_cast<int>(p / w), x = static_cast<int>(p - static_cast<long long>(y) * w);
  const int fh = __ldg(&d->fh), fw = __ldg(&d->fw);
  uint8_t* dst = out + __ldg(&d->dst) + 3 * p;

  // _build_P: (arange(-w, w, 2) + 1.0) / w, the numerator an exact integer
  const double xn = __ddiv_rn(static_cast<double>(2 * x + 1 - w), static_cast<double>(w));
  const double yn = __ddiv_rn(static_cast<double>(2 * y + 1 - h), static_cast<double>(h));
  double sx = __dadd_rn(__dadd_rn(s_t[0], __dmul_rn(s_t[2], xn)), __dmul_rn(s_t[4], yn));
  double sy = __dadd_rn(__dadd_rn(s_t[1], __dmul_rn(s_t[3], xn)), __dmul_rn(s_t[5], yn));
  const double dyt = __dsub_rn(yn, -1.0), dyb = __dsub_rn(yn, 1.0);
  const double dyt2 = __dmul_rn(dyt, dyt), dyb2 = __dmul_rn(dyb, dyb);
  const double* tm = s_t + 6;
#pragma unroll 1
  for (int e = 0; e < 2; ++e) {                                     // top fiducials m = j, then bottom m = k + j
    const double dy2 = e == 0 ? dyt2 : dyb2;
    for (int j = 0; j < k; ++j, tm += 2) {
      const double dx = __dsub_rn(xn, s_cx[j]);
      const double r = __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), dy2));
      const double phi = __dmul_rn(__dmul_rn(r, r), log(__dadd_rn(r, 1e-6)));
      sx = __dadd_rn(sx, __dmul_rn(tm[0], phi));
      sy = __dadd_rn(sy, __dmul_rn(tm[1], phi));
    }
  }
  region_sample(frames, &d->src, fh, fw, sx, sy, dst);
}

}  // namespace pq
