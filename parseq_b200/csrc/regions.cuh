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
#pragma once
#include <cstdint>

namespace pq {

constexpr int REGION_THREADS = 256;
constexpr int REGION_MAX_SIDE = 8192;       // output sides, the raw-crop path's limit
constexpr int REGION_MAX_FRAME_SIDE = 32768;

// One region as the warp kernel reads it
struct RegionDesc {
  double a[8];                              // PIL PERSPECTIVE coefficients: output (x + .5, y + .5) -> frame
  long long src;                            // byte offset of the region's frame in `frames` (HWC RGB)
  long long dst;                            // byte offset of the region's crop in `out` (HWC RGB, packed)
  int fh, fw;                               // frame size
  int h, w;                                 // crop size
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
  // outside the frame: 0 (written so that a NaN, which the host checks rule out, also gives 0)
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
  const uint8_t* src = frames + __ldg(&d->src);
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

}  // namespace pq
