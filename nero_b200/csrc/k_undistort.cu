// Lens undistortion: the keypoint inversion of the SIMPLE_RADIAL model and the image warp to the undistorted pinhole
// camera.  The convention is stated in include/nero_undistort.h, the host side (camera rule, project rewrite) in
// nero_b200/undistort.py.
//
//   points   one thread per point: fp64 Newton inversion with a fixed step count, then the validity test.
//   image    one thread per output pixel: distort the pixel centre's ray into the input, bilinear over four RGB8 taps,
//            round half up.  12 bytes gathered and 3 written per pixel; neighbouring threads read neighbouring taps.
//
// No atomics and no reductions: every output is a fixed sequence of correctly rounded fp64 operations on its inputs, which
// oracle/nero_oracle_undistort.py repeats bit for bit.
#include <cmath>

#include "common.cuh"
#include "../../include/nero_undistort.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_UNDISTORT_BLOCK;

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void __launch_bounds__(kBlock) points_kernel(const double* __restrict__ xy, int n, double f, double cx, double cy,
                                                        double k, double* __restrict__ xn, int* __restrict__ valid) {
  const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (p >= n) return;
  const double xd = dd(ds(xy[2 * p], cx), f), yd = dd(ds(xy[2 * p + 1], cy), f);
  const double rd = __dsqrt_rn(da(dm(xd, xd), dm(yd, yd)));
  double r = rd;
#pragma unroll 1
  for (int it = 0; it < NERO_UNDISTORT_NEWTON; ++it) {
    const double t = dm(k, dm(r, r));
    const double e = ds(dm(r, da(1.0, t)), rd);
    r = ds(r, dd(e, da(1.0, dm(3.0, t))));
  }
  const double t = dm(k, dm(r, r));
  const double e = ds(dm(r, da(1.0, t)), rd);
  const bool ok = da(1.0, dm(3.0, t)) > 0.0 && fabs(e) <= NERO_UNDISTORT_TOL && r >= 0.0;
  double x = xd, y = yd;
  if (rd > 0.0) {
    const double s = dd(r, rd);
    x = dm(xd, s);
    y = dm(yd, s);
  }
  xn[2 * p] = x;
  xn[2 * p + 1] = y;
  valid[p] = ok ? 1 : 0;
}

// one bilinear axis: the two clamped taps and the weight of the second
__device__ __forceinline__ void axis(double t, int n, int& i0, int& i1, double& a) {
  const double f0 = floor(t);
  a = ds(t, f0);
  const int c = (int)fmin(fmax(f0, -1.0), (double)n);
  i0 = clampi(c, 0, n - 1);
  i1 = clampi(c + 1, 0, n - 1);
}

__global__ void __launch_bounds__(kBlock) image_kernel(const unsigned char* __restrict__ src, int w, int h, double f, double cx,
                                                       double cy, double k, unsigned char* __restrict__ dst, int w2, int h2,
                                                       double cx2, double cy2) {
  const long long p = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (p >= (long long)w2 * h2) return;
  const int i = (int)(p % w2), j = (int)(p / w2);
  const double x = dd(ds(da((double)i, 0.5), cx2), f), y = dd(ds(da((double)j, 0.5), cy2), f);
  const double d = da(1.0, dm(k, da(dm(x, x), dm(y, y))));
  const double u = da(dm(dm(f, x), d), cx), v = da(dm(dm(f, y), d), cy);
  int x0, x1, y0, y1;
  double a, b;
  axis(ds(u, 0.5), w, x0, x1, a);
  axis(ds(v, 0.5), h, y0, y1, b);
  const double a0 = ds(1.0, a), b0 = ds(1.0, b);
  const unsigned char* r0 = src + (long long)y0 * w * 3;
  const unsigned char* r1 = src + (long long)y1 * w * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const double p00 = __ldg(r0 + 3 * x0 + c), p01 = __ldg(r0 + 3 * x1 + c);
    const double p10 = __ldg(r1 + 3 * x0 + c), p11 = __ldg(r1 + 3 * x1 + c);
    const double top = da(dm(a0, p00), dm(a, p01)), bot = da(dm(a0, p10), dm(a, p11));
    const double val = floor(da(da(dm(b0, top), dm(b, bot)), 0.5));
    dst[3 * p + c] = (unsigned char)fmin(fmax(val, 0.0), 255.0);
  }
}

inline unsigned nblocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

inline bool finite(double v) { return std::isfinite(v); }

}  // namespace

extern "C" {

int nero_undistort_points(const double* xy, int n, double f, double cx, double cy, double k, double* xn, int* valid,
                          void* stream) {
  if (n < 0 || !(f > 0.0) || !finite(f) || !finite(cx) || !finite(cy) || !finite(k)) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!xy || !xn || !valid) return NERO_ERR_ARG;
  points_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(xy, n, f, cx, cy, k, xn, valid);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_undistort_image(const unsigned char* src, int w, int h, double f, double cx, double cy, double k,
                         unsigned char* dst, int w2, int h2, double cx2, double cy2, void* stream) {
  if (!src || !dst || w < 1 || h < 1 || w2 < 1 || h2 < 1 || (long long)w * h >= (1LL << 31) ||
      (long long)w2 * h2 >= (1LL << 31))
    return NERO_ERR_ARG;
  if (!(f > 0.0) || !finite(f) || !finite(cx) || !finite(cy) || !finite(k) || !finite(cx2) || !finite(cy2))
    return NERO_ERR_ARG;
  image_kernel<<<nblocks((long long)w2 * h2), kBlock, 0, (cudaStream_t)stream>>>(src, w, h, f, cx, cy, k, dst, w2, h2, cx2,
                                                                                 cy2);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
