// Incremental structure from motion: the GPU replacement of the correspondence graph, absolute pose, triangulation and
// bundle-adjustment stages of COLMAP's mapper.  The protocol is stated in nero_b200/sfm.py, the ABI in include/nero_sfm.h.
//
//   tracks       union-find over the inlier edges (union_find.cuh), roots compacted in node order (compact.cuh)
//   p3p          one thread per hypothesis: 3 hashed draws, Lambda Twist, integer inlier counts of each pose; one block
//                picks the winner (largest count, then lower hypothesis) and marks its inliers
//   triangulate  one thread per track: 4 x 4 normal matrix in observation order, cyclic Jacobi, depth / error / angle
//   filter       one thread per point: reprojection errors of its observations and its largest ray angle
//   ba_*         one Levenberg-Marquardt iteration: per-point linearisation and Schur elimination, the reduced camera
//                system by segments of a sorted (o, o') list cut into chunks (one block per chunk sums in entry order, one
//                block per segment adds the chunks in a fixed shape), back-substitution, and the cost as per-block
//                partials added in block order
// All arithmetic is fp64; nothing is placed or summed by an atomic, so every result is the same on every run.
#include <cmath>

#include <math_constants.h>

#include "common.cuh"
#include "compact.cuh"
#include "hash.cuh"
#include "union_find.cuh"
#include "../../include/nero_sfm.h"
#include "../../include/nero_sfm_radial.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_SFM_BLOCK;
constexpr int kMaxDraws = 32;
constexpr int kTriSweeps = 10, kEigSweeps = 12;

inline unsigned blocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

// ------------------------------------------------------------------------------------------------ small algebra
__device__ __forceinline__ void load_pose(const double* __restrict__ pose, int i, double R[9], double t[3]) {
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = pose[12 * i + k];
#pragma unroll
  for (int k = 0; k < 3; ++k) t[k] = pose[12 * i + 9 + k];
}

__device__ __forceinline__ void mat3_vec(const double R[9], const double x[3], double y[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r) y[r] = R[3 * r] * x[0] + R[3 * r + 1] * x[1] + R[3 * r + 2] * x[2];
}

__device__ __forceinline__ double det3(const double m[9]) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// inverse of a 3 x 3 matrix by its adjugate; false when det == 0
__device__ __forceinline__ bool inv3(const double m[9], double out[9]) {
  const double d = det3(m);
  if (d == 0.0) return false;
  const double id = 1.0 / d;
  out[0] = (m[4] * m[8] - m[5] * m[7]) * id;
  out[1] = (m[2] * m[7] - m[1] * m[8]) * id;
  out[2] = (m[1] * m[5] - m[2] * m[4]) * id;
  out[3] = (m[5] * m[6] - m[3] * m[8]) * id;
  out[4] = (m[0] * m[8] - m[2] * m[6]) * id;
  out[5] = (m[2] * m[3] - m[0] * m[5]) * id;
  out[6] = (m[3] * m[7] - m[4] * m[6]) * id;
  out[7] = (m[1] * m[6] - m[0] * m[7]) * id;
  out[8] = (m[0] * m[4] - m[1] * m[3]) * id;
  return true;
}

// cyclic Jacobi on the symmetric N x N matrix A (row-major); V receives the eigenvectors as columns.  Fully unrolled, so
// every index is a constant and both matrices stay in registers.
template <int N, int kSweeps>
__device__ __forceinline__ void jacobi(double A[N * N], double V[N * N]) {
#pragma unroll
  for (int k = 0; k < N * N; ++k) V[k] = (k / N == k % N) ? 1.0 : 0.0;
#pragma unroll 1
  for (int sw = 0; sw < kSweeps; ++sw) {
#pragma unroll
    for (int p = 0; p < N - 1; ++p) {
#pragma unroll
      for (int q = p + 1; q < N; ++q) {
        const double apq = A[p * N + q];
        if (apq != 0.0) {
          const double theta = (A[q * N + q] - A[p * N + p]) / (2.0 * apq);
          const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
          for (int k = 0; k < N; ++k) {
            const double akp = A[k * N + p], akq = A[k * N + q];
            A[k * N + p] = c * akp - s * akq;
            A[k * N + q] = s * akp + c * akq;
          }
#pragma unroll
          for (int k = 0; k < N; ++k) {
            const double apk = A[p * N + k], aqk = A[q * N + k];
            A[p * N + k] = c * apk - s * aqk;
            A[q * N + k] = s * apk + c * aqk;
          }
#pragma unroll
          for (int k = 0; k < N; ++k) {
            const double vkp = V[k * N + p], vkq = V[k * N + q];
            V[k * N + p] = c * vkp - s * vkq;
            V[k * N + q] = s * vkp + c * vkq;
          }
        }
      }
    }
  }
}

// R <- exp([w]x) R (Rodrigues)
__device__ __forceinline__ void rotate_left(const double w[3], const double R[9], double out[9]) {
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double a, b;
  if (th < 1e-12) {
    a = 1.0;
    b = 0.0;
  } else {
    double sn, cs;
    sincospi(th / CUDART_PI, &sn, &cs);   // the pi-scaled form has no large-argument reduction, so no local memory
    a = sn / th;
    b = (1.0 - cs) / (th * th);
  }
  const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  double E[9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double kk = K[3 * r] * K[c] + K[3 * r + 1] * K[3 + c] + K[3 * r + 2] * K[6 + c];
      E[3 * r + c] = (r == c ? 1.0 : 0.0) + a * K[3 * r + c] + b * kk;
    }
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) out[3 * r + c] = E[3 * r] * R[c] + E[3 * r + 1] * R[3 + c] + E[3 * r + 2] * R[6 + c];
}

// camera-frame point, its projection residual and the unit ray from the camera centre.  kCam is the number of free
// parameters of a camera: 1 (SIMPLE_PINHOLE: f) or 2 (SIMPLE_RADIAL: f, k; include/nero_sfm_radial.h).
struct Cam {
  double R[9], t[3], f, cx, cy, k;
};

template <int kCam = 1>
__device__ __forceinline__ Cam load_cam(const double* pose, const int* img_cam, const double* focal, const double* pp, int i,
                                        const double* radial = nullptr) {
  Cam c;
  load_pose(pose, i, c.R, c.t);
  const int k = img_cam[i];
  c.f = focal[k];
  c.cx = pp[2 * k];
  c.cy = pp[2 * k + 1];
  c.k = kCam == 2 ? radial[k] : 0.0;
  return c;
}

// SIMPLE_RADIAL: normalised point (x, y) = (Y_x, Y_y) / Y_z, r2 = x^2 + y^2, d = 1 + k r2, pixel ((f x) d + cx, (f y) d + cy)
__device__ __forceinline__ void radial_pixel(const Cam& c, double x, double y, double* r2, double* d, double* pu, double* pv) {
  *r2 = x * x + y * y;
  *d = 1.0 + c.k * *r2;
  *pu = (c.f * x) * *d + c.cx;
  *pv = (c.f * y) * *d + c.cy;
}

// (depth, squared reprojection error) of X seen at (x, y), in the (distorted) image
template <int kCam = 1>
__device__ __forceinline__ double reproj2(const Cam& c, const double X[3], double x, double y, double* depth) {
  double Y[3];
  mat3_vec(c.R, X, Y);
  Y[0] += c.t[0];
  Y[1] += c.t[1];
  Y[2] += c.t[2];
  *depth = Y[2];
  double ex, ey;
  if constexpr (kCam == 1) {
    ex = c.f * Y[0] / Y[2] + c.cx - x;
    ey = c.f * Y[1] / Y[2] + c.cy - y;
  } else {
    const double iz = 1.0 / Y[2];
    double r2, d, pu, pv;
    radial_pixel(c, Y[0] * iz, Y[1] * iz, &r2, &d, &pu, &pv);
    ex = pu - x;
    ey = pv - y;
  }
  return ex * ex + ey * ey;
}

// unit vector from the centre -R^T t of camera c to X
__device__ __forceinline__ void ray(const Cam& c, const double X[3], double r[3]) {
  double C[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) C[k] = -(c.R[k] * c.t[0] + c.R[3 + k] * c.t[1] + c.R[6 + k] * c.t[2]);
  double n = 0.0;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    r[k] = X[k] - C[k];
    n += r[k] * r[k];
  }
  n = 1.0 / sqrt(n);
#pragma unroll
  for (int k = 0; k < 3; ++k) r[k] *= n;
}

// the largest pairwise angle of the rays of observations o0 .. o1 - 1 to X
__device__ double largest_angle(long long o0, long long o1, const int* obs_img, const double* pose, const int* img_cam, const double* focal,
                                const double* pp, const double X[3]) {
  double cmin = 1.0;
  for (long long a = o0; a < o1; ++a) {
    const Cam ca = load_cam(pose, img_cam, focal, pp, obs_img[a]);
    double ra[3];
    ray(ca, X, ra);
    for (long long b = a + 1; b < o1; ++b) {
      const Cam cb = load_cam(pose, img_cam, focal, pp, obs_img[b]);
      double rb[3];
      ray(cb, X, rb);
      cmin = fmin(cmin, ra[0] * rb[0] + ra[1] * rb[1] + ra[2] * rb[2]);
    }
  }
  return acos(fmax(-1.0, fmin(1.0, cmin)));
}

// ------------------------------------------------------------------------------------------------ tracks
__global__ void __launch_bounds__(kBlock) hook_kernel(const int* __restrict__ edges, int E, int* parent) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e < E) uf_unite(parent, edges[2 * e], edges[2 * e + 1]);
}

__global__ void __launch_bounds__(kBlock) root_count_kernel(const int* __restrict__ label, int N, int* __restrict__ blk_cnt) {
  __shared__ int s_w[kBlock / 32];
  const int v = blockIdx.x * kBlock + threadIdx.x;
  int total;
  block_scan<kBlock>(v < N && label[v] == v ? 1 : 0, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) root_emit_kernel(const int* __restrict__ label, int N, const long long* __restrict__ blk_off,
                                                           int* __restrict__ track) {
  __shared__ int s_w[kBlock / 32];
  const int v = blockIdx.x * kBlock + threadIdx.x;
  const bool root = v < N && label[v] == v;
  int total;
  const int r = block_scan<kBlock>(root ? 1 : 0, s_w, &total);
  if (root) track[v] = int(blk_off[blockIdx.x] + r);
}

// non-roots read their root's rank, which the previous launch wrote
__global__ void __launch_bounds__(kBlock) track_map_kernel(const int* __restrict__ label, int N, int* __restrict__ track) {
  const int v = blockIdx.x * kBlock + threadIdx.x;
  if (v < N && label[v] != v) track[v] = track[label[v]];
}

// ------------------------------------------------------------------------------------------------ P3P (Lambda Twist)
__device__ __forceinline__ uint32_t draw_key(unsigned seed, int image, int hyp, int draw) {
  uint32_t h = rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u);
  h = rl_mix(h ^ (uint32_t)image);
  h = rl_mix(h ^ (uint32_t)hyp);
  return rl_mix(h ^ (uint32_t)draw);
}

__device__ __forceinline__ double det_cols(const double A[9], const double B[9], const double C[9]) {
  // det of the matrix whose columns are column 0 of A, column 1 of B, column 2 of C
  const double m[9] = {A[0], B[1], C[2], A[3], B[4], C[5], A[6], B[7], C[8]};
  return det3(m);
}

// the largest real root of c3 g^3 + c2 g^2 + c1 g + c0 (c3 != 0), polished by two Newton steps
__device__ __forceinline__ double largest_cubic_root(double c3, double c2, double c1, double c0) {
  const double a = c2 / c3, b = c1 / c3, c = c0 / c3;
  const double p = b - a * a / 3.0, q = 2.0 * a * a * a / 27.0 - a * b / 3.0 + c;
  const double disc = q * q / 4.0 + p * p * p / 27.0;
  double g;
  if (disc > 0.0) {
    const double s = sqrt(disc);
    g = cbrt(-q / 2.0 + s) + cbrt(-q / 2.0 - s) - a / 3.0;
  } else {
    const double m = 2.0 * sqrt(fmax(-p / 3.0, 0.0));
    const double arg = m > 0.0 ? fmax(-1.0, fmin(1.0, 3.0 * q / (p * m))) : 0.0;
    g = m * cospi(acos(arg) / (3.0 * CUDART_PI)) - a / 3.0;
  }
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const double fv = ((g + a) * g + b) * g + c, df = (3.0 * g + 2.0 * a) * g + b;
    if (df != 0.0) g -= fv / df;
  }
  return g;
}

// one of three values for a run-time i in 0..2, by selects on the values (not on their addresses), so arrays stay in registers
__device__ __forceinline__ double pick3(double v0, double v1, double v2, int i) { return i == 0 ? v0 : i == 1 ? v1 : v2; }

__device__ __forceinline__ int quad_roots(double a, double b, double c, double r[2]) {
  const double disc = b * b - 4.0 * a * c;
  if (disc < 0.0) return 0;
  if (a == 0.0) {
    if (b == 0.0) return 0;
    r[0] = -c / b;
    return 1;
  }
  const double sq = sqrt(disc);
  const double q = -0.5 * (b + (b >= 0.0 ? sq : -sq));
  r[0] = q / a;
  r[1] = q != 0.0 ? c / q : r[0];
  return 2;
}

// poses of bearings y[3][3] toward world points x[3][3]: emit(R, t) for each (at most 4), in solution order; returns their
// number.  Each pose is handed over as it is found, so no pose array is indexed at run time.
template <class Emit>
__device__ __forceinline__ int p3p(const double y[9], const double x[9], Emit&& emit) {
  const double b12 = -2.0 * (y[0] * y[3] + y[1] * y[4] + y[2] * y[5]);
  const double b13 = -2.0 * (y[0] * y[6] + y[1] * y[7] + y[2] * y[8]);
  const double b23 = -2.0 * (y[3] * y[6] + y[4] * y[7] + y[5] * y[8]);
  double d12[3], d13[3], d23[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    d12[k] = x[k] - x[3 + k];
    d13[k] = x[k] - x[6 + k];
    d23[k] = x[3 + k] - x[6 + k];
  }
  const double a12 = d12[0] * d12[0] + d12[1] * d12[1] + d12[2] * d12[2];
  const double a13 = d13[0] * d13[0] + d13[1] * d13[1] + d13[2] * d13[2];
  const double a23 = d23[0] * d23[0] + d23[1] * d23[1] + d23[2] * d23[2];
  const double M12[9] = {1.0, b12 / 2, 0.0, b12 / 2, 1.0, 0.0, 0.0, 0.0, 0.0};
  const double M13[9] = {1.0, 0.0, b13 / 2, 0.0, 0.0, 0.0, b13 / 2, 0.0, 1.0};
  const double M23[9] = {0.0, 0.0, 0.0, 0.0, 1.0, b23 / 2, 0.0, b23 / 2, 1.0};
  double D1[9], D2[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    D1[k] = M12[k] * a23 - M23[k] * a12;
    D2[k] = M13[k] * a23 - M23[k] * a13;
  }
  const double c3 = det3(D2), c0 = det3(D1);
  const double c2 = det_cols(D1, D2, D2) + det_cols(D2, D1, D2) + det_cols(D2, D2, D1);
  const double c1 = det_cols(D2, D1, D1) + det_cols(D1, D2, D1) + det_cols(D1, D1, D2);
  if (c3 == 0.0) return 0;
  const double g = largest_cubic_root(c3, c2, c1, c0);
  double A[9], V[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) A[k] = D1[k] + g * D2[k];
  jacobi<3, kEigSweeps>(A, V);
  // eigenvalues by |value| descending (ties: lower index); the two largest span the degenerate conic's plane pair
  int o0 = 0, o1 = 1, o2 = 2;
  const double e[3] = {A[0], A[4], A[8]};
  if (fabs(e[o1]) > fabs(e[o0])) { const int s = o0; o0 = o1; o1 = s; }
  if (fabs(e[o2]) > fabs(e[o1])) { const int s = o1; o1 = o2; o2 = s; }
  if (fabs(e[o1]) > fabs(e[o0])) { const int s = o0; o0 = o1; o1 = s; }
  const double s1 = pick3(e[0], e[1], e[2], o0), s2 = pick3(e[0], e[1], e[2], o1);
  if (s1 * s2 > 0.0 || s1 == 0.0) return 0;
  double u1[3], u2[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double row[3] = {V[3 * k], V[3 * k + 1], V[3 * k + 2]};
    u1[k] = pick3(row[0], row[1], row[2], o0);
    u2[k] = pick3(row[0], row[1], row[2], o1);
  }
  const double s = sqrt(-s2 / s1);
  int n = 0;
#pragma unroll 1
  for (int sg = 0; sg < 2; ++sg) {
    const double sgn = sg == 0 ? 1.0 : -1.0;
    double nrm[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) nrm[k] = u1[k] - sgn * s * u2[k];
    int k = 0;
    if (fabs(nrm[1]) > fabs(nrm[k])) k = 1;
    if (fabs(nrm[2]) > fabs(nrm[k])) k = 2;
    const int i = k == 0 ? 1 : 0, j = k == 2 ? 1 : 2;
    const double wi = -pick3(nrm[0], nrm[1], nrm[2], i) / pick3(nrm[0], nrm[1], nrm[2], k), wj = -pick3(nrm[0], nrm[1], nrm[2], j) / pick3(nrm[0], nrm[1], nrm[2], k);
    double e0[3], e1[3];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      e0[m] = m == i ? 1.0 : m == k ? wi : 0.0;
      e1[m] = m == j ? 1.0 : m == k ? wj : 0.0;
    }
    double De0[3], De1[3];
    mat3_vec(D2, e0, De0);
    mat3_vec(D2, e1, De1);
    const double q00 = e0[0] * De0[0] + e0[1] * De0[1] + e0[2] * De0[2];
    const double q01 = e0[0] * De1[0] + e0[1] * De1[1] + e0[2] * De1[2];
    const double q11 = e1[0] * De1[0] + e1[1] * De1[1] + e1[2] * De1[2];
    double taus[2];
    const int nt = quad_roots(q00, 2.0 * q01, q11, taus);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      if (r >= nt) continue;
      double d[3], Md[3];
#pragma unroll
      for (int m = 0; m < 3; ++m) d[m] = e0[m] * taus[r] + e1[m];
      mat3_vec(M23, d, Md);
      const double qq = d[0] * Md[0] + d[1] * Md[1] + d[2] * Md[2];
      if (qq <= 0.0) continue;
      const double sc = sqrt(a23 / qq);
      double l[3] = {d[0] * sc, d[1] * sc, d[2] * sc};
      if (pick3(l[0], l[1], l[2], j) < 0.0) {
        l[0] = -l[0];
        l[1] = -l[1];
        l[2] = -l[2];
      }
      if (!(l[0] > 0.0 && l[1] > 0.0 && l[2] > 0.0)) continue;
      // two Gauss-Newton steps on the three distance equations
      for (int it = 0; it < 2; ++it) {
        const double r3[3] = {l[0] * l[0] + l[1] * l[1] + b12 * l[0] * l[1] - a12, l[0] * l[0] + l[2] * l[2] + b13 * l[0] * l[2] - a13,
                              l[1] * l[1] + l[2] * l[2] + b23 * l[1] * l[2] - a23};
        const double J[9] = {2 * l[0] + b12 * l[1], 2 * l[1] + b12 * l[0], 0.0, 2 * l[0] + b13 * l[2], 0.0, 2 * l[2] + b13 * l[0],
                             0.0, 2 * l[1] + b23 * l[2], 2 * l[2] + b23 * l[1]};
        double Ji[9];
        if (!inv3(J, Ji)) break;
        double dl[3];
        mat3_vec(Ji, r3, dl);
        l[0] -= dl[0];
        l[1] -= dl[1];
        l[2] -= dl[2];
      }
      // R from the difference vectors and their cross product, t = Y1 - R x1
      double Y[9];
#pragma unroll
      for (int m = 0; m < 3; ++m)
#pragma unroll
        for (int c = 0; c < 3; ++c) Y[3 * m + c] = l[m] * y[3 * m + c];
      const double a[3] = {Y[0] - Y[3], Y[1] - Y[4], Y[2] - Y[5]}, bb[3] = {Y[0] - Y[6], Y[1] - Y[7], Y[2] - Y[8]};
      const double ab[3] = {a[1] * bb[2] - a[2] * bb[1], a[2] * bb[0] - a[0] * bb[2], a[0] * bb[1] - a[1] * bb[0]};
      const double cd[3] = {d12[1] * d13[2] - d12[2] * d13[1], d12[2] * d13[0] - d12[0] * d13[2], d12[0] * d13[1] - d12[1] * d13[0]};
      const double My[9] = {a[0], bb[0], ab[0], a[1], bb[1], ab[1], a[2], bb[2], ab[2]};
      const double Mx[9] = {d12[0], d13[0], cd[0], d12[1], d13[1], cd[1], d12[2], d13[2], cd[2]};
      double Mxi[9];
      if (!inv3(Mx, Mxi)) continue;
      double R[9], tt[3];
#pragma unroll
      for (int rr = 0; rr < 3; ++rr)
#pragma unroll
        for (int c = 0; c < 3; ++c) R[3 * rr + c] = My[3 * rr] * Mxi[c] + My[3 * rr + 1] * Mxi[3 + c] + My[3 * rr + 2] * Mxi[6 + c];
      double Rx[3];
      mat3_vec(R, x, Rx);
      tt[0] = Y[0] - Rx[0];
      tt[1] = Y[1] - Rx[1];
      tt[2] = Y[2] - Rx[2];
      emit(R, tt);
      ++n;
    }
  }
  return n;
}

__device__ __forceinline__ bool pose_inlier(const double R[9], const double t[3], const double* xy, const double* X, int m, double f, double cx,
                                            double cy, double max_err2) {
  const double P[3] = {X[3 * m], X[3 * m + 1], X[3 * m + 2]};
  double Y[3];
  mat3_vec(R, P, Y);
  Y[0] += t[0];
  Y[1] += t[1];
  Y[2] += t[2];
  const double ex = f * Y[0] / Y[2] + cx - xy[2 * m], ey = f * Y[1] / Y[2] + cy - xy[2 * m + 1];
  return Y[2] > 0.0 && ex * ex + ey * ey <= max_err2;
}

__global__ void __launch_bounds__(kBlock) p3p_kernel(const double* __restrict__ xy, const double* __restrict__ X, int n, double f, double cx,
                                                     double cy, int image, int H, unsigned seed, double max_err2, int* __restrict__ counts,
                                                     double* __restrict__ poses) {
  const int h = blockIdx.x * kBlock + threadIdx.x;
  if (h >= H) return;
  int i0 = -1, i1 = -1, i2 = -1, k = 0;
  for (int d = 0; d < kMaxDraws && k < 3; ++d) {
    const int m = (int)(draw_key(seed, image, h, d) % (uint32_t)n);
    if (m == i0 || m == i1) continue;
    if (k == 0) i0 = m; else if (k == 1) i1 = m; else i2 = m;
    ++k;
  }
  int best = -1;
  double bR[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, bt[3] = {0, 0, 0};
  if (k == 3) {
    double y[9], x[9];
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const int m = j == 0 ? i0 : j == 1 ? i1 : i2;
      const double u = (xy[2 * m] - cx) / f, v = (xy[2 * m + 1] - cy) / f;
      const double nn = 1.0 / sqrt(u * u + v * v + 1.0);
      y[3 * j] = u * nn;
      y[3 * j + 1] = v * nn;
      y[3 * j + 2] = nn;
      x[3 * j] = X[3 * m];
      x[3 * j + 1] = X[3 * m + 1];
      x[3 * j + 2] = X[3 * m + 2];
    }
    p3p(y, x, [&](const double R[9], const double t[3]) {
      int c = 0;
      for (int m = 0; m < n; ++m) c += pose_inlier(R, t, xy, X, m, f, cx, cy, max_err2);
      if (c > best) {
        best = c;
#pragma unroll
        for (int e = 0; e < 9; ++e) bR[e] = R[e];
#pragma unroll
        for (int e = 0; e < 3; ++e) bt[e] = t[e];
      }
    });
  }
  counts[h] = best;
#pragma unroll
  for (int e = 0; e < 9; ++e) poses[12 * h + e] = bR[e];
#pragma unroll
  for (int e = 0; e < 3; ++e) poses[12 * h + 9 + e] = bt[e];
}

// one block: the winner (largest count, ties to the lower hypothesis), then its inliers
__global__ void __launch_bounds__(kBlock) p3p_select_kernel(const double* __restrict__ xy, const double* __restrict__ X, int n, double f,
                                                            double cx, double cy, int H, double max_err2, const int* __restrict__ counts,
                                                            const double* __restrict__ poses, int* __restrict__ best,
                                                            double* __restrict__ pose, unsigned char* __restrict__ inlier) {
  __shared__ int s_c[kBlock], s_h[kBlock];
  __shared__ double s_pose[12];
  int bc = -2, bh = H;
  for (int h = threadIdx.x; h < H; h += kBlock)
    if (counts[h] > bc) {
      bc = counts[h];
      bh = h;
    }
  s_c[threadIdx.x] = bc;
  s_h[threadIdx.x] = bh;
  __syncthreads();
  for (int w = kBlock / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) {
      const int oc = s_c[threadIdx.x + w], oh = s_h[threadIdx.x + w];
      if (oc > s_c[threadIdx.x] || (oc == s_c[threadIdx.x] && oh < s_h[threadIdx.x])) {
        s_c[threadIdx.x] = oc;
        s_h[threadIdx.x] = oh;
      }
    }
    __syncthreads();
  }
  const int w = s_h[0], c = s_c[0];
  if (threadIdx.x < 12) {
    s_pose[threadIdx.x] = poses[12 * w + threadIdx.x];
    pose[threadIdx.x] = s_pose[threadIdx.x];
  }
  if (threadIdx.x == 0) {
    best[0] = w;
    best[1] = max(c, 0);
  }
  __syncthreads();
  double R[9], t[3];
#pragma unroll
  for (int e = 0; e < 9; ++e) R[e] = s_pose[e];
#pragma unroll
  for (int e = 0; e < 3; ++e) t[e] = s_pose[9 + e];
  for (int m = threadIdx.x; m < n; m += kBlock) inlier[m] = c >= 0 && pose_inlier(R, t, xy, X, m, f, cx, cy, max_err2);
}

// ------------------------------------------------------------------------------------------------ triangulation, filter
__global__ void __launch_bounds__(kBlock) triangulate_kernel(const long long* __restrict__ off, int T, const int* __restrict__ obs_img,
                                                             const double* __restrict__ obs_xy, const double* __restrict__ pose,
                                                             const int* __restrict__ img_cam, const double* __restrict__ focal,
                                                             const double* __restrict__ pp, double* __restrict__ Xout,
                                                             double* __restrict__ stat) {
  const int k = blockIdx.x * kBlock + threadIdx.x;
  if (k >= T) return;
  const long long o0 = off[k], o1 = off[k + 1];
  double A[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) A[e] = 0.0;
  for (long long o = o0; o < o1; ++o) {
    const Cam c = load_cam(pose, img_cam, focal, pp, obs_img[o]);
    const double u = (obs_xy[2 * o] - c.cx) / c.f, v = (obs_xy[2 * o + 1] - c.cy) / c.f;
    const double P2[4] = {c.R[6], c.R[7], c.R[8], c.t[2]};
    double r0[4], r1[4];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      r0[m] = u * P2[m] - c.R[m];
      r1[m] = v * P2[m] - c.R[3 + m];
    }
    r0[3] = u * P2[3] - c.t[0];
    r1[3] = v * P2[3] - c.t[1];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) A[4 * r + q] += r0[r] * r0[q];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) A[4 * r + q] += r1[r] * r1[q];
  }
  double V[16];
  jacobi<4, kTriSweeps>(A, V);
  int m = 0;
  double amin = A[0];
#pragma unroll
  for (int e = 1; e < 4; ++e)
    if (A[5 * e] < amin) {
      amin = A[5 * e];
      m = e;
    }
  double ev[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) ev[e] = m == 0 ? V[4 * e] : m == 1 ? V[4 * e + 1] : m == 2 ? V[4 * e + 2] : V[4 * e + 3];
  const double X[3] = {ev[0] / ev[3], ev[1] / ev[3], ev[2] / ev[3]};
  double dmin = INFINITY, emax = 0.0;
  for (long long o = o0; o < o1; ++o) {
    const Cam c = load_cam(pose, img_cam, focal, pp, obs_img[o]);
    double z;
    const double e2 = reproj2(c, X, obs_xy[2 * o], obs_xy[2 * o + 1], &z);
    dmin = fmin(dmin, z);
    emax = fmax(emax, sqrt(e2));
  }
#pragma unroll
  for (int e = 0; e < 3; ++e) Xout[3 * k + e] = X[e];
  stat[3 * k] = dmin;
  stat[3 * k + 1] = emax;
  stat[3 * k + 2] = largest_angle(o0, o1, obs_img, pose, img_cam, focal, pp, X);
}

template <int kCam>
__global__ void __launch_bounds__(kBlock) filter_kernel(const long long* __restrict__ pt_off, int P, const int* __restrict__ obs_img,
                                                        const double* __restrict__ obs_xy, const double* __restrict__ pose,
                                                        const int* __restrict__ img_cam, const double* __restrict__ focal,
                                                        const double* __restrict__ pp, const double* __restrict__ Xin,
                                                        double* __restrict__ err, double* __restrict__ angle,
                                                        const double* __restrict__ radial) {
  const int p = blockIdx.x * kBlock + threadIdx.x;
  if (p >= P) return;
  const double X[3] = {Xin[3 * p], Xin[3 * p + 1], Xin[3 * p + 2]};
  const long long o0 = pt_off[p], o1 = pt_off[p + 1];
  for (long long o = o0; o < o1; ++o) {
    const Cam c = load_cam<kCam>(pose, img_cam, focal, pp, obs_img[o], radial);
    double z;
    const double e2 = reproj2<kCam>(c, X, obs_xy[2 * o], obs_xy[2 * o + 1], &z);
    err[2 * o] = z;
    err[2 * o + 1] = sqrt(e2);
  }
  angle[p] = largest_angle(o0, o1, obs_img, pose, img_cam, focal, pp, X);
}

// ------------------------------------------------------------------------------------------------ bundle adjustment
// Per observation the camera-side columns are (w, t) and the kCam camera parameters: kNc = 6 + kCam of them.  Jc is
// [n, 2, kNc], Y [n, kNc, 3].
template <int kCam>
constexpr int kNc = 6 + kCam;

// Residual res [2] of Y = R X + t seen at xy [2], its derivative dY [2][3] with respect to Y, and the camera-parameter
// columns jf [2][kCam].  Pinhole: dr/dY = (f / Y_z) [[1, 0, -u], [0, 1, -v]], dr/df = (u, v).  Radial, with (x, y) the
// normalised point: dr/d(x, y) = f [[d + 2k x^2, 2k x y], [2k x y, d + 2k y^2]], d(x, y)/dY = (1 / Y_z) [[1, 0, -x],
// [0, 1, -y]], dr/df = (x d, y d), dr/dk = (f x r2, f y r2).
template <int kCam>
__device__ __forceinline__ void project_jacobian(const Cam& c, const double Y[3], const double* __restrict__ xy, double* __restrict__ res,
                                                 double dY[2][3], double jf[2][kCam]) {
  const double iz = 1.0 / Y[2], u = Y[0] * iz, v = Y[1] * iz;
  if constexpr (kCam == 1) {
    const double fz = c.f * iz;
    res[0] = c.f * u + c.cx - xy[0];
    res[1] = c.f * v + c.cy - xy[1];
    dY[0][0] = fz;
    dY[0][1] = 0.0;
    dY[0][2] = -fz * u;
    dY[1][0] = 0.0;
    dY[1][1] = fz;
    dY[1][2] = -fz * v;
    jf[0][0] = u;
    jf[1][0] = v;
  } else {
    double r2, d, pu, pv;
    radial_pixel(c, u, v, &r2, &d, &pu, &pv);
    res[0] = pu - xy[0];
    res[1] = pv - xy[1];
    const double a = c.f * (d + 2.0 * c.k * u * u), b = c.f * (2.0 * c.k * u * v), e = c.f * (d + 2.0 * c.k * v * v);
    dY[0][0] = a * iz;
    dY[0][1] = b * iz;
    dY[0][2] = -(a * u + b * v) * iz;
    dY[1][0] = b * iz;
    dY[1][1] = e * iz;
    dY[1][2] = -(b * u + e * v) * iz;
    jf[0][0] = u * d;
    jf[1][0] = v * d;
    jf[0][1] = c.f * u * r2;
    jf[1][1] = c.f * v * r2;
  }
}

template <int kCam>
__global__ void __launch_bounds__(kBlock) linearize_kernel(const long long* __restrict__ pt_off, int P, const int* __restrict__ obs_img,
                                                           const double* __restrict__ obs_xy, const double* __restrict__ pose,
                                                           const int* __restrict__ img_cam, const double* __restrict__ focal,
                                                           const double* __restrict__ pp, const double* __restrict__ Xin,
                                                           double* __restrict__ res, double* __restrict__ Jc, double* __restrict__ Jp,
                                                           const double* __restrict__ radial) {
  constexpr int NC = kNc<kCam>;
  const int p = blockIdx.x * kBlock + threadIdx.x;
  if (p >= P) return;
  const double X[3] = {Xin[3 * p], Xin[3 * p + 1], Xin[3 * p + 2]};
  for (long long o = pt_off[p]; o < pt_off[p + 1]; ++o) {
    const Cam c = load_cam<kCam>(pose, img_cam, focal, pp, obs_img[o], radial);
    double RX[3];
    mat3_vec(c.R, X, RX);
    const double Y[3] = {RX[0] + c.t[0], RX[1] + c.t[1], RX[2] + c.t[2]};
    double dY[2][3], jf[2][kCam];
    project_jacobian<kCam>(c, Y, obs_xy + 2 * o, res + 2 * o, dY, jf);
    // dY/dw = -[RX]x; dY/dt = I; dY/dX = R
    const double H[9] = {0.0, RX[2], -RX[1], -RX[2], 0.0, RX[0], RX[1], -RX[0], 0.0};   // -[RX]x
    double* jc = Jc + 2 * NC * o;
    double* jp = Jp + 6 * o;
#pragma unroll
    for (int r = 0; r < 2; ++r) {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        jc[NC * r + q] = dY[r][0] * H[q] + dY[r][1] * H[3 + q] + dY[r][2] * H[6 + q];
        jc[NC * r + 3 + q] = dY[r][q];
        jp[3 * r + q] = dY[r][0] * c.R[q] + dY[r][1] * c.R[3 + q] + dY[r][2] * c.R[6 + q];
      }
#pragma unroll
      for (int q = 0; q < kCam; ++q) jc[NC * r + 6 + q] = jf[r][q];
    }
  }
}

// W_o [a][k] = (Jc_o^T Jp_o) [a][k]
template <int NC>
__device__ __forceinline__ double w_entry(const double* jc, const double* jp, int a, int k) {
  return jc[a] * jp[k] + jc[NC + a] * jp[3 + k];
}

template <int kCam>
__global__ void __launch_bounds__(kBlock) points_kernel(const long long* __restrict__ pt_off, int P, const double* __restrict__ res,
                                                        const double* __restrict__ Jc, const double* __restrict__ Jp, double lambda,
                                                        int fix_points, double* __restrict__ Vinv, double* __restrict__ gp,
                                                        double* __restrict__ Y) {
  constexpr int NC = kNc<kCam>;
  const int p = blockIdx.x * kBlock + threadIdx.x;
  if (p >= P) return;
  const long long o0 = pt_off[p], o1 = pt_off[p + 1];
  double V[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
  for (long long o = o0; o < o1; ++o) {
    const double* jp = Jp + 6 * o;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) V[3 * r + c] += jp[r] * jp[c] + jp[3 + r] * jp[3 + c];
      g[r] += jp[r] * res[2 * o] + jp[3 + r] * res[2 * o + 1];
    }
  }
  V[0] *= 1.0 + lambda;
  V[4] *= 1.0 + lambda;
  V[8] *= 1.0 + lambda;
  double Vi[9];
  const bool ok = !fix_points && det3(V) > 0.0 && inv3(V, Vi);
  if (!ok)
#pragma unroll
    for (int e = 0; e < 9; ++e) Vi[e] = 0.0;
#pragma unroll
  for (int e = 0; e < 9; ++e) Vinv[9 * p + e] = Vi[e];
#pragma unroll
  for (int e = 0; e < 3; ++e) gp[3 * p + e] = g[e];
  for (long long o = o0; o < o1; ++o) {
    const double* jc = Jc + 2 * NC * o;
    const double* jp = Jp + 6 * o;
#pragma unroll
    for (int a = 0; a < NC; ++a) {
      const double w0 = w_entry<NC>(jc, jp, a, 0), w1 = w_entry<NC>(jc, jp, a, 1), w2 = w_entry<NC>(jc, jp, a, 2);
#pragma unroll
      for (int k = 0; k < 3; ++k) Y[3 * NC * o + 3 * a + k] = w0 * Vi[k] + w1 * Vi[3 + k] + w2 * Vi[6 + k];
    }
  }
}

// block b < nimg: image b's 6 columns at 6 b; block nimg + c: camera c's kCam columns at 6 nimg + kCam c, local columns
// 6 .. 5 + kCam of an observation
template <int kCam>
__device__ __forceinline__ void block_geom(int blk, int nimg, int* col0, int* width, int* local0) {
  if (blk < nimg) {
    *col0 = 6 * blk;
    *width = 6;
    *local0 = 0;
  } else {
    *col0 = 6 * nimg + kCam * (blk - nimg);
    *width = kCam;
    *local0 = 6;
  }
}

constexpr int kReduceThreads = 64;

// Stage 1 of the reduced system: one block per chunk (at most NERO_SFM_CHUNK consecutive entries of one segment), one
// thread per entry of the (row block, column block) pair, summed in entry order into partial [chunk, 36] (slot 6 r + c).
// The damping is applied per chunk: (1 + lambda) u + s sums to (1 + lambda) U + S over the chunks.
template <int kCam>
__global__ void __launch_bounds__(kReduceThreads) reduce_chunk_kernel(const int* __restrict__ ent, const long long* __restrict__ chunk,
                                                                      const int* __restrict__ chunk_key, int nimg, const double* __restrict__ Jc,
                                                                      const double* __restrict__ Jp, const double* __restrict__ Y, double lambda,
                                                                      double* __restrict__ partial) {
  constexpr int NC = kNc<kCam>;
  const int k = blockIdx.x;
  int r0, rw, rl, c0, cw, cl;
  block_geom<kCam>(chunk_key[2 * k], nimg, &r0, &rw, &rl);
  block_geom<kCam>(chunk_key[2 * k + 1], nimg, &c0, &cw, &cl);
  const int r = threadIdx.x / 6, c = threadIdx.x % 6;
  if (r >= rw || c >= cw) return;
  const int lr = rl + r, lc = cl + c;
  double u = 0.0, sc = 0.0;
  for (long long e = chunk[2 * k]; e < chunk[2 * k + 1]; ++e) {
    const int o = ent[2 * e], o2 = ent[2 * e + 1];
    const double* jc2 = Jc + 2 * NC * (long long)o2;
    const double* jp2 = Jp + 6 * (long long)o2;
    if (o == o2) u += jc2[lr] * jc2[lc] + jc2[NC + lr] * jc2[NC + lc];
    const double* y = Y + 3 * NC * (long long)o + 3 * lr;
    sc -= y[0] * w_entry<NC>(jc2, jp2, lc, 0) + y[1] * w_entry<NC>(jc2, jp2, lc, 1) + y[2] * w_entry<NC>(jc2, jp2, lc, 2);
  }
  partial[36 * (long long)k + 6 * r + c] = r0 + r == c0 + c ? u + lambda * u + sc : u + sc;
}

// Stage 1 of the right-hand side: one block per chunk of one block's observation list, partial [chunk, 6] (slot r)
template <int kCam>
__global__ void __launch_bounds__(kReduceThreads) rhs_chunk_kernel(const int* __restrict__ obs_seg, const long long* __restrict__ chunk,
                                                                   const int* __restrict__ chunk_blk, const int* __restrict__ obs_pt, int nimg,
                                                                   const double* __restrict__ Jc, const double* __restrict__ res,
                                                                   const double* __restrict__ Y, const double* __restrict__ gp,
                                                                   double* __restrict__ partial) {
  constexpr int NC = kNc<kCam>;
  const int k = blockIdx.x;
  int r0, rw, rl;
  block_geom<kCam>(chunk_blk[k], nimg, &r0, &rw, &rl);
  const int r = threadIdx.x;
  if (r >= rw) return;
  const int lr = rl + r;
  double acc = 0.0;
  for (long long e = chunk[2 * k]; e < chunk[2 * k + 1]; ++e) {
    const int o = obs_seg[2 * e];
    const double* jc = Jc + 2 * NC * (long long)o;
    const double* y = Y + 3 * NC * (long long)o + 3 * lr;
    const double* g = gp + 3 * (long long)obs_pt[o];
    acc += jc[lr] * res[2 * (long long)o] + jc[NC + lr] * res[2 * (long long)o + 1] - (y[0] * g[0] + y[1] * g[1] + y[2] * g[2]);
  }
  partial[6 * (long long)k + r] = acc;
}

// Stage 2: one block per segment adds its chunks' partials in a fixed shape: thread t sums chunks t, t + 64, ... in
// order, then a fixed tree over the 64 threads.  kSlots = 36 writes S (fixed parameters: the identity), kSlots = 6 writes
// b = -sum (fixed parameters: 0).
template <int kSlots, int kCam>
__global__ void __launch_bounds__(kReduceThreads) segment_sum_kernel(const long long* __restrict__ seg_chunk, const int* __restrict__ seg_key,
                                                                     int nimg, int ncol, const double* __restrict__ partial,
                                                                     const unsigned char* __restrict__ fixed, double* __restrict__ out) {
  __shared__ double s_acc[kSlots][kReduceThreads];
  const int s = blockIdx.x, t = threadIdx.x;
  int r0, rw, rl, c0 = 0, cw = 1, cl = 0;
  if (kSlots == 36) {
    block_geom<kCam>(seg_key[2 * s], nimg, &r0, &rw, &rl);
    block_geom<kCam>(seg_key[2 * s + 1], nimg, &c0, &cw, &cl);
  } else {
    block_geom<kCam>(seg_key[s], nimg, &r0, &rw, &rl);
  }
  double acc[kSlots];
#pragma unroll
  for (int e = 0; e < kSlots; ++e) acc[e] = 0.0;
  for (long long k = seg_chunk[s] + t; k < seg_chunk[s + 1]; k += kReduceThreads) {
    const double* pk = partial + kSlots * k;
#pragma unroll
    for (int e = 0; e < kSlots; ++e) {
      const bool valid = kSlots == 36 ? (e / 6 < rw && e % 6 < cw) : e < rw;
      if (valid) acc[e] += pk[e];
    }
  }
#pragma unroll
  for (int e = 0; e < kSlots; ++e) s_acc[e][t] = acc[e];
  __syncthreads();
#pragma unroll
  for (int w = kReduceThreads / 2; w > 0; w >>= 1) {
    if (t < w)
#pragma unroll
      for (int e = 0; e < kSlots; ++e) s_acc[e][t] += s_acc[e][t + w];
    __syncthreads();
  }
  if (kSlots == 36) {
    const int r = t / 6, c = t % 6;
    if (t >= 36 || r >= rw || c >= cw) return;
    const int gr = r0 + r, gc = c0 + c;
    out[(long long)gr * ncol + gc] = (fixed[gr] || fixed[gc]) ? (gr == gc ? 1.0 : 0.0) : s_acc[t][0];
  } else {
    if (t >= rw) return;
    out[r0 + t] = fixed[r0 + t] ? 0.0 : -s_acc[t][0];
  }
}

template <int kCam>
__global__ void __launch_bounds__(kBlock) backsub_kernel(const long long* __restrict__ pt_off, int P, const int* __restrict__ obs_img,
                                                         const int* __restrict__ img_cam, int nimg, int ncam, const double* __restrict__ Jc,
                                                         const double* __restrict__ Jp, const double* __restrict__ Vinv,
                                                         const double* __restrict__ gp, const double* __restrict__ dc,
                                                         const double* __restrict__ pose, const double* __restrict__ focal,
                                                         const double* __restrict__ Xin, double* __restrict__ pose_new,
                                                         double* __restrict__ focal_new, double* __restrict__ X_new,
                                                         const double* __restrict__ radial, double* __restrict__ radial_new) {
  constexpr int NC = kNc<kCam>;
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx < P) {
    const int p = (int)idx;
    double acc[3] = {gp[3 * p], gp[3 * p + 1], gp[3 * p + 2]};
    for (long long o = pt_off[p]; o < pt_off[p + 1]; ++o) {
      const int i = obs_img[o];
      double dn[NC];
#pragma unroll
      for (int a = 0; a < 6; ++a) dn[a] = dc[6 * i + a];
#pragma unroll
      for (int a = 0; a < kCam; ++a) dn[6 + a] = dc[6 * nimg + kCam * img_cam[i] + a];
      const double* jc = Jc + 2 * NC * o;
      const double* jp = Jp + 6 * o;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        double s = 0.0;
#pragma unroll
        for (int a = 0; a < NC; ++a) s += w_entry<NC>(jc, jp, a, k) * dn[a];
        acc[k] += s;
      }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double dx = -(Vinv[9 * p + 3 * k] * acc[0] + Vinv[9 * p + 3 * k + 1] * acc[1] + Vinv[9 * p + 3 * k + 2] * acc[2]);
      X_new[3 * p + k] = Xin[3 * p + k] + dx;
    }
  } else if (idx < (long long)P + nimg) {
    const int i = (int)(idx - P);
    double R[9], t[3], Rn[9];
    load_pose(pose, i, R, t);
    const double w[3] = {dc[6 * i], dc[6 * i + 1], dc[6 * i + 2]};
    rotate_left(w, R, Rn);
#pragma unroll
    for (int e = 0; e < 9; ++e) pose_new[12 * i + e] = Rn[e];
#pragma unroll
    for (int e = 0; e < 3; ++e) pose_new[12 * i + 9 + e] = t[e] + dc[6 * i + 3 + e];
  } else if (idx < (long long)P + nimg + ncam) {
    const int c = (int)(idx - P - nimg);
    focal_new[c] = focal[c] + dc[6 * nimg + kCam * c];
    if constexpr (kCam == 2) radial_new[c] = radial[c] + dc[6 * nimg + 2 * c + 1];
  }
}

template <int kCam>
__global__ void __launch_bounds__(kBlock) cost_kernel(const long long* __restrict__ pt_off, int P, const int* __restrict__ obs_img,
                                                      const double* __restrict__ obs_xy, const double* __restrict__ pose,
                                                      const int* __restrict__ img_cam, const double* __restrict__ focal,
                                                      const double* __restrict__ pp, const double* __restrict__ Xin,
                                                      double* __restrict__ partial, const double* __restrict__ radial) {
  __shared__ double s_v[kBlock];
  const int p = blockIdx.x * kBlock + threadIdx.x;
  double acc = 0.0;
  if (p < P) {
    const double X[3] = {Xin[3 * p], Xin[3 * p + 1], Xin[3 * p + 2]};
    for (long long o = pt_off[p]; o < pt_off[p + 1]; ++o) {
      const Cam c = load_cam<kCam>(pose, img_cam, focal, pp, obs_img[o], radial);
      double z;
      acc += reproj2<kCam>(c, X, obs_xy[2 * o], obs_xy[2 * o + 1], &z);
    }
  }
  s_v[threadIdx.x] = acc;
  __syncthreads();
  for (int w = kBlock / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s_v[threadIdx.x] += s_v[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = s_v[0];
}

__global__ void cost_sum_kernel(const double* __restrict__ partial, int nblk, double* __restrict__ cost) {
  double s = 0.0;
  for (int k = 0; k < nblk; ++k) s += partial[k];
  cost[0] = s;
}

// the reduced system of either camera model (kCam parameters per camera), checked and launched
template <int kCam>
int reduce(const int* ent, const long long* chunk, const int* chunk_key, int nchunk, const long long* seg_chunk, const int* seg_key,
           int nseg, const int* obs_seg, const long long* rchunk, const int* rchunk_blk, int nrchunk, const long long* rseg_chunk,
           const int* rseg_blk, int nrseg, const int* obs_pt, const int* img_cam, int nimg, int ncam, const double* Jc,
           const double* Jp, const double* res, const double* Y, const double* gp, double lambda, const unsigned char* fixed,
           double* partial, double* rpartial, double* S, double* b, void* stream) {
  if (nchunk < 0 || nseg < 0 || nrchunk < 0 || nrseg < 0 || nimg < 1 || nimg > NERO_SFM_MAX_IMAGES || ncam < 1 || ncam > nimg ||
      !(lambda >= 0.0) || !fixed || !S || !b || (nchunk > 0) != (nseg > 0) || (nrchunk > 0) != (nrseg > 0) ||
      (nchunk > 0 && (!ent || !chunk || !chunk_key || !seg_chunk || !seg_key || !Jc || !Jp || !Y || !partial)) ||
      (nrchunk > 0 && (!obs_seg || !rchunk || !rchunk_blk || !rseg_chunk || !rseg_blk || !obs_pt || !img_cam || !Jc || !res || !Y || !gp ||
                       !rpartial)))
    return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int ncol = 6 * nimg + kCam * ncam;
  if (nchunk > 0) {
    reduce_chunk_kernel<kCam><<<nchunk, kReduceThreads, 0, s>>>(ent, chunk, chunk_key, nimg, Jc, Jp, Y, lambda, partial);
    segment_sum_kernel<36, kCam><<<nseg, kReduceThreads, 0, s>>>(seg_chunk, seg_key, nimg, ncol, partial, fixed, S);
  }
  if (nrchunk > 0) {
    rhs_chunk_kernel<kCam><<<nrchunk, kReduceThreads, 0, s>>>(obs_seg, rchunk, rchunk_blk, obs_pt, nimg, Jc, res, Y, gp, rpartial);
    segment_sum_kernel<6, kCam><<<nrseg, kReduceThreads, 0, s>>>(rseg_chunk, rseg_blk, nimg, ncol, rpartial, fixed, b);
  }
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace

extern "C" {

int nero_sfm_tracks(const int* edges, int E, int N, int* label, int* blk_count, long long* blk_off, long long* total, int* track,
                    void* stream) {
  if (E < 0 || N < 1 || (E > 0 && !edges) || !label || !blk_count || !blk_off || !total || !track) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  uf_init(label, N, s);
  if (E > 0) hook_kernel<<<blocks(E), kBlock, 0, s>>>(edges, E, label);
  uf_flatten(label, N, s);
  const unsigned nb = blocks(N);
  root_count_kernel<<<nb, kBlock, 0, s>>>(label, N, blk_count);
  block_offsets<1>(blk_count, blk_off, total, nb, s);
  root_emit_kernel<<<nb, kBlock, 0, s>>>(label, N, blk_off, track);
  track_map_kernel<<<nb, kBlock, 0, s>>>(label, N, track);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_p3p(const double* xy, const double* X, int n, double f, double cx, double cy, int image, int hypotheses,
                 unsigned int seed, double max_err2, int* counts, double* poses, int* best, double* pose, unsigned char* inlier,
                 void* stream) {
  if (n < 3 || !xy || !X || !counts || !poses || !best || !pose || !inlier || hypotheses < 1 || hypotheses > NERO_SFM_MAX_HYP ||
      !(f > 0.0) || !(max_err2 >= 0.0))
    return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  p3p_kernel<<<blocks(hypotheses), kBlock, 0, s>>>(xy, X, n, f, cx, cy, image, hypotheses, seed, max_err2, counts, poses);
  p3p_select_kernel<<<1, kBlock, 0, s>>>(xy, X, n, f, cx, cy, hypotheses, max_err2, counts, poses, best, pose, inlier);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_triangulate(const long long* off, int T, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                         const double* focal, const double* pp, double* X, double* stat, void* stream) {
  if (T < 0 || (T > 0 && (!off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !X || !stat))) return NERO_ERR_ARG;
  if (T == 0) return NERO_OK;
  triangulate_kernel<<<blocks(T), kBlock, 0, (cudaStream_t)stream>>>(off, T, obs_img, obs_xy, pose, img_cam, focal, pp, X, stat);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_filter(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                    const double* focal, const double* pp, const double* X, double* err, double* angle, void* stream) {
  if (P < 0 || (P > 0 && (!pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !X || !err || !angle))) return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  filter_kernel<1><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, err, angle, nullptr);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_ba_linearize(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose,
                          const int* img_cam, const double* focal, const double* pp, const double* X, double* res, double* Jc,
                          double* Jp, void* stream) {
  if (P < 0 || (P > 0 && (!pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !X || !res || !Jc || !Jp)))
    return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  linearize_kernel<1><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, res, Jc, Jp,
                                                                      nullptr);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_ba_points(const long long* pt_off, int P, const double* res, const double* Jc, const double* Jp, double lambda, int fix_points,
                       double* Vinv, double* gp, double* Y, void* stream) {
  if (P < 0 || !(lambda >= 0.0) || (P > 0 && (!pt_off || !res || !Jc || !Jp || !Vinv || !gp || !Y))) return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  points_kernel<1><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, res, Jc, Jp, lambda, fix_points, Vinv, gp, Y);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_ba_reduce(const int* ent, const long long* chunk, const int* chunk_key, int nchunk, const long long* seg_chunk, const int* seg_key,
                       int nseg, const int* obs_seg, const long long* rchunk, const int* rchunk_blk, int nrchunk, const long long* rseg_chunk,
                       const int* rseg_blk, int nrseg, const int* obs_pt, const int* img_cam, int nimg, int ncam, const double* Jc,
                       const double* Jp, const double* res, const double* Y, const double* gp, double lambda, const unsigned char* fixed,
                       double* partial, double* rpartial, double* S, double* b, void* stream) {
  return reduce<1>(ent, chunk, chunk_key, nchunk, seg_chunk, seg_key, nseg, obs_seg, rchunk, rchunk_blk, nrchunk, rseg_chunk, rseg_blk, nrseg,
                   obs_pt, img_cam, nimg, ncam, Jc, Jp, res, Y, gp, lambda, fixed, partial, rpartial, S, b, stream);
}

int nero_sfm_ba_backsub(const long long* pt_off, int P, const int* obs_img, const int* img_cam, int nimg, int ncam, const double* Jc,
                        const double* Jp, const double* Vinv, const double* gp, const double* dc, const double* pose, const double* focal,
                        const double* X, double* pose_new, double* focal_new, double* X_new, void* stream) {
  if (P < 0 || nimg < 1 || ncam < 1 || !dc || !pose || !focal || !pose_new || !focal_new || !img_cam ||
      (P > 0 && (!pt_off || !obs_img || !Jc || !Jp || !Vinv || !gp || !X || !X_new)))
    return NERO_ERR_ARG;
  backsub_kernel<1><<<blocks((long long)P + nimg + ncam), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, img_cam, nimg, ncam, Jc, Jp,
                                                                                             Vinv, gp, dc, pose, focal, X, pose_new, focal_new,
                                                                                             X_new, nullptr, nullptr);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_ba_cost(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                     const double* focal, const double* pp, const double* X, double* partial, double* cost, void* stream) {
  if (P < 1 || !pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !X || !partial || !cost) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const unsigned nb = blocks(P);
  cost_kernel<1><<<nb, kBlock, 0, s>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, partial, nullptr);
  cost_sum_kernel<<<1, 1, 0, s>>>(partial, (int)nb, cost);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_radial_filter(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                           const double* focal, const double* pp, const double* radial, const double* X, double* err, double* angle,
                           void* stream) {
  if (P < 0 || (P > 0 && (!pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !radial || !X || !err || !angle)))
    return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  filter_kernel<2><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, err, angle, radial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_radial_ba_linearize(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose,
                                 const int* img_cam, const double* focal, const double* pp, const double* radial, const double* X,
                                 double* res, double* Jc, double* Jp, void* stream) {
  if (P < 0 || (P > 0 && (!pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !radial || !X || !res || !Jc || !Jp)))
    return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  linearize_kernel<2><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, res, Jc, Jp,
                                                                      radial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_radial_ba_points(const long long* pt_off, int P, const double* res, const double* Jc, const double* Jp, double lambda,
                              int fix_points, double* Vinv, double* gp, double* Y, void* stream) {
  if (P < 0 || !(lambda >= 0.0) || (P > 0 && (!pt_off || !res || !Jc || !Jp || !Vinv || !gp || !Y))) return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  points_kernel<2><<<blocks(P), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, res, Jc, Jp, lambda, fix_points, Vinv, gp, Y);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_radial_ba_reduce(const int* ent, const long long* chunk, const int* chunk_key, int nchunk, const long long* seg_chunk,
                              const int* seg_key, int nseg, const int* obs_seg, const long long* rchunk, const int* rchunk_blk, int nrchunk,
                              const long long* rseg_chunk, const int* rseg_blk, int nrseg, const int* obs_pt, const int* img_cam, int nimg,
                              int ncam, const double* Jc, const double* Jp, const double* res, const double* Y, const double* gp,
                              double lambda, const unsigned char* fixed, double* partial, double* rpartial, double* S, double* b,
                              void* stream) {
  return reduce<2>(ent, chunk, chunk_key, nchunk, seg_chunk, seg_key, nseg, obs_seg, rchunk, rchunk_blk, nrchunk, rseg_chunk, rseg_blk, nrseg,
                   obs_pt, img_cam, nimg, ncam, Jc, Jp, res, Y, gp, lambda, fixed, partial, rpartial, S, b, stream);
}

int nero_sfm_radial_ba_backsub(const long long* pt_off, int P, const int* obs_img, const int* img_cam, int nimg, int ncam, const double* Jc,
                               const double* Jp, const double* Vinv, const double* gp, const double* dc, const double* pose,
                               const double* focal, const double* radial, const double* X, double* pose_new, double* focal_new,
                               double* radial_new, double* X_new, void* stream) {
  if (P < 0 || nimg < 1 || ncam < 1 || !dc || !pose || !focal || !radial || !pose_new || !focal_new || !radial_new || !img_cam ||
      (P > 0 && (!pt_off || !obs_img || !Jc || !Jp || !Vinv || !gp || !X || !X_new)))
    return NERO_ERR_ARG;
  backsub_kernel<2><<<blocks((long long)P + nimg + ncam), kBlock, 0, (cudaStream_t)stream>>>(pt_off, P, obs_img, img_cam, nimg, ncam, Jc, Jp,
                                                                                             Vinv, gp, dc, pose, focal, X, pose_new, focal_new,
                                                                                             X_new, radial, radial_new);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_sfm_radial_ba_cost(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                            const double* focal, const double* pp, const double* radial, const double* X, double* partial, double* cost,
                            void* stream) {
  if (P < 1 || !pt_off || !obs_img || !obs_xy || !pose || !img_cam || !focal || !pp || !radial || !X || !partial || !cost) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const unsigned nb = blocks(P);
  cost_kernel<2><<<nb, kBlock, 0, s>>>(pt_off, P, obs_img, obs_xy, pose, img_cam, focal, pp, X, partial, radial);
  cost_sum_kernel<<<1, 1, 0, s>>>(partial, (int)nb, cost);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
