// Geometric verification of matched image pairs: the GPU replacement of the two-view geometry stage of COLMAP's
// exhaustive_matcher.  The protocol is stated in nero_b200/features.py, the ABI in include/nero_features.h.
//
//   verify   one block (one warp) per pair.  Each lane solves every 32nd of the pair's hypotheses: 8 distinct matches
//            drawn by hash, the normalised 8-point system summed in draw order, its null vector by cyclic Jacobi on the 9 x 9
//            normal matrix, the rank-2 projection through a 3 x 3 Jacobi, and an inlier count by the Sampson distance.
//            The Jacobi matrices live in the lane's own column of shared memory ([entry][lane]), so nothing spills.  Lane 0
//            picks the winner (largest count, then lower hypothesis) and refits it once on its inliers, summing in match
//            order; the refit's inliers are final.
// All arithmetic is fp64; the winner and the inlier sets do not depend on scheduling.
#include <cmath>

#include "common.cuh"
#include "hash.cuh"
#include "../../include/nero_features.h"

namespace nero {
namespace {

constexpr int kLanes = 32;
constexpr int kSweeps9 = 12, kSweeps3 = 8;
constexpr int kMaxDraws = 64;

struct Norm {
  double c1x, c1y, s1, c2x, c2y, s2;
};

// cyclic Jacobi on the symmetric n x n matrix A (entry (r, c) at A[(r n + c) kLanes]); V receives the eigenvectors (columns)
__device__ __forceinline__ void jacobi(double* A, double* V, int n, int sweeps) {
#define EA(r, c) A[((r) * n + (c)) * kLanes]
#define EV(r, c) V[((r) * n + (c)) * kLanes]
  for (int r = 0; r < n; ++r)
    for (int c = 0; c < n; ++c) EV(r, c) = r == c ? 1.0 : 0.0;
  for (int sw = 0; sw < sweeps; ++sw)
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        const double apq = EA(p, q);
        if (apq == 0.0) continue;
        const double theta = (EA(q, q) - EA(p, p)) / (2.0 * apq);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < n; ++k) {
          const double akp = EA(k, p), akq = EA(k, q);
          EA(k, p) = c * akp - s * akq;
          EA(k, q) = s * akp + c * akq;
        }
        for (int k = 0; k < n; ++k) {
          const double apk = EA(p, k), aqk = EA(q, k);
          EA(p, k) = c * apk - s * aqk;
          EA(q, k) = s * apk + c * aqk;
        }
        for (int k = 0; k < n; ++k) {
          const double vkp = EV(k, p), vkq = EV(k, q);
          EV(k, p) = c * vkp - s * vkq;
          EV(k, q) = s * vkp + c * vkq;
        }
      }
}

// index of the smallest diagonal entry (ties: lower)
__device__ __forceinline__ int smallest(const double* A, int n) {
  int m = 0;
  for (int k = 1; k < n; ++k)
    if (EA(k, k) < EA(m, m)) m = k;
  return m;
}
#undef EA
#undef EV

// adds a a^T of the epipolar row of one normalised correspondence to M
__device__ __forceinline__ void accumulate(double* M, const double* p, const Norm& nm) {
  const double x1 = (p[0] - nm.c1x) * nm.s1, y1 = (p[1] - nm.c1y) * nm.s1;
  const double x2 = (p[2] - nm.c2x) * nm.s2, y2 = (p[3] - nm.c2y) * nm.s2;
  const double a[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
#pragma unroll
  for (int r = 0; r < 9; ++r)
#pragma unroll
    for (int c = 0; c < 9; ++c) M[(r * 9 + c) * kLanes] += a[r] * a[c];
}

// F (pixel coordinates, unit norm, largest |entry| positive) from the normal matrix M of normalised rows; M and V are
// scratch
__device__ __forceinline__ void solve_F(double* M, double* V, const Norm& nm, double F[9]) {
  jacobi(M, V, 9, kSweeps9);
  const int m = smallest(M, 9);
  double f[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) f[k] = V[(k * 9 + m) * kLanes];
  // rank 2: f <- f (I - v v^T) with v the eigenvector of f^T f of the smallest eigenvalue
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) M[(r * 3 + c) * kLanes] = f[r] * f[c] + f[3 + r] * f[3 + c] + f[6 + r] * f[6 + c];
  jacobi(M, V, 3, kSweeps3);
  const int s = smallest(M, 3);
  const double v[3] = {V[(0 * 3 + s) * kLanes], V[(1 * 3 + s) * kLanes], V[(2 * 3 + s) * kLanes]};
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double fv = f[3 * r] * v[0] + f[3 * r + 1] * v[1] + f[3 * r + 2] * v[2];
#pragma unroll
    for (int c = 0; c < 3; ++c) f[3 * r + c] -= fv * v[c];
  }
  // F = T2^T f T1, T = [[s, 0, -s cx], [0, s, -s cy], [0, 0, 1]]
  const double t1[6] = {nm.s1, 0.0, -nm.s1 * nm.c1x, 0.0, nm.s1, -nm.s1 * nm.c1y};
  const double t2[6] = {nm.s2, 0.0, -nm.s2 * nm.c2x, 0.0, nm.s2, -nm.s2 * nm.c2y};
  double g[9];   // f T1
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    g[3 * r + 0] = f[3 * r] * t1[0];
    g[3 * r + 1] = f[3 * r + 1] * t1[4];
    g[3 * r + 2] = f[3 * r] * t1[2] + f[3 * r + 1] * t1[5] + f[3 * r + 2];
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    F[c] = t2[0] * g[c];
    F[3 + c] = t2[4] * g[3 + c];
    F[6 + c] = t2[2] * g[c] + t2[5] * g[3 + c] + g[6 + c];
  }
  double n2 = 0.0, big = F[0];   // the first entry of the largest magnitude
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    n2 += F[k] * F[k];
    big = fabs(F[k]) > fabs(big) ? F[k] : big;
  }
  const double inv = (big < 0.0 ? -1.0 : 1.0) / sqrt(n2);
#pragma unroll
  for (int k = 0; k < 9; ++k) F[k] *= inv;
}

__device__ __forceinline__ bool inlier_of(const double F[9], const double* p, double max_err2) {
  const double x1 = p[0], y1 = p[1], x2 = p[2], y2 = p[3];
  const double l0 = F[0] * x1 + F[1] * y1 + F[2], l1 = F[3] * x1 + F[4] * y1 + F[5], l2 = F[6] * x1 + F[7] * y1 + F[8];
  const double m0 = F[0] * x2 + F[3] * y2 + F[6], m1 = F[1] * x2 + F[4] * y2 + F[7];
  const double e = x2 * l0 + y2 * l1 + l2;
  return e * e <= max_err2 * (l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1);
}

__device__ __forceinline__ uint32_t draw_key(unsigned seed, int pair, int hyp, int draw) {
  uint32_t h = rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u);
  h = rl_mix(h ^ (uint32_t)pair);
  h = rl_mix(h ^ (uint32_t)hyp);
  return rl_mix(h ^ (uint32_t)draw);
}

__global__ void __launch_bounds__(kLanes) verify_kernel(const double* __restrict__ pts, const long long* __restrict__ off, int hypotheses,
                                                        unsigned seed, double max_err2, double* __restrict__ Fout, int* __restrict__ best,
                                                        int* __restrict__ count, unsigned char* __restrict__ inlier) {
  __shared__ double sM[81 * kLanes], sV[81 * kLanes];
  __shared__ double sF[9 * kLanes];
  __shared__ int sCnt[kLanes], sHyp[kLanes], sIdx[8 * kLanes];
  __shared__ Norm sN;
  const int lane = threadIdx.x, p = blockIdx.x;
  const long long base = off[p];
  const int n = (int)(off[p + 1] - base);
  const double* P = pts + 4 * base;
  if (n < 8) {
    for (int m = lane; m < n; m += kLanes) inlier[base + m] = 0;
    if (lane < 9) Fout[9 * p + lane] = 0.0;
    if (lane == 0) {
      best[2 * p] = -1;
      best[2 * p + 1] = 0;
      count[p] = 0;
    }
    return;
  }
  if (lane == 0) {
    double sx1 = 0, sy1 = 0, sx2 = 0, sy2 = 0;
    for (int m = 0; m < n; ++m) {
      sx1 += P[4 * m]; sy1 += P[4 * m + 1]; sx2 += P[4 * m + 2]; sy2 += P[4 * m + 3];
    }
    Norm nm;
    nm.c1x = sx1 / n; nm.c1y = sy1 / n; nm.c2x = sx2 / n; nm.c2y = sy2 / n;
    double d1 = 0, d2 = 0;
    for (int m = 0; m < n; ++m) {
      d1 += sqrt((P[4 * m] - nm.c1x) * (P[4 * m] - nm.c1x) + (P[4 * m + 1] - nm.c1y) * (P[4 * m + 1] - nm.c1y));
      d2 += sqrt((P[4 * m + 2] - nm.c2x) * (P[4 * m + 2] - nm.c2x) + (P[4 * m + 3] - nm.c2y) * (P[4 * m + 3] - nm.c2y));
    }
    nm.s1 = d1 > 0.0 ? 1.4142135623730951 * n / d1 : 1.0;
    nm.s2 = d2 > 0.0 ? 1.4142135623730951 * n / d2 : 1.0;
    sN = nm;
  }
  __syncthreads();
  const Norm nm = sN;
  double* M = sM + lane;
  double* V = sV + lane;
  int* idx = sIdx + lane;
  int bc = -1, bh = -1;
  for (int h = lane; h < hypotheses; h += kLanes) {
    int k = 0;
    for (int d = 0; d < kMaxDraws && k < 8; ++d) {
      const int m = (int)(draw_key(seed, p, h, d) % (uint32_t)n);
      bool dup = false;
      for (int j = 0; j < k; ++j) dup = dup || idx[j * kLanes] == m;
      if (!dup) idx[(k++) * kLanes] = m;
    }
    if (k < 8) continue;
    for (int e = 0; e < 81; ++e) M[e * kLanes] = 0.0;
    for (int j = 0; j < 8; ++j) accumulate(M, P + 4 * idx[j * kLanes], nm);
    double F[9];
    solve_F(M, V, nm, F);
    int c = 0;
    for (int m = 0; m < n; ++m) c += inlier_of(F, P + 4 * m, max_err2);
    if (c > bc) {
      bc = c;
      bh = h;
#pragma unroll
      for (int e = 0; e < 9; ++e) sF[e * kLanes + lane] = F[e];
    }
  }
  sCnt[lane] = bc;
  sHyp[lane] = bh;
  __syncthreads();
  __shared__ int sWin;
  if (lane == 0) {
    int w = 0;
    for (int l = 1; l < kLanes; ++l)
      if (sCnt[l] > sCnt[w] || (sCnt[l] == sCnt[w] && (unsigned)sHyp[l] < (unsigned)sHyp[w])) w = l;
    sWin = w;
    best[2 * p] = sHyp[w];
    best[2 * p + 1] = max(sCnt[w], 0);
  }
  __syncthreads();
  const int w = sWin;
  double F[9];
#pragma unroll
  for (int e = 0; e < 9; ++e) F[e] = sF[e * kLanes + w];
  for (int m = lane; m < n; m += kLanes) inlier[base + m] = sHyp[w] >= 0 && inlier_of(F, P + 4 * m, max_err2);
  __syncthreads();
  if (lane == 0) {
    if (sCnt[w] >= 8) {
      for (int e = 0; e < 81; ++e) M[e * kLanes] = 0.0;
      for (int m = 0; m < n; ++m)
        if (inlier[base + m]) accumulate(M, P + 4 * m, nm);
      solve_F(M, V, nm, F);
    } else if (sHyp[w] < 0) {
#pragma unroll
      for (int e = 0; e < 9; ++e) F[e] = 0.0;
    }
#pragma unroll
    for (int e = 0; e < 9; ++e) sF[e * kLanes] = F[e];
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < 9; ++e) F[e] = sF[e * kLanes];
  int c = 0;
  for (int m0 = 0; m0 < n; m0 += kLanes) {
    const int m = m0 + lane;
    const bool in = m < n && sHyp[w] >= 0 && inlier_of(F, P + 4 * (size_t)min(m, n - 1), max_err2);
    if (m < n) inlier[base + m] = in;
    c += __popc(__ballot_sync(0xffffffffu, in));
  }
  if (lane < 9) Fout[9 * p + lane] = sF[lane * kLanes];
  if (lane == 0) count[p] = c;
}

}  // namespace

extern "C" {

int nero_features_verify(const double* pts, const long long* off, int P, int hypotheses, unsigned int seed, double max_err2, double* F,
                         int* best, int* count, unsigned char* inlier, void* stream) {
  if (P < 0 || (P > 0 && (!pts || !off || !F || !best || !count || !inlier)) || hypotheses < 1 || hypotheses > NERO_FEATURES_MAX_HYP ||
      !(max_err2 >= 0.0))
    return NERO_ERR_ARG;
  if (P == 0) return NERO_OK;
  verify_kernel<<<P, kLanes, 0, (cudaStream_t)stream>>>(pts, off, hypotheses, seed, max_err2, F, best, count, inlier);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
