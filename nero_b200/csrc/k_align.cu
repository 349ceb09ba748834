// Mesh registration kernels: the similarity transform of source points, the point-to-plane Gauss-Newton terms of one ICP
// iteration, the moments of the principal-axis start, the trimmed score of its candidates, and the fixed-order reduction of
// their per-block partials.  include/nero_align.h states every operation; oracle/nero_oracle_align.py repeats them in numpy
// bit for bit.
//
// Every block-partial kernel sums its 256 points by the same pairwise tree: levels h = 1 .. 16 inside a warp by
// __shfl_down_sync (lane t, t divisible by 2h, adds lane t + h), then levels 32 .. 128 over the eight warp sums in shared
// memory.  No floating-point atomics: the sums do not depend on scheduling.
#include <cmath>

#include "common.cuh"
#include "../../include/nero_align.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_ALIGN_BLOCK;
constexpr int kWarps = kBlock / 32;
constexpr int kTerms = NERO_ALIGN_TERMS;
constexpr int kMoments = NERO_ALIGN_MOMENTS;
constexpr int kMaxWidth = NERO_ALIGN_MAX_WIDTH;
static_assert(kBlock == 256, "the pairwise tree of include/nero_align.h sums 256 values per block");

struct D3 { double x, y, z; };

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ D3 sub(const D3& a, const D3& b) { return {ds(a.x, b.x), ds(a.y, b.y), ds(a.z, b.z)}; }
__device__ __forceinline__ double dot(const D3& a, const D3& b) { return da(da(dm(a.x, b.x), dm(a.y, b.y)), dm(a.z, b.z)); }
__device__ __forceinline__ D3 cross(const D3& a, const D3& b) {
  return {ds(dm(a.y, b.z), dm(a.z, b.y)), ds(dm(a.z, b.x), dm(a.x, b.z)), ds(dm(a.x, b.y), dm(a.y, b.x))};
}

__device__ __forceinline__ D3 vert(const float* __restrict__ verts, int i) {
  return {(double)__ldg(verts + 3 * i), (double)__ldg(verts + 3 * i + 1), (double)__ldg(verts + 3 * i + 2)};
}

// levels h = 1 .. 16 of the pairwise tree: lane 0 ends with the sum of the warp's 32 values
__device__ __forceinline__ double warp_tree(double v) {
#pragma unroll
  for (int h = 1; h < 32; h <<= 1) v = da(v, __shfl_down_sync(0xffffffffu, v, h));
  return v;
}

// levels h = 32 .. 128: the pairwise tree over the eight warp sums of column v
__device__ __forceinline__ double warps_tree(const double (*s)[kMaxWidth], int v) {
  return da(da(da(s[0][v], s[1][v]), da(s[2][v], s[3][v])), da(da(s[4][v], s[5][v]), da(s[6][v], s[7][v])));
}

// column v of the block: the warp level, and lane 0 keeps the warp's sum for warps_tree after the caller's barrier
__device__ __forceinline__ void put(double (*s)[kMaxWidth], int v, double x) {
  x = warp_tree(x);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5][v] = x;
}

__global__ void transform_kernel(const double* __restrict__ points, long long n, const double* __restrict__ mats, int k,
                                 double* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= n * k) return;
  const long long j = idx / n, i = idx - j * n;
  const double x = points[3 * i], y = points[3 * i + 1], z = points[3 * i + 2];
  const double* m = mats + 12 * j;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    out[3 * idx + r] = da(da(da(dm(__ldg(m + 4 * r), x), dm(__ldg(m + 4 * r + 1), y)), dm(__ldg(m + 4 * r + 2), z)), __ldg(m + 4 * r + 3));
}

__global__ void __launch_bounds__(kBlock) terms_kernel(const double* __restrict__ points, long long n, const int* __restrict__ tri,
                                                       const double* __restrict__ closest, const float* __restrict__ verts,
                                                       const int* __restrict__ tris, D3 center, double* __restrict__ partial) {
  __shared__ double s[kWarps][kMaxWidth];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  double J[7] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  double r = 0.0, used = 0.0, degenerate = 0.0;
  const int id = i < n ? tri[i] : -1;
  if (id >= 0) {
    const D3 a = vert(verts, __ldg(tris + 3 * id)), b = vert(verts, __ldg(tris + 3 * id + 1)), c = vert(verts, __ldg(tris + 3 * id + 2));
    const D3 m = cross(sub(b, a), sub(c, a));
    if (m.x == 0.0 && m.y == 0.0 && m.z == 0.0) {
      degenerate = 1.0;
    } else {
      const double l = __dsqrt_rn(dot(m, m));
      const D3 nrm{dd(m.x, l), dd(m.y, l), dd(m.z, l)};
      const D3 y{points[3 * i], points[3 * i + 1], points[3 * i + 2]};
      const D3 q{closest[3 * i], closest[3 * i + 1], closest[3 * i + 2]};
      const D3 d = sub(y, center);
      r = dot(nrm, sub(y, q));
      const D3 w = cross(d, nrm);
      J[0] = w.x; J[1] = w.y; J[2] = w.z;
      J[3] = nrm.x; J[4] = nrm.y; J[5] = nrm.z;
      J[6] = dot(nrm, d);
      used = 1.0;
    }
  }
  int v = 0;
#pragma unroll
  for (int a = 0; a < 7; ++a)
#pragma unroll
    for (int b = a; b < 7; ++b) put(s, v++, dm(J[a], J[b]));
#pragma unroll
  for (int a = 0; a < 7; ++a) put(s, v++, dm(J[a], r));
  put(s, v++, dm(r, r));
  put(s, v++, used);
  put(s, v++, degenerate);
  __syncthreads();
  if (threadIdx.x < kTerms) partial[(long long)blockIdx.x * kTerms + threadIdx.x] = warps_tree(s, threadIdx.x);
}

__global__ void __launch_bounds__(kBlock) moments_kernel(const double* __restrict__ points, long long n, D3 origin,
                                                         double* __restrict__ partial) {
  __shared__ double s[kWarps][kMaxWidth];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  D3 d{0.0, 0.0, 0.0};
  double one = 0.0;
  if (i < n) {
    d = sub(D3{points[3 * i], points[3 * i + 1], points[3 * i + 2]}, origin);
    one = 1.0;
  }
  put(s, 0, one);
  put(s, 1, d.x);
  put(s, 2, d.y);
  put(s, 3, d.z);
  put(s, 4, dm(d.x, d.x));
  put(s, 5, dm(d.x, d.y));
  put(s, 6, dm(d.x, d.z));
  put(s, 7, dm(d.y, d.y));
  put(s, 8, dm(d.y, d.z));
  put(s, 9, dm(d.z, d.z));
  __syncthreads();
  if (threadIdx.x < kMoments) partial[(long long)blockIdx.x * kMoments + threadIdx.x] = warps_tree(s, threadIdx.x);
}

// grid (blocks per segment, segments)
__global__ void __launch_bounds__(kBlock) score_kernel(const double* __restrict__ dist, long long m, double tau,
                                                       double* __restrict__ partial) {
  __shared__ double s[kWarps][kMaxWidth];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  double x = 0.0;
  if (i < m) {
    const double v = fmin(dist[(long long)blockIdx.y * m + i], tau);
    x = dm(v, v);
  }
  put(s, 0, x);
  __syncthreads();
  if (threadIdx.x == 0) partial[(long long)blockIdx.y * gridDim.x + blockIdx.x] = warps_tree(s, 0);
}

// one block per segment, reducing its rows in place level by level (include/nero_align.h, Reduce).  A level writes row c
// only after every thread has read chunk c (rows 256 c and up), so no row is overwritten before it is read.
__global__ void __launch_bounds__(kBlock) reduce_kernel(double* partial, long long blocks, int width, double* __restrict__ out) {
  __shared__ double s[kWarps][kMaxWidth];
  double* base = partial + (long long)blockIdx.x * blocks * width;
  for (long long m = blocks; m > 1;) {
    const long long chunks = (m + kBlock - 1) / kBlock;
    for (long long c = 0; c < chunks; ++c) {
      const long long row = c * kBlock + threadIdx.x;
      for (int v = 0; v < width; ++v) put(s, v, row < m ? base[row * width + v] : 0.0);
      __syncthreads();
      if (threadIdx.x < width) base[c * width + threadIdx.x] = warps_tree(s, threadIdx.x);
      __syncthreads();
    }
    m = chunks;
  }
  if (threadIdx.x < width) out[(long long)blockIdx.x * width + threadIdx.x] = base[threadIdx.x];
}

inline unsigned blocks_of(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

}  // namespace

extern "C" int nero_align_transform(const double* points, long long n, const double* mats, int k, double* out, void* stream) {
  if (n < 0 || k < 1) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!points || !mats || !out) return NERO_ERR_ARG;
  transform_kernel<<<blocks_of(n * k), kBlock, 0, (cudaStream_t)stream>>>(points, n, mats, k, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_align_terms(const double* points, long long n, const int* tri, const double* closest, const float* verts,
                                const int* tris, double cx, double cy, double cz, double* partial, void* stream) {
  if (n < 0) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!points || !tri || !closest || !verts || !tris || !partial) return NERO_ERR_ARG;
  terms_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(points, n, tri, closest, verts, tris, D3{cx, cy, cz}, partial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_align_moments(const double* points, long long n, double ox, double oy, double oz, double* partial, void* stream) {
  if (n < 0) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!points || !partial) return NERO_ERR_ARG;
  moments_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(points, n, D3{ox, oy, oz}, partial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_align_score(const double* dist, long long m, int k, double tau, double* partial, void* stream) {
  if (m < 1 || k < 1 || k > 65535 || !(tau >= 0.0) || !dist || !partial) return NERO_ERR_ARG;
  score_kernel<<<dim3(blocks_of(m), unsigned(k)), kBlock, 0, (cudaStream_t)stream>>>(dist, m, tau, partial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_align_reduce(double* partial, int segments, long long blocks, int width, double* out, void* stream) {
  if (segments < 1 || blocks < 1 || width < 1 || width > kMaxWidth || !partial || !out) return NERO_ERR_ARG;
  reduce_kernel<<<unsigned(segments), kBlock, 0, (cudaStream_t)stream>>>(partial, blocks, width, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
