// Dense multi-view stereo: the GPU replacement of COLMAP's patch_match_stereo and stereo_fusion in the custom-object
// workflow.  The protocol is stated in nero_b200/mvs.py, the ABI in include/nero_mvs.h.
//
//   grey        one thread per output pixel: integer luma sum over its s x s block, one division.
//   ref stats   one thread per pixel: mean and variance of its reference window (they do not depend on the hypothesis).
//   init        one thread per pixel: a random plane and its cost.
//   pass        the hot loop.  One thread per pixel of one colour of the checkerboard (consecutive threads take consecutive
//               pixels of that colour in a row); up to 11 hypotheses x S sources x (2r/step + 1)^2 software-bilinear
//               samples through the plane-induced homography.  The source table sits in shared memory.
//   filter      one thread per pixel, fp64: forward-backward reprojection into each source.
//
// No atomics, no reductions across threads and no transcendental functions: every output is a fixed sequence of
// correctly rounded operations on its inputs, which oracle/nero_oracle_mvs.py repeats bit for bit.
#include <cmath>

#include "common.cuh"
#include "hash.cuh"
#include "../../include/nero_mvs.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_MVS_BLOCK;
constexpr int kMaxSrc = NERO_MVS_MAX_SOURCES;
constexpr int kBest = 3;                 // the aggregate cost is the mean of the kBest smallest source costs
constexpr float kMinVar = 1e-5f;         // a window with a smaller variance has no NCC
constexpr float kNoCost = 2.0f;

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fd(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

struct Src {
  const float* img;
  int w, h;
  float A[9], b[3];
};

struct View {
  const float* grey;
  const float* stats;
  int w, h;
  float ifx, ify, ocx, ocy;
  int radius, step, S;
  float dmin, dmax;
  unsigned seed;
  int view;
};

// the random stream of one pixel at one stage: u(dim) = (mix(h ^ dim) >> 8) 2^-24
__device__ __forceinline__ uint32_t stream_key(unsigned seed, int view, int stage, int pixel) {
  uint32_t h = rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u);
  h = rl_mix(h ^ (uint32_t)view);
  h = rl_mix(h ^ (uint32_t)stage);
  return rl_mix(h ^ (uint32_t)pixel);
}

__device__ __forceinline__ float uniform(uint32_t key, int dim) {
  return fm(__uint2float_rn(rl_mix(key ^ (uint32_t)dim) >> 8), 5.9604644775390625e-8f);
}

// software bilinear at image point (X, Y): texel centres at (i + 1/2, j + 1/2), clamp to edge
__device__ __forceinline__ float bilinear(const float* __restrict__ img, int w, int h, float X, float Y) {
  X = fminf(fmaxf(X, -1.0f), (float)w + 1.0f);
  Y = fminf(fmaxf(Y, -1.0f), (float)h + 1.0f);
  const float fx = fs(X, 0.5f), fy = fs(Y, 0.5f);
  const float x0 = floorf(fx), y0 = floorf(fy);
  const float a = fs(fx, x0), b = fs(fy, y0);
  const int ix = (int)x0, iy = (int)y0;
  const int xa = clampi(ix, 0, w - 1), xb = clampi(ix + 1, 0, w - 1);
  const int ya = clampi(iy, 0, h - 1), yb = clampi(iy + 1, 0, h - 1);
  const float i00 = __ldg(img + (size_t)ya * w + xa), i01 = __ldg(img + (size_t)ya * w + xb);
  const float i10 = __ldg(img + (size_t)yb * w + xa), i11 = __ldg(img + (size_t)yb * w + xb);
  const float a1 = fs(1.0f, a);
  const float top = fa(fm(a1, i00), fm(a, i01));
  const float bot = fa(fm(a1, i10), fm(a, i11));
  return fa(fm(fs(1.0f, b), top), fm(b, bot));
}

// 1 - NCC of the reference window of pixel (x, y) against source s under the homography H (row-major), in [0, 2]
__device__ __forceinline__ float source_cost(const View& v, const Src& s, const float* H, int x, int y, float mr, float vr) {
  const float u = fa((float)x, 0.5f), w = fa((float)y, 0.5f);
  const float c2 = fa(fa(fm(H[6], u), fm(H[7], w)), H[8]);
  if (!(c2 > 0.0f)) return kNoCost;
  const float cx = fd(fa(fa(fm(H[0], u), fm(H[1], w)), H[2]), c2);
  const float cy = fd(fa(fa(fm(H[3], u), fm(H[4], w)), H[5]), c2);
  if (!(cx >= 0.0f && cx < (float)s.w && cy >= 0.0f && cy < (float)s.h)) return kNoCost;
  float sum = 0.0f, sum2 = 0.0f, cross = 0.0f;
  int n = 0;
  for (int l = -v.radius; l <= v.radius; l += v.step) {
    const float pv = fa(w, (float)l);
    const float* row = v.grey + (size_t)clampi(y + l, 0, v.h - 1) * v.w;
    for (int k = -v.radius; k <= v.radius; k += v.step) {
      const float pu = fa(u, (float)k);
      const float h2 = fa(fa(fm(H[6], pu), fm(H[7], pv)), H[8]);
      const float X = fd(fa(fa(fm(H[0], pu), fm(H[1], pv)), H[2]), h2);
      const float Y = fd(fa(fa(fm(H[3], pu), fm(H[4], pv)), H[5]), h2);
      const float val = bilinear(s.img, s.w, s.h, X, Y);
      const float ref = __ldg(row + clampi(x + k, 0, v.w - 1));
      sum = fa(sum, val);
      sum2 = fa(sum2, fm(val, val));
      cross = fa(cross, fm(ref, val));
      ++n;
    }
  }
  const float fn = (float)n;
  const float ms = fd(sum, fn);
  const float vs = fs(fd(sum2, fn), fm(ms, ms));
  if (!(vs >= kMinVar)) return kNoCost;
  const float cov = fs(fd(cross, fn), fm(mr, ms));
  const float c = fs(1.0f, fd(cov, __fsqrt_rn(fm(vr, vs))));
  return fminf(fmaxf(c, 0.0f), kNoCost);
}

// aggregate cost of the plane (d, n) at pixel (x, y) with centre ray (rx, ry, 1)
__device__ float plane_cost(const View& v, const Src* __restrict__ src, int x, int y, float rx, float ry, float mr, float vr,
                            float d, float n0, float n1, float n2) {
  if (!(vr >= kMinVar)) return kNoCost;
  const float q = fm(d, fa(fa(fm(n0, rx), fm(n1, ry)), n2));
  const float m0 = fd(fm(n0, v.ifx), q);
  const float m1 = fd(fm(n1, v.ify), q);
  const float m2 = fd(fa(fa(fm(n0, v.ocx), fm(n1, v.ocy)), n2), q);
  float b0 = kNoCost, b1 = kNoCost, b2 = kNoCost;     // the kBest smallest source costs, ascending
  for (int j = 0; j < v.S; ++j) {
    const Src& s = src[j];
    float H[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      H[3 * r + 0] = fa(s.A[3 * r + 0], fm(s.b[r], m0));
      H[3 * r + 1] = fa(s.A[3 * r + 1], fm(s.b[r], m1));
      H[3 * r + 2] = fa(s.A[3 * r + 2], fm(s.b[r], m2));
    }
    const float c = source_cost(v, s, H, x, y, mr, vr);
    if (c < b0) { b2 = b1; b1 = b0; b0 = c; }
    else if (c < b1) { b2 = b1; b1 = c; }
    else if (c < b2) { b2 = c; }
  }
  if (v.S >= kBest) return fd(fa(fa(b0, b1), b2), 3.0f);
  return fd(fa(b0, b1), 2.0f);       // S == 2
}

// a fresh random hypothesis: inverse depth uniform in [1/dmax, 1/dmin), normal = normalised uniform [-1, 1]^3 facing the
// camera (negative dot with the ray); the dims are dim0 (depth) and dim0 + 1 .. dim0 + 3 (normal)
__device__ __forceinline__ void random_plane(const View& v, uint32_t key, int dim0, float rx, float ry, float* p) {
  const float lo = fd(1.0f, v.dmax), hi = fd(1.0f, v.dmin);
  p[0] = fd(1.0f, fa(lo, fm(uniform(key, dim0), fs(hi, lo))));
  float a = fs(fm(2.0f, uniform(key, dim0 + 1)), 1.0f);
  float b = fs(fm(2.0f, uniform(key, dim0 + 2)), 1.0f);
  float c = fs(fm(2.0f, uniform(key, dim0 + 3)), 1.0f);
  const float nn = fa(fa(fm(a, a), fm(b, b)), fm(c, c));
  if (!(nn > 0.0f)) { a = 0.0f; b = 0.0f; c = -1.0f; }
  else {
    const float l = __fsqrt_rn(nn);
    a = fd(a, l); b = fd(b, l); c = fd(c, l);
  }
  const float den = fa(fa(fm(a, rx), fm(b, ry)), c);
  if (den > 0.0f) { a = -a; b = -b; c = -c; }
  else if (!(den < 0.0f)) { a = 0.0f; b = 0.0f; c = -1.0f; }
  p[1] = a; p[2] = b; p[3] = c;
}

__device__ __forceinline__ void load_sources(const long long* src_img, const int* src_wh, const float* src_geo, int S, Src* s_src) {
  for (int j = threadIdx.x; j < S; j += blockDim.x) {
    s_src[j].img = (const float*)src_img[j];
    s_src[j].w = src_wh[2 * j];
    s_src[j].h = src_wh[2 * j + 1];
    for (int a = 0; a < 9; ++a) s_src[j].A[a] = src_geo[NERO_MVS_GEO * j + a];
    for (int a = 0; a < 3; ++a) s_src[j].b[a] = src_geo[NERO_MVS_GEO * j + 9 + a];
  }
  __syncthreads();
}

__device__ __forceinline__ float ray_x(const View& v, int x) { return fa(fm(fa((float)x, 0.5f), v.ifx), v.ocx); }
__device__ __forceinline__ float ray_y(const View& v, int y) { return fa(fm(fa((float)y, 0.5f), v.ify), v.ocy); }

// ------------------------------------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(kBlock) grey_kernel(const unsigned char* __restrict__ rgb, int w, int h, int s, int wo, int ho,
                                                      float* __restrict__ grey) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)wo * ho) return;
  const int xo = int(i % wo), yo = int(i / wo);
  int acc = 0;
  for (int dy = 0; dy < s; ++dy) {
    const unsigned char* row = rgb + ((size_t)(yo * s + dy) * w + (size_t)xo * s) * 3;
    for (int dx = 0; dx < s; ++dx) acc += 299 * row[3 * dx] + 587 * row[3 * dx + 1] + 114 * row[3 * dx + 2];
  }
  grey[i] = fd((float)acc, (float)(255000 * s * s));
}

__global__ void __launch_bounds__(kBlock) ref_stats_kernel(const float* __restrict__ grey, int w, int h, int radius, int step,
                                                           float* __restrict__ stats) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)w * h) return;
  const int x = int(i % w), y = int(i / w);
  float sum = 0.0f, sum2 = 0.0f;
  int n = 0;
  for (int l = -radius; l <= radius; l += step) {
    const float* row = grey + (size_t)clampi(y + l, 0, h - 1) * w;
    for (int k = -radius; k <= radius; k += step) {
      const float r = row[clampi(x + k, 0, w - 1)];
      sum = fa(sum, r);
      sum2 = fa(sum2, fm(r, r));
      ++n;
    }
  }
  const float fn = (float)n;
  const float m = fd(sum, fn);
  stats[2 * i] = m;
  stats[2 * i + 1] = fs(fd(sum2, fn), fm(m, m));
}

__global__ void __launch_bounds__(kBlock) init_kernel(const View v, const long long* __restrict__ src_img, const int* __restrict__ src_wh,
                                                      const float* __restrict__ src_geo, float4* __restrict__ planes,
                                                      float* __restrict__ cost) {
  __shared__ Src s_src[kMaxSrc];
  load_sources(src_img, src_wh, src_geo, v.S, s_src);
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)v.w * v.h) return;
  const int x = int(i % v.w), y = int(i / v.w);
  const float rx = ray_x(v, x), ry = ray_y(v, y);
  float p[4];
  random_plane(v, stream_key(v.seed, v.view, 0, int(i)), 0, rx, ry, p);
  const float2 st = reinterpret_cast<const float2*>(v.stats)[i];
  planes[i] = make_float4(p[0], p[1], p[2], p[3]);
  cost[i] = plane_cost(v, s_src, x, y, rx, ry, st.x, st.y, p[0], p[1], p[2], p[3]);
}

__global__ void __launch_bounds__(kBlock) pass_kernel(const View v, const long long* __restrict__ src_img, const int* __restrict__ src_wh,
                                                      const float* __restrict__ src_geo, int iteration, int colour,
                                                      float4* __restrict__ planes, float* __restrict__ cost) {
  __shared__ Src s_src[kMaxSrc];
  load_sources(src_img, src_wh, src_geo, v.S, s_src);
  const int half = (v.w + 1) >> 1;
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= (long long)half * v.h) return;
  const int y = int(t / half);
  const int x = 2 * int(t % half) + ((y + colour) & 1);
  if (x >= v.w) return;
  const long long i = (long long)y * v.w + x;
  const float rx = ray_x(v, x), ry = ray_y(v, y);
  const float2 st = reinterpret_cast<const float2*>(v.stats)[i];
  float4 best = planes[i];
  float best_c = cost[i];
  // the neighbours' planes, re-intersected with this pixel's ray
  // order: (-1, 0), (1, 0), (0, -1), (0, 1), then the same at distance 5
#pragma unroll 1
  for (int k = 0; k < 8; ++k) {
    const int dist = k < 4 ? 1 : 5, sgn = (k & 1) ? dist : -dist;
    const int xn = (k & 2) ? x : x + sgn, yn = (k & 2) ? y + sgn : y;
    if (xn < 0 || xn >= v.w || yn < 0 || yn >= v.h) continue;
    const float4 pn = planes[(size_t)yn * v.w + xn];
    const float qn = fm(pn.x, fa(fa(fm(pn.y, ray_x(v, xn)), fm(pn.z, ray_y(v, yn))), pn.w));
    const float den = fa(fa(fm(pn.y, rx), fm(pn.z, ry)), pn.w);
    if (!(den < 0.0f)) continue;
    const float d = fd(qn, den);
    if (!(d >= v.dmin && d <= v.dmax)) continue;
    const float c = plane_cost(v, s_src, x, y, rx, ry, st.x, st.y, d, pn.y, pn.z, pn.w);
    if (c < best_c) { best_c = c; best = make_float4(d, pn.y, pn.z, pn.w); }
  }
  const uint32_t key = stream_key(v.seed, v.view, 1 + 2 * iteration + colour, int(i));
  const float cur[4] = {planes[i].x, planes[i].y, planes[i].z, planes[i].w};
  // perturbation of the depth: inverse depth +- 2^-(iteration + 2) of the inverse-depth range
  {
    const float lo = fd(1.0f, v.dmax), hi = fd(1.0f, v.dmin);
    const float scale = __int_as_float((125 - iteration) << 23);
    const float id = fa(fd(1.0f, cur[0]), fm(fs(fm(2.0f, uniform(key, 0)), 1.0f), fm(fs(hi, lo), scale)));
    const float d = fd(1.0f, id);
    if (d >= v.dmin && d <= v.dmax) {
      const float c = plane_cost(v, s_src, x, y, rx, ry, st.x, st.y, d, cur[1], cur[2], cur[3]);
      if (c < best_c) { best_c = c; best = make_float4(d, cur[1], cur[2], cur[3]); }
    }
  }
  // perturbation of the normal: each component +- 2^-(iteration + 1), renormalised, kept if it faces the camera
  {
    const float scale = __int_as_float((126 - iteration) << 23);
    float a = fa(cur[1], fm(fs(fm(2.0f, uniform(key, 1)), 1.0f), scale));
    float b = fa(cur[2], fm(fs(fm(2.0f, uniform(key, 2)), 1.0f), scale));
    float c = fa(cur[3], fm(fs(fm(2.0f, uniform(key, 3)), 1.0f), scale));
    const float nn = fa(fa(fm(a, a), fm(b, b)), fm(c, c));
    if (nn > 0.0f) {
      const float l = __fsqrt_rn(nn);
      a = fd(a, l); b = fd(b, l); c = fd(c, l);
      if (fa(fa(fm(a, rx), fm(b, ry)), c) < 0.0f) {
        const float cc = plane_cost(v, s_src, x, y, rx, ry, st.x, st.y, cur[0], a, b, c);
        if (cc < best_c) { best_c = cc; best = make_float4(cur[0], a, b, c); }
      }
    }
  }
  // a fresh random hypothesis
  {
    float p[4];
    random_plane(v, key, 4, rx, ry, p);
    const float c = plane_cost(v, s_src, x, y, rx, ry, st.x, st.y, p[0], p[1], p[2], p[3]);
    if (c < best_c) { best_c = c; best = make_float4(p[0], p[1], p[2], p[3]); }
  }
  planes[i] = best;
  cost[i] = best_c;
}

struct FilterView {
  int w, h;
  double fx, fy, cx, cy;
  double max_cost, reproj2, rel_depth, cos_max;
  int min_consistent, S;
};

// y = R x + t (R row-major 3x3 at g, t at g + 9), uncontracted, sums left to right
__device__ __forceinline__ void rigid(const double* g, const double* x, double* y) {
#pragma unroll
  for (int r = 0; r < 3; ++r) y[r] = da(da(da(dm(g[3 * r], x[0]), dm(g[3 * r + 1], x[1])), dm(g[3 * r + 2], x[2])), g[9 + r]);
}

__device__ __forceinline__ void rotate(const double* g, const double* x, double* y) {
#pragma unroll
  for (int r = 0; r < 3; ++r) y[r] = da(da(dm(g[3 * r], x[0]), dm(g[3 * r + 1], x[1])), dm(g[3 * r + 2], x[2]));
}

__global__ void __launch_bounds__(kBlock) filter_kernel(const FilterView v, const float4* __restrict__ planes, const float* __restrict__ cost,
                                                        const long long* __restrict__ src_planes, const long long* __restrict__ src_cost,
                                                        const int* __restrict__ src_wh, const double* __restrict__ geo,
                                                        float* __restrict__ depth, int* __restrict__ count) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)v.w * v.h) return;
  const int x = int(i % v.w), y = int(i / v.w);
  int agree = 0;
  const float4 p = planes[i];
  if ((double)cost[i] <= v.max_cost) {
    const double d = p.x, n[3] = {p.y, p.z, p.w};
    const double u = (double)x + 0.5, w = (double)y + 0.5;
    const double X[3] = {dm(d, dd(ds(u, v.cx), v.fx)), dm(d, dd(ds(w, v.cy), v.fy)), d};
    for (int j = 0; j < v.S; ++j) {
      const double* g = geo + NERO_MVS_FGEO * j;
      double Y[3];
      rigid(g, X, Y);
      if (!(Y[2] > 0.0)) continue;
      const double pu = da(dm(g[24], dd(Y[0], Y[2])), g[26]);
      const double pv = da(dm(g[25], dd(Y[1], Y[2])), g[27]);
      const int wj = src_wh[2 * j], hj = src_wh[2 * j + 1];
      if (!(pu >= 0.0 && pu < (double)wj && pv >= 0.0 && pv < (double)hj)) continue;
      const int px = (int)floor(pu), py = (int)floor(pv);
      const size_t k = (size_t)py * wj + px;
      if (!((double)((const float*)src_cost[j])[k] <= v.max_cost)) continue;
      const float4 q = ((const float4*)src_planes[j])[k];
      const double dj = q.x, nj[3] = {q.y, q.z, q.w};
      const double Z[3] = {dm(dj, dd(ds((double)px + 0.5, g[26]), g[24])), dm(dj, dd(ds((double)py + 0.5, g[27]), g[25])), dj};
      double W[3], m[3];
      rigid(g + 12, Z, W);
      if (!(W[2] > 0.0)) continue;
      const double eu = ds(da(dm(v.fx, dd(W[0], W[2])), v.cx), u);
      const double ev = ds(da(dm(v.fy, dd(W[1], W[2])), v.cy), w);
      rotate(g + 12, nj, m);
      const double cosv = da(da(dm(n[0], m[0]), dm(n[1], m[1])), dm(n[2], m[2]));
      if (da(dm(eu, eu), dm(ev, ev)) <= v.reproj2 && fabs(ds(W[2], d)) <= dm(v.rel_depth, d) && cosv >= v.cos_max) ++agree;
    }
  }
  count[i] = agree;
  depth[i] = agree >= v.min_consistent ? p.x : 0.0f;
}

inline unsigned nblocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

bool view_ok(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats, const long long* src_img,
             const int* src_wh, const float* src_geo, int S, int radius, int step, float dmin, float dmax, const float* planes, const float* cost) {
  return grey && stats && src_img && src_wh && src_geo && planes && cost && w >= 1 && h >= 1 && (long long)w * h <= 0x7fffffffLL &&
         S >= 2 && S <= kMaxSrc && radius >= 0 && step >= 1 && radius <= 64 && std::isfinite(ifx) && std::isfinite(ify) &&
         std::isfinite(ocx) && std::isfinite(ocy) && dmin > 0.0f && dmax >= dmin && std::isfinite(dmax);
}

View make_view(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats, int S, int radius,
               int step, float dmin, float dmax, unsigned seed, int view) {
  View v;
  v.grey = grey; v.stats = stats; v.w = w; v.h = h;
  v.ifx = ifx; v.ify = ify; v.ocx = ocx; v.ocy = ocy;
  v.radius = radius; v.step = step; v.S = S;
  v.dmin = dmin; v.dmax = dmax; v.seed = seed; v.view = view;
  return v;
}

}  // namespace

extern "C" {

int nero_mvs_grey(const unsigned char* rgb, int w, int h, int s, float* grey, void* stream) {
  if (!rgb || !grey || w < 1 || h < 1 || s < 1 || s > 91 || w / s < 1 || h / s < 1) return NERO_ERR_ARG;
  const int wo = w / s, ho = h / s;
  grey_kernel<<<nblocks((long long)wo * ho), kBlock, 0, (cudaStream_t)stream>>>(rgb, w, h, s, wo, ho, grey);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mvs_ref_stats(const float* grey, int w, int h, int radius, int step, float* stats, void* stream) {
  if (!grey || !stats || w < 1 || h < 1 || radius < 0 || radius > 64 || step < 1) return NERO_ERR_ARG;
  ref_stats_kernel<<<nblocks((long long)w * h), kBlock, 0, (cudaStream_t)stream>>>(grey, w, h, radius, step, stats);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mvs_init(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats,
                  const long long* src_img, const int* src_wh, const float* src_geo, int S, int radius, int step, float dmin,
                  float dmax, unsigned int seed, int view, float* planes, float* cost, void* stream) {
  if (!view_ok(grey, w, h, ifx, ify, ocx, ocy, stats, src_img, src_wh, src_geo, S, radius, step, dmin, dmax, planes, cost))
    return NERO_ERR_ARG;
  const View v = make_view(grey, w, h, ifx, ify, ocx, ocy, stats, S, radius, step, dmin, dmax, seed, view);
  init_kernel<<<nblocks((long long)w * h), kBlock, 0, (cudaStream_t)stream>>>(v, src_img, src_wh, src_geo, (float4*)planes, cost);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mvs_pass(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats,
                  const long long* src_img, const int* src_wh, const float* src_geo, int S, int radius, int step, float dmin,
                  float dmax, unsigned int seed, int view, int iteration, int colour, float* planes, float* cost, void* stream) {
  if (!view_ok(grey, w, h, ifx, ify, ocx, ocy, stats, src_img, src_wh, src_geo, S, radius, step, dmin, dmax, planes, cost) ||
      iteration < 0 || iteration > 100 || (colour != 0 && colour != 1))
    return NERO_ERR_ARG;
  const View v = make_view(grey, w, h, ifx, ify, ocx, ocy, stats, S, radius, step, dmin, dmax, seed, view);
  pass_kernel<<<nblocks((long long)((w + 1) / 2) * h), kBlock, 0, (cudaStream_t)stream>>>(v, src_img, src_wh, src_geo, iteration, colour,
                                                                                        (float4*)planes, cost);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mvs_filter(int w, int h, double fx, double fy, double cx, double cy, const float* planes, const float* cost,
                    const long long* src_planes, const long long* src_cost, const int* src_wh, const double* geo, int S,
                    double max_cost, double reproj2, double rel_depth, double cos_max, int min_consistent, float* depth,
                    int* count, void* stream) {
  if (!planes || !cost || !depth || !count || w < 1 || h < 1 || (long long)w * h > 0x7fffffffLL || S < 0 || S > kMaxSrc ||
      (S > 0 && (!src_planes || !src_cost || !src_wh || !geo)) || !(fx != 0.0) || !(fy != 0.0) || !std::isfinite(cx) ||
      !std::isfinite(cy) || !(reproj2 >= 0.0) || !(rel_depth >= 0.0) || !std::isfinite(cos_max) || min_consistent < 0)
    return NERO_ERR_ARG;
  FilterView v;
  v.w = w; v.h = h; v.fx = fx; v.fy = fy; v.cx = cx; v.cy = cy;
  v.max_cost = max_cost; v.reproj2 = reproj2; v.rel_depth = rel_depth; v.cos_max = cos_max;
  v.min_consistent = min_consistent; v.S = S;
  filter_kernel<<<nblocks((long long)w * h), kBlock, 0, (cudaStream_t)stream>>>(v, (const float4*)planes, cost, src_planes, src_cost,
                                                                               src_wh, geo, depth, count);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
