// Point-to-mesh distance: one thread per query, a closest-point search over the BVH of k_bvh.cu (32-byte nodes in
// depth-first order, left child = index + 1), nearer child first.  The convention -- the triangle routine, the degenerate
// rule, the tie rule and the conservative box bound -- is stated in include/nero_meshdist.h; oracle/nero_oracle_meshdist.py
// repeats the routine in numpy over every triangle, bit for bit.
//
// Per visited inner node: both children's boxes (four float4 loads) and their directed-rounding lower bounds; per leaf
// triangle: tri_ids -> tris -> verts (one int, three ints, nine floats) and the fp64 routine.  No atomics except the
// status flag of a stack overrun; every output is a fixed sequence of correctly rounded operations of its own inputs.
#include <cfloat>
#include <climits>
#include <cmath>
#include <math_constants.h>

#include "common.cuh"
#include "../../include/nero_meshdist.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_MESHDIST_BLOCK;
constexpr int kStack = NERO_MESHDIST_STACK;
constexpr double kRho = 0x1p-40;   // relative margin of the box bound
constexpr double kAbs = 0x1p-40;   // absolute margin, times the root box's largest |coordinate|

struct D3 { double x, y, z; };

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double dd(double a, double b) { return __ddiv_rn(a, b); }

__device__ __forceinline__ D3 sub(const D3& a, const D3& b) { return {ds(a.x, b.x), ds(a.y, b.y), ds(a.z, b.z)}; }
__device__ __forceinline__ double dot(const D3& a, const D3& b) { return da(da(dm(a.x, b.x), dm(a.y, b.y)), dm(a.z, b.z)); }
__device__ __forceinline__ D3 lerp(const D3& x, double t, const D3& e) { return {da(x.x, dm(t, e.x)), da(x.y, dm(t, e.y)), da(x.z, dm(t, e.z))}; }

__device__ __forceinline__ D3 vert(const float* __restrict__ verts, int i) {
  return {(double)__ldg(verts + 3 * i), (double)__ldg(verts + 3 * i + 1), (double)__ldg(verts + 3 * i + 2)};
}

// the closest point of segment x + [0, 1] e to p, xp = p - x
__device__ __forceinline__ D3 seg_point(const D3& x, const D3& y, const D3& e, const D3& xp) {
  const double m = dot(xp, e), l = dot(e, e);
  if (m <= 0.0) return x;
  if (m >= l) return y;
  return lerp(x, dd(m, l), e);
}

__device__ __forceinline__ double dist2(const D3& p, const D3& q) {
  const D3 d = sub(p, q);
  return dot(d, d);
}

__device__ D3 segments(const D3& p, const D3& a, const D3& b, const D3& c, const D3& ab, const D3& ac, const D3& bc, const D3& ap,
                       const D3& bp) {
  D3 q = seg_point(a, b, ab, ap);
  double best = dist2(p, q);
  const D3 q1 = seg_point(a, c, ac, ap);
  const double d1 = dist2(p, q1);
  if (d1 < best) { best = d1; q = q1; }
  const D3 q2 = seg_point(b, c, bc, bp);
  if (dist2(p, q2) < best) q = q2;
  return q;
}

// Ericson 5.1.5 with the degenerate rule of include/nero_meshdist.h
__device__ D3 closest_on_triangle(const D3& p, const D3& a, const D3& b, const D3& c) {
  const D3 ab = sub(b, a), ac = sub(c, a), ap = sub(p, a), bp = sub(p, b), cp = sub(p, c), bc = sub(c, b);
  const double nx = ds(dm(ab.y, ac.z), dm(ab.z, ac.y)), ny = ds(dm(ab.z, ac.x), dm(ab.x, ac.z)),
               nz = ds(dm(ab.x, ac.y), dm(ab.y, ac.x));
  if (nx == 0.0 && ny == 0.0 && nz == 0.0) return segments(p, a, b, c, ab, ac, bc, ap, bp);
  const double d1 = dot(ab, ap), d2 = dot(ac, ap);
  if (d1 <= 0.0 && d2 <= 0.0) return a;
  const double d3 = dot(ab, bp), d4 = dot(ac, bp);
  if (d3 >= 0.0 && d4 <= d3) return b;
  const double vc = ds(dm(d1, d4), dm(d3, d2));
  if (vc <= 0.0 && d1 >= 0.0 && d3 <= 0.0) {
    const double den = ds(d1, d3);
    return den > 0.0 ? lerp(a, dd(d1, den), ab) : segments(p, a, b, c, ab, ac, bc, ap, bp);
  }
  const double d5 = dot(ab, cp), d6 = dot(ac, cp);
  if (d6 >= 0.0 && d5 <= d6) return c;
  const double vb = ds(dm(d5, d2), dm(d1, d6));
  if (vb <= 0.0 && d2 >= 0.0 && d6 <= 0.0) {
    const double den = ds(d2, d6);
    return den > 0.0 ? lerp(a, dd(d2, den), ac) : segments(p, a, b, c, ab, ac, bc, ap, bp);
  }
  const double va = ds(dm(d3, d6), dm(d5, d4));
  const double e = ds(d4, d3), f = ds(d5, d6);
  if (va <= 0.0 && e >= 0.0 && f >= 0.0) {
    const double den = da(e, f);
    return den > 0.0 ? lerp(b, dd(e, den), bc) : segments(p, a, b, c, ab, ac, bc, ap, bp);
  }
  const double s = da(da(va, vb), vc);
  if (va >= 0.0 && vb >= 0.0 && vc >= 0.0 && s > 0.0) {
    const double v = dd(vb, s), w = dd(vc, s);
    return lerp(lerp(a, v, ab), w, ac);
  }
  return segments(p, a, b, c, ab, ac, bc, ap, bp);
}

__device__ __forceinline__ D3 triangle_closest(const D3& p, const int* __restrict__ tris, const float* __restrict__ verts, int id) {
  const int i0 = __ldg(tris + 3 * id), i1 = __ldg(tris + 3 * id + 1), i2 = __ldg(tris + 3 * id + 2);
  return closest_on_triangle(p, vert(verts, i0), vert(verts, i1), vert(verts, i2));
}

// lower bound of the squared distance from p to the box [lo, hi] (float32 corners, exact in float64)
__device__ __forceinline__ double box_d2(const D3& p, const float4& lo, const float4& hi) {
  const double gx = fmax(fmax(__dsub_rd((double)lo.x, p.x), __dsub_rd(p.x, (double)hi.x)), 0.0);
  const double gy = fmax(fmax(__dsub_rd((double)lo.y, p.y), __dsub_rd(p.y, (double)hi.y)), 0.0);
  const double gz = fmax(fmax(__dsub_rd((double)lo.z, p.z), __dsub_rd(p.z, (double)hi.z)), 0.0);
  return __dadd_rd(__dadd_rd(__dmul_rd(gx, gx), __dmul_rd(gy, gy)), __dmul_rd(gz, gz));
}

// R2 of include/nero_meshdist.h: a node whose box bound exceeds it holds no triangle with computed d2 <= best
__device__ __forceinline__ double visit_bound(double best, double max_dist, double margin) {
  const double r = __dadd_ru(__dmul_ru(fmin(max_dist, __dsqrt_ru(best)), 1.0 + kRho), margin);
  return __dmul_ru(r, r);
}

__global__ void __launch_bounds__(kBlock) meshdist_kernel(const double* __restrict__ points, long long n, const float4* __restrict__ n4,
                                                          const int* __restrict__ tri_ids, const float* __restrict__ verts,
                                                          const int* __restrict__ tris, double max_dist, double* __restrict__ dist,
                                                          int* __restrict__ tri, double* __restrict__ closest, int* __restrict__ status) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const D3 p{points[3 * i], points[3 * i + 1], points[3 * i + 2]};
  const float4 root_lo = __ldg(n4), root_hi = __ldg(n4 + 1);
  const double m = fmax(fmax(fmax(fabs((double)root_lo.x), fabs((double)root_hi.x)), fmax(fabs((double)root_lo.y), fabs((double)root_hi.y))),
                        fmax(fabs((double)root_lo.z), fabs((double)root_hi.z)));
  const double margin = m * kAbs;
  double best = CUDART_INF;
  int best_id = INT_MAX;
  double bound = visit_bound(best, max_dist, margin);
  int stack_node[kStack];
  float stack_d2[kStack];
  int sp = 0;
  int node = box_d2(p, root_lo, root_hi) <= bound ? 0 : -1;
  while (node >= 0) {
    const float4 a = __ldg(n4 + 2 * node), b = __ldg(n4 + 2 * node + 1);
    const int cnt = __float_as_int(b.w), first_or_right = __float_as_int(a.w);
    if (cnt > 0) {
      node = -1;
      for (int k = 0; k < cnt; ++k) {
        const int id = __ldg(tri_ids + first_or_right + k);
        const double d2 = dist2(p, triangle_closest(p, tris, verts, id));
        if (d2 < best || (d2 == best && id < best_id)) {
          best = d2;
          best_id = id;
          bound = visit_bound(best, max_dist, margin);
        }
      }
    } else {
      int near = node + 1, far = first_or_right;
      double dn = box_d2(p, __ldg(n4 + 2 * near), __ldg(n4 + 2 * near + 1));
      double df = box_d2(p, __ldg(n4 + 2 * far), __ldg(n4 + 2 * far + 1));
      if (df < dn) {
        const int t = near; near = far; far = t;
        const double u = dn; dn = df; df = u;
      }
      if (df <= bound) {
        if (sp == kStack) {   // unreachable for T < 2^31 (see the header); never a silent wrong answer
          atomicOr(status, 1);
          best_id = -2;
          break;
        }
        stack_node[sp] = far;
        stack_d2[sp] = __double2float_rd(df);
        ++sp;
      }
      node = dn <= bound ? near : -1;
    }
    while (node < 0 && sp > 0) {
      --sp;
      if ((double)stack_d2[sp] <= bound) node = stack_node[sp];
    }
  }
  if (best_id == -2) {
    dist[i] = CUDART_NAN;
    tri[i] = -2;
    if (closest) closest[3 * i] = closest[3 * i + 1] = closest[3 * i + 2] = CUDART_NAN;
    return;
  }
  const double d = __dsqrt_rn(best);
  if (best_id == INT_MAX || d > max_dist) {
    dist[i] = CUDART_INF;
    tri[i] = -1;
    if (closest) closest[3 * i] = closest[3 * i + 1] = closest[3 * i + 2] = CUDART_NAN;
    return;
  }
  dist[i] = d;
  tri[i] = best_id;
  if (closest) {
    const D3 q = triangle_closest(p, tris, verts, best_id);
    closest[3 * i] = q.x;
    closest[3 * i + 1] = q.y;
    closest[3 * i + 2] = q.z;
  }
}

inline bool bad_max_dist(double v) { return !(v >= 0.0); }   // NaN or negative; +inf is allowed

}  // namespace

extern "C" int nero_meshdist_query(const double* points, long long n, const float* nodes, const int* tri_ids, const float* verts,
                                   const int* tris, double max_dist, double* dist, int* tri, double* closest, int* status,
                                   void* stream) {
  if (n < 0 || bad_max_dist(max_dist)) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!points || !nodes || !tri_ids || !verts || !tris || !dist || !tri || !status) return NERO_ERR_ARG;
  meshdist_kernel<<<unsigned((n + kBlock - 1) / kBlock), kBlock, 0, (cudaStream_t)stream>>>(
      points, n, reinterpret_cast<const float4*>(nodes), tri_ids, verts, tris, max_dist, dist, tri, closest, status);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero

