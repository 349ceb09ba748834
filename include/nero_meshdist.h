/* libnero_b200 -- C ABI of the point-to-mesh distance: for each query point the closest point of a triangle mesh, found by
 * a closest-point search over the mesh's BVH (nero_b200/meshdist.py sequences it; oracle/nero_oracle_meshdist.py restates it
 * in numpy by brute force over every triangle).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 *
 * Inputs.  Queries p are float64 [n,3].  The mesh is verts [V,3] float32 and tris [T,3] int32; each vertex is converted
 * exactly to float64.  The distance is computed from these original vertices, read through tri_ids -> tris -> verts, never
 * from the BVH's (v0, e1, e2) triples (v0 + e1 is not v1 in float32).
 *
 * Distance to one triangle (a, b, c).  Every float64 operation below is one correctly rounded __dadd_rn / __dsub_rn /
 * __dmul_rn / __ddiv_rn / __dsqrt_rn, never contracted into an FMA, so numpy reproduces every bit.  Vectors are taken
 * component by component, dot(u, v) = (u.x v.x + u.y v.y) + u.z v.z, cross(u, v) = (u.y v.z - u.z v.y, u.z v.x - u.x v.z,
 * u.x v.y - u.y v.x).
 *   ab = b - a, ac = c - a, ap = p - a, bp = p - b, cp = p - c, bc = c - b.
 *   If cross(ab, ac) == (0, 0, 0): the triangle is its three edge segments (below).
 *   Otherwise the Voronoi regions of Ericson, Real-Time Collision Detection, 5.1.5, tested in this order:
 *     d1 = dot(ab, ap), d2 = dot(ac, ap)            d1 <= 0 and d2 <= 0                      -> q = a
 *     d3 = dot(ab, bp), d4 = dot(ac, bp)            d3 >= 0 and d4 <= d3                     -> q = b
 *     vc = d1 d4 - d3 d2                            vc <= 0 and d1 >= 0 and d3 <= 0          -> edge ab, t = d1 / (d1 - d3)
 *     d5 = dot(ab, cp), d6 = dot(ac, cp)            d6 >= 0 and d5 <= d6                     -> q = c
 *     vb = d5 d2 - d1 d6                            vb <= 0 and d2 >= 0 and d6 <= 0          -> edge ac, t = d2 / (d2 - d6)
 *     va = d3 d6 - d5 d4, e = d4 - d3, f = d5 - d6  va <= 0 and e >= 0 and f >= 0            -> edge bc, t = e / (e + f)
 *     s = (va + vb) + vc                            va >= 0, vb >= 0, vc >= 0 and s > 0      -> face
 *     anything else                                                                           -> the three edge segments
 *   Edge xy: q = x + t (y - x) (t multiplies each component of the stored difference ab, ac or bc); a zero denominator
 *   (only possible when both its terms are 0) selects the three edge segments instead.  Face: v = vb / s, w = vc / s (two
 *   divisions, not one reciprocal: each lies in [0, 1] and none overflows), q = (a + ab v) + ac w.
 *   Edge segments (the degenerate rule: zero-length edges, collinear and repeated vertices, and the rare rounded cases
 *   whose region denominators vanish): for (x, y, e, xp) in (a, b, ab, ap), (a, c, ac, ap), (b, c, bc, bp): m = dot(xp, e),
 *   l = dot(e, e); q = x if m <= 0, y if m >= l, else x + (m / l) e; the first segment of least d2 wins.
 *   Then dx = p - q and d2 = dot(dx, dx).  Every division has a positive denominator no smaller than its numerator, so
 *   finite inputs never give NaN.
 *
 * Result per query.  d2 = the minimum over triangles; tri = the ORIGINAL index of the minimising triangle, ties to the lowest
 * index, so the result depends neither on the BVH nor on the traversal order; dist = __dsqrt_rn(d2); closest = that
 * triangle's q.  max_dist: if dist > max_dist (or there is no triangle within it), dist = +inf, tri = -1 and closest = NaN.
 *
 * Pruning (why the result is the brute-force minimum bit for bit).  A node is skipped only if no triangle under it can give
 * a computed d2 <= the current best.  The bound on the node box is a lower bound on the true squared distance, taken with
 * directed rounding: per axis g = max(lo - p, p - hi, 0) with __dsub_rd, d2_box = (g0 g0 + g1 g1) + g2 g2 with __dmul_rd /
 * __dadd_rd.  The routine's computed q lies within 21 u M of the triangle (u = 2^-53, M = the largest |coordinate| of the
 * root box), hence of every box holding the triangle, and its computed d2 is at least (1 - 5u) |p - q|^2.  With the margins
 * rho = 2^-40 (relative) and E = 2^-40 M (absolute), r = min(max_dist, sqrt_ru(best)) (1 + rho) + E and R2 = r r, both
 * rounded up, a node is visited iff d2_box <= R2.  A stack entry keeps its d2_box rounded down to float32 and is tested
 * again against R2 when it is popped.
 *
 * Stack bound.  One entry per inner node on the path from the root.  nero_bvh_build_host splits by binned SAH above depth
 * 28 and by the median below, with leaves of at most 4 triangles, so a path has at most 28 + ceil(log2(T / 4)) <= 57 inner
 * nodes for T < 2^31.  The kernel keeps 64 entries (NERO_MESHDIST_STACK); should a push ever find the stack full, the
 * query stops with tri = -2, dist = NaN and *status |= 1, so an overrun is never a silent wrong answer.
 */
#ifndef NERO_MESHDIST_H_
#define NERO_MESHDIST_H_

#include "nero_b200.h"

#define NERO_MESHDIST_STACK 64
#define NERO_MESHDIST_BLOCK 128

#ifdef __cplusplus
extern "C" {
#endif

/* Distances from points [n,3] float64 to the mesh (verts [V,3] float32, tris [T,3] int32) whose BVH nodes and tri_ids are
 * nero_bvh_build_host's outputs for that mesh.  Outputs dist [n] float64 and tri [n] int32 are required; closest [n,3]
 * float64 is written when it is not NULL.  status [1] int32 must hold 0 on entry (see Stack bound).  max_dist may be +inf.
 * Returns 1 for NULL required buffers (n > 0), n < 0, or max_dist < 0 or NaN. */
int nero_meshdist_query(const double* points, long long n, const float* nodes, const int* tri_ids, const float* verts,
                        const int* tris, double max_dist, double* dist, int* tri, double* closest, int* status, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_MESHDIST_H_ */
