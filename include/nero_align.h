/* libnero_b200 -- C ABI of mesh registration: the per-point kernels of a trimmed point-to-plane similarity ICP and of its
 * principal-axis start, each writing per-block partial sums, and the fixed-order reduction of those partials
 * (nero_b200/align.py sequences them around nero_meshdist_query; oracle/nero_oracle_align.py restates every kernel in numpy).
 *
 * Same library and conventions as include/nero_meshdist.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed
 * as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 * Every float64 operation below is one correctly rounded __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn, never
 * contracted into an FMA, so numpy reproduces every bit; dot(u, v) = (u.x v.x + u.y v.y) + u.z v.z and
 * cross(u, v) = (u.y v.z - u.z v.y, u.z v.x - u.x v.z, u.x v.y - u.y v.x), as in nero_meshdist.h.
 *
 * Transform.  mats [k,3,4] float64 rows (m0 | m1 | m2) of y = A x + b; for matrix j and point i, output row j n + i is
 * y_r = ((m_r0 x + m_r1 y) + m_r2 z) + m_r3.
 *
 * Terms (one row of the Gauss-Newton system per source point y).  A point with tri < 0 contributes exact zeros.  Otherwise
 * (a, b, c) = the triangle's original vertices (float32 converted exactly), ab = b - a, ac = c - a, m = cross(ab, ac); if
 * m == (0, 0, 0) the point contributes zeros except a 1 in the degenerate count.  Else l = sqrt(dot(m, m)),
 * n = (m.x / l, m.y / l, m.z / l), d = y - center, e = y - q (q = the query's closest point), r = dot(n, e) and the Jacobian
 * row J = (cross(d, n), n, dot(n, d)) of the update y' = c + (1 + sigma)(I + [w]x)(y - c) + dt in the order (w, dt, sigma).
 * The point's NERO_ALIGN_TERMS values: J_i J_j for i <= j in row-major order (28), J_i r (7), r r, 1 (rows used), 0
 * (degenerate count).
 *
 * Moments.  d = p - origin; the NERO_ALIGN_MOMENTS values 1, d.x, d.y, d.z, d.x d.x, d.x d.y, d.x d.z, d.y d.y, d.y d.z, d.z d.z.
 *
 * Score.  dist [k m] holds k segments of m distances (+inf where nero_meshdist_query found nothing within its max_dist); the
 * value of each is v v with v = min(dist, tau).  Segment j's points are its own blocks: block b of segment j covers
 * dist[j m + 256 b ...] up to the segment's end, so each segment is a whole number of blocks.
 *
 * Block partial (the terms, moments and score kernels).  Block b of 256 consecutive points writes partial[b * width + v] =
 * the pairwise tree over its 256 values of column v, points past the end (or the segment's end) counting as +0: level
 * h = 1, 2, 4, ..., 128 replaces x[i] by x[i] + x[i + h] for every i divisible by 2h, and x[0] is the sum.
 *
 * Reduce.  partial holds `segments` runs of `blocks` rows of `width` values.  Each segment is reduced by levels: its current
 * rows are cut into chunks of 256 consecutive rows, the last padded with +0, each chunk is summed column by column by the
 * same pairwise tree and its sum becomes row c of the next level, until one row is left; out[s * width + v] is that row.
 * This is the pairwise tree over the block partials padded with zeros to a power of 256 (equal, up to the sign of a zero
 * sum, to padding to a power of two).  The partials are overwritten.  No floating-point atomics anywhere: every output is a
 * fixed sequence of correctly rounded operations of the inputs.
 */
#ifndef NERO_ALIGN_H_
#define NERO_ALIGN_H_

#include "nero_b200.h"

#define NERO_ALIGN_BLOCK 256
#define NERO_ALIGN_TERMS 38
#define NERO_ALIGN_MOMENTS 10
#define NERO_ALIGN_MAX_WIDTH 64

#ifdef __cplusplus
extern "C" {
#endif

/* out [k n, 3] float64 = the k transforms mats [k,3,4] float64 applied to points [n,3] float64.  Returns 1 for n < 0, k < 1
 * or NULL buffers (n > 0). */
int nero_align_transform(const double* points, long long n, const double* mats, int k, double* out, void* stream);

/* Partials [ceil(n / 256), NERO_ALIGN_TERMS] float64 of points [n,3] with nero_meshdist_query's tri [n] and closest [n,3]
 * against the mesh verts [V,3] float32 / tris [T,3] int32, about the centre (cx, cy, cz).  Returns 1 for n < 0 or NULL
 * buffers (n > 0). */
int nero_align_terms(const double* points, long long n, const int* tri, const double* closest, const float* verts, const int* tris,
                     double cx, double cy, double cz, double* partial, void* stream);

/* Partials [ceil(n / 256), NERO_ALIGN_MOMENTS] float64 of points [n,3] about the origin (ox, oy, oz).  Returns 1 for n < 0
 * or NULL buffers (n > 0). */
int nero_align_moments(const double* points, long long n, double ox, double oy, double oz, double* partial, void* stream);

/* Partials [k ceil(m / 256)] float64 of min(dist, tau)^2 over k segments of m distances.  Returns 1 for m < 1, k < 1,
 * tau < 0 or NaN, or NULL buffers. */
int nero_align_score(const double* dist, long long m, int k, double tau, double* partial, void* stream);

/* out [segments, width] float64 = the fixed-order sums of partial [segments, blocks, width] (overwritten).  Returns 1 for
 * segments < 1, blocks < 1, width < 1 or > NERO_ALIGN_MAX_WIDTH, or NULL buffers. */
int nero_align_reduce(double* partial, int segments, long long blocks, int width, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_ALIGN_H_ */
