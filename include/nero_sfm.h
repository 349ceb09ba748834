/* libnero_b200 -- C ABI of incremental structure from motion: tracks from verified matches, P3P RANSAC, multi-view
 * triangulation, and the pieces of one Levenberg-Marquardt iteration of bundle adjustment with the Schur complement over
 * the points.
 *
 * Same library and conventions as include/nero_features.h: pointers are DEVICE pointers unless stated otherwise, `stream`
 * is a cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument
 * (checked before any launch), 2 on a CUDA launch error.  Plain arguments only.  The protocol is stated in
 * nero_b200/sfm.py and restated in numpy by oracle/nero_oracle_sfm.py.  All arithmetic is fp64 and no floating-point
 * atomics are used: every sum has a fixed order.
 *
 * Poses pose [m, 12] fp64: R row-major, then t (x_cam = R x + t).  A camera has a focal f and a principal point (cx, cy);
 * projection u = f Y_x / Y_z + cx, v = f Y_y / Y_z + cy of Y = R X + t.
 *
 * Track length.  The triangulate and filter kernels spend O(m) projections and O(m^2) ray angles on a track of m
 * observations, in one thread.  A track has at most one observation per image (nero_b200.sfm drops the others), so m is
 * at most the number of images of the reconstruction, <= NERO_SFM_MAX_IMAGES; the kernels need no other bound.
 *
 * Bundle adjustment.  Observations o are ordered by point: point p owns o = pt_off[p] .. pt_off[p + 1] - 1.  obs_img [n]
 * is the image of o (0 .. nimg - 1), img_cam [nimg] the camera of an image (0 .. ncam - 1).  The reduced system has
 * 6 nimg + ncam columns: image k's rotation update w (R <- exp(w) R) and translation update at 6 k .. 6 k + 5, camera c's
 * focal at 6 nimg + c.  Per observation the 7 camera-side columns are (w, t, f).
 */
#ifndef NERO_SFM_H_
#define NERO_SFM_H_

#define NERO_SFM_BLOCK 256          /* threads per block of the per-node, per-observation and per-point kernels */
#define NERO_SFM_MAX_HYP 8192       /* P3P hypotheses per registration */
#define NERO_SFM_MAX_IMAGES 500     /* images of one reconstruction (the reduced system is dense) */
#define NERO_SFM_CHUNK 256          /* reduced-system entries (or right-hand-side observations) summed by one block */

#ifdef __cplusplus
extern "C" {
#endif

/* Tracks of N nodes joined by E edges [E, 2] int: union-find (label [N] = the smallest node of each component), then the
 * roots compacted in node order: track [N] = the rank of the node's label among the roots; *total (DEVICE int64) = the
 * number of tracks.  blk_count [nblk] int, blk_off [nblk] int64 are scratch with nblk = ceil(N / NERO_SFM_BLOCK). */
int nero_sfm_tracks(const int* edges, int E, int N, int* label, int* blk_count, long long* blk_off, long long* total, int* track,
                    void* stream);

/* P3P RANSAC of one image: n correspondences xy [n, 2] (pixels) -> X [n, 3], camera (f, cx, cy).  Hypothesis h draws 3
 * distinct correspondences, draw d being rl_mix(rl_mix(rl_mix(rl_mix(seed 0x9e3779b9 + 0x7f4a7c15) ^ image) ^ h) ^ d) mod n
 * (at most 32 draws), and solves them by Lambda Twist (at most 4 poses); a pose's count is the correspondences in front of
 * it with squared reprojection error <= max_err2, a hypothesis keeps its first best pose.  counts [H] int (-1: no pose),
 * poses [H, 12]; the winner is the largest count, ties to the lower hypothesis: best [2] int = (hypothesis, count),
 * pose [12], inlier [n] uint8.  1 <= H <= NERO_SFM_MAX_HYP, n >= 3. */
int nero_sfm_p3p(const double* xy, const double* X, int n, double f, double cx, double cy, int image, int hypotheses,
                 unsigned int seed, double max_err2, int* counts, double* poses, int* best, double* pose, unsigned char* inlier,
                 void* stream);

/* Multi-view DLT of T tracks: track k owns observations off[k] .. off[k + 1] - 1 (m >= 2 of them, one thread reads all), each
 * with its image obs_img and pixel obs_xy [n, 2]; image i has pose [i], camera img_cam[i] with focal[c] and pp [c, 2].  The
 * 4 x 4 normal matrix of the rows x^ P3 - P1, y^ P3 - P2 (x^ = (x - cx) / f) is summed in observation order; X [T, 3] is the
 * eigenvector of its smallest diagonal entry after 10 cyclic Jacobi sweeps.  stat [T, 3] = (smallest depth, largest
 * reprojection error in px, largest pairwise ray angle in radians). */
int nero_sfm_triangulate(const long long* off, int T, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                         const double* focal, const double* pp, double* X, double* stat, void* stream);

/* Per observation of the point-ordered list: the point's depth and reprojection error err [n, 2] (px), and per point
 * angle [P] = the largest pairwise angle (radians) of the rays of its observations. */
int nero_sfm_filter(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                    const double* focal, const double* pp, const double* X, double* err, double* angle, void* stream);

/* Per observation: res [n, 2] (projection - observation), Jc [n, 2, 7] (w, t, f) and Jp [n, 2, 3]. */
int nero_sfm_ba_linearize(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose,
                          const int* img_cam, const double* focal, const double* pp, const double* X, double* res, double* Jc,
                          double* Jp, void* stream);

/* Per point: V = sum Jp^T Jp with its diagonal times (1 + lambda), Vinv [P, 9] (0 when fix_points or det V <= 0),
 * gp [P, 3] = sum Jp^T r, both summed in observation order; per observation Y [n, 7, 3] = (Jc^T Jp) Vinv. */
int nero_sfm_ba_points(const long long* pt_off, int P, const double* res, const double* Jc, const double* Jp, double lambda, int fix_points,
                       double* Vinv, double* gp, double* Y, void* stream);

/* The reduced camera system, in two fixed-order stages.  ent [M, 2] int = (o, o') pairs of observations of one point,
 * ordered by (row block, column block) and then in (point, o, o') order: block b < nimg is image b's 6 columns, block
 * nimg + c camera c's focal.  A segment is the run of one (row block, column block) key; it is cut into chunks of at most
 * NERO_SFM_CHUNK consecutive entries, chunk k being ent[chunk[k][0] .. chunk[k][1] - 1] with key chunk_key [k, 2] int, and
 * segment s owning chunks seg_chunk[s] .. seg_chunk[s + 1] - 1 with key seg_key [s, 2].  Stage 1: per chunk and entry of
 * the block pair, sum [o == o'] Jc_o^T Jc_o' (times 1 + lambda on the system's diagonal) - Y_o (Jc_o'^T Jp_o')^T in entry
 * order into partial [nchunk, 36] (slot 6 r + c).  Stage 2: per segment, thread t of 64 adds chunks t, t + 64, ... in
 * order, then a fixed tree over the threads; the sum lands in S [ncol, ncol] (ncol = 6 nimg + ncam), rows and columns of
 * fixed [ncol] (uint8) parameters become the identity.  Entries of S outside every segment are not written.  The
 * right-hand side the same way: obs_seg [Q, 2] int = (observation, block) ordered by block and then observation, chunks
 * rchunk [nrchunk, 2] of one block each (rchunk_blk [nrchunk]), segments rseg_chunk [nrseg + 1] / rseg_blk [nrseg],
 * rpartial [nrchunk, 6]; b [col] = -sum (Jc_o^T r_o - Y_o gp_p), 0 for fixed parameters.  obs_pt [n] is the point of each
 * observation.  1 <= ncam <= nimg <= NERO_SFM_MAX_IMAGES.  No segment is summed by one thread: with one shared camera the
 * focal segments hold every pair, and the chunks spread them over the GPU while the order stays fixed. */
int nero_sfm_ba_reduce(const int* ent, const long long* chunk, const int* chunk_key, int nchunk, const long long* seg_chunk, const int* seg_key,
                       int nseg, const int* obs_seg, const long long* rchunk, const int* rchunk_blk, int nrchunk, const long long* rseg_chunk,
                       const int* rseg_blk, int nrseg, const int* obs_pt, const int* img_cam, int nimg, int ncam, const double* Jc,
                       const double* Jp, const double* res, const double* Y, const double* gp, double lambda, const unsigned char* fixed,
                       double* partial, double* rpartial, double* S, double* b, void* stream);

/* Back-substitution and the candidate parameters: dX_p = -Vinv_p (gp_p + sum_o (Jc_o^T Jp_o)^T dc_o) in observation order,
 * X_new = X + dX; pose_new = (exp(w) R, t + dt) and focal_new = f + df from dc [ncol]. */
int nero_sfm_ba_backsub(const long long* pt_off, int P, const int* obs_img, const int* img_cam, int nimg, int ncam, const double* Jc,
                        const double* Jp, const double* Vinv, const double* gp, const double* dc, const double* pose, const double* focal,
                        const double* X, double* pose_new, double* focal_new, double* X_new, void* stream);

/* cost [1] = the sum of squared residuals of the point-ordered observations: each point's in observation order, per-block
 * partials [ceil(P / NERO_SFM_BLOCK)] of the points in a fixed tree order, then added in block order.  P >= 1. */
int nero_sfm_ba_cost(const long long* pt_off, int P, const int* obs_img, const double* obs_xy, const double* pose, const int* img_cam,
                     const double* focal, const double* pp, const double* X, double* partial, double* cost, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_SFM_H_ */
