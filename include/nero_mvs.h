/* libnero_b200 -- C ABI of dense multi-view stereo: grey image preparation, PatchMatch plane hypotheses per pixel with an
 * NCC matching cost over plane-induced homographies, and the fp64 geometric-consistency filter.
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in
 * nero_b200/mvs.py and restated in numpy by oracle/nero_oracle_mvs.py.
 *
 * Images are row-major; pixel (x, y) is the image point (x + 1/2, y + 1/2).  A view's hypotheses are planes [h*w, 4] fp32
 * (z-depth d, then the unit camera-frame normal n facing the camera) and cost [h*w] fp32.  Every fp32 expression on the
 * PatchMatch path is evaluated uncontracted (__fmul_rn / __fadd_rn, IEEE division and square root) in the order the
 * module docstring states; every fp64 expression of the filter likewise (__dmul_rn / __dadd_rn).
 *
 * Source tables (DEVICE arrays, S <= NERO_MVS_MAX_SOURCES entries):
 *   src_img [S]   device addresses of the sources' grey images (fp32), as int64;
 *   src_wh  [S,2] their width and height;
 *   src_geo [S,12] fp32: A (row-major 3x3) = K_j R_ij K_i^-1 and b = K_j t_ij, with (R_ij, t_ij) the reference-to-source
 *                 camera transform, so a plane n.X = q of the reference maps pixel point p to A p + b (n^T K_i^-1 p) / q.
 */
#ifndef NERO_MVS_H_
#define NERO_MVS_H_

#define NERO_MVS_MAX_SOURCES 16    /* sources per reference view */
#define NERO_MVS_BLOCK 128         /* threads per block of every kernel */
#define NERO_MVS_GEO 12            /* fp32 per entry of src_geo */
#define NERO_MVS_FGEO 28           /* fp64 per entry of the filter's geo: R_ij, t_ij, R_ji, t_ji, fx, fy, cx, cy of j */

#ifdef __cplusplus
extern "C" {
#endif

/* grey [(h/s) * (w/s)] (integer division) of rgb [h,w,3] uint8: over the s x s block of each output pixel,
 * g = sum(299 R + 587 G + 114 B) / (255000 s^2), the sum in integers, one fp32 division.  1 <= s, s s 255000 < 2^31. */
int nero_mvs_grey(const unsigned char* rgb, int w, int h, int s, float* grey, void* stream);

/* stats [h*w, 2] = (mean, variance) of the reference window of every pixel: samples grey[clamp(y + l), clamp(x + k)] for
 * l, k = -radius, -radius + step, .., radius (l outer), summed in that order (sum and sum of squares), n = samples,
 * mean = sum / n, variance = sum2 / n - mean mean. */
int nero_mvs_ref_stats(const float* grey, int w, int h, int radius, int step, float* stats, void* stream);

/* Random initial hypotheses of every pixel and their costs.  kinv: ray (x + 1/2) ifx + ocx, (y + 1/2) ify + ocy, 1.
 * [dmin, dmax]: depth range; seed, view: the random stream. */
int nero_mvs_init(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats,
                  const long long* src_img, const int* src_wh, const float* src_geo, int S, int radius, int step, float dmin,
                  float dmax, unsigned int seed, int view, float* planes, float* cost, void* stream);

/* One PatchMatch pass: every pixel with (x + y) & 1 == colour evaluates its current hypothesis (its stored cost), the 8
 * neighbours' planes at distance 1 and 5 along the axes (other colour), two perturbations of its hypothesis at scale
 * 2^-iteration and a fresh random hypothesis, and keeps the lowest cost (ties: the earlier).  Reads only the other
 * colour's hypotheses and its own, so the result does not depend on scheduling. */
int nero_mvs_pass(const float* grey, int w, int h, float ifx, float ify, float ocx, float ocy, const float* stats,
                  const long long* src_img, const int* src_wh, const float* src_geo, int S, int radius, int step, float dmin,
                  float dmax, unsigned int seed, int view, int iteration, int colour, float* planes, float* cost, void* stream);

/* Geometric consistency in fp64.  A pixel with cost <= max_cost is tested against each source j (src_planes [S],
 * src_cost [S]: device addresses of j's hypotheses and costs, src_wh [S,2]; geo [S,28] fp64): its point at the pixel
 * centre goes to j, takes the depth and normal of the pixel containing the projection (when that pixel's cost is
 * <= max_cost), back-projects that depth at that pixel's centre and returns to the reference.  j agrees when the
 * reprojection error squared is <= reproj2, |z - d| <= rel_depth d and the cosine of the two normals (in the reference
 * frame) is >= cos_max.  count [h*w] = agreeing sources (0 when the cost fails), depth [h*w] = d where
 * count >= min_consistent, else 0.  K = (fx, fy, cx, cy) of the reference, scaled like its grey image. */
int nero_mvs_filter(int w, int h, double fx, double fy, double cx, double cy, const float* planes, const float* cost,
                    const long long* src_planes, const long long* src_cost, const int* src_wh, const double* geo, int S,
                    double max_cost, double reproj2, double rel_depth, double cos_max, int min_consistent, float* depth,
                    int* count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_MVS_H_ */
