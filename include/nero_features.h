/* libnero_b200 -- C ABI of sparse features for structure from motion: the SIFT scale space, keypoint detection,
 * refinement, orientation and RootSIFT descriptors; all-pair descriptor matching on the integer tensor cores; and RANSAC
 * verification of each matched pair with a fundamental matrix.
 *
 * Same library and conventions as include/nero_mvs.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in
 * nero_b200/features.py and restated in numpy by oracle/nero_oracle_features.py.
 *
 * Images are row-major fp32; sample (x, y) of an octave is its pixel (x, y).  Every fp32 operation of the scale space is
 * uncontracted (__fmul_rn / __fadd_rn) in the order stated below, so the Gaussian and DoG levels are bit-reproducible.
 *
 * Keypoint records kp [n, NERO_FEATURES_KP] fp32: x, y (octave samples), sigma (octave samples), response (the refined DoG
 * value), octave, level (the integer Gaussian level whose gradients it uses), scale (the refined fractional level), ok
 * (1 when the candidate survives refinement, else 0).
 */
#ifndef NERO_FEATURES_H_
#define NERO_FEATURES_H_

#define NERO_FEATURES_BLOCK 128        /* threads per block of the scale-space, detection and mutual-match kernels */
#define NERO_FEATURES_MAX_RADIUS 32    /* Gaussian taps per side */
#define NERO_FEATURES_BORDER 5         /* extrema are not searched within this many samples of the edge */
#define NERO_FEATURES_KP 8             /* fp32 per keypoint record */
#define NERO_FEATURES_MAX_OCTAVES 8
#define NERO_FEATURES_DIM 128          /* descriptor bytes */
#define NERO_FEATURES_ORI 2            /* orientations kept per keypoint */
#define NERO_FEATURES_TILE 128         /* descriptor rows per match tile and per column chunk */
#define NERO_FEATURES_MAX_HYP 4096     /* RANSAC hypotheses per pair */

#ifdef __cplusplus
extern "C" {
#endif

/* dst [h,w] = the separable Gaussian of src [h,w] with taps t[0..radius] (t[k] weighs offsets +-k), clamp to edge.  A
 * horizontal pass into tmp [h,w], then a vertical pass into dst, each  acc = t0 x0;  acc = acc + t_k (x_-k + x_+k)  for
 * k = 1..radius.  1 <= radius <= NERO_FEATURES_MAX_RADIUS; taps is a DEVICE array. */
int nero_features_blur(const float* src, int w, int h, const float* taps, int radius, float* tmp, float* dst, void* stream);

/* dog [n] = b - a (one rounding). */
int nero_features_dog(const float* a, const float* b, long long n, float* dog, void* stream);

/* dst [h / 2, w / 2] (integer division) = src [2y, 2x]. */
int nero_features_decimate(const float* src, int w, int h, float* dst, void* stream);

/* Candidate extrema of one octave's DoG stack dog [levels, h, w]: sample (x, y) of level l in 1..levels-2, at least
 * NERO_FEATURES_BORDER from every edge, with |D| > threshold and D strictly greater (or strictly smaller) than its 26
 * neighbours.  cand [cap, 3] int = (x, y, l) in (l, y, x) order; *total (DEVICE int64) = the number of candidates, of which
 * the first min(total, cap) are written.  blk_count [nblk] int and blk_off [nblk] int64 are scratch with
 * nblk = ceil((levels - 2) h w / NERO_FEATURES_BLOCK). */
int nero_features_extrema(const float* dog, int w, int h, int levels, float threshold, int* blk_count, long long* blk_off,
                          long long* total, int* cand, long long cap, void* stream);

/* Quadratic refinement in fp64 of n candidates cand [n,3] of octave `octave` (dog [levels, h, w]): at most 5 moves of one
 * sample each; a candidate is kept (ok = 1) when its last offset is below 1.5 in each coordinate, its refined |D| is
 * >= peak and tr(H)^2 / det(H) < (edge + 1)^2 / edge with det(H) > 0.  sigma = sigma0 2^(scale / (levels - 2)).  Writes
 * kp [n, NERO_FEATURES_KP]; cand and kp may be NULL when n = 0 (an octave without extrema). */
int nero_features_refine(const float* dog, int w, int h, int levels, const int* cand, int n, int octave, double sigma0,
                         double peak, double edge, float* kp, void* stream);

/* Orientations and descriptors of n keypoints kp [n, NERO_FEATURES_KP] (any octaves).  gauss [O]: DEVICE addresses (int64)
 * of each octave's Gaussian stack [levels, h, w]; oct_wh [O, 2] their widths and heights.  For each keypoint a 36-bin
 * gradient-orientation histogram, six circular [1 1 1] / 3 smoothings, then up to NERO_FEATURES_ORI peaks >= 0.8 of the
 * maximum in descending order (ties: lower bin), each interpolated by a parabola; for each orientation a 4 x 4 x 8
 * histogram with trilinear binning, L2-normalised, clamped at 0.2, L2-normalised, L1-normalised and square-rooted, then
 * min(255, round(512 v)).  angle [n, 2] fp32 (radians), desc [n, 2, 128] uint8, nori [n] int (0..2). */
int nero_features_describe(const float* kp, int n, const long long* gauss, const int* oct_wh, int O, int levels, float* angle,
                           unsigned char* desc, int* nori, void* stream);

/* Row bests of the directed tiles of an all-pair match.  desc [rows, 128] uint8 and norms [rows] int (|d|^2) hold every
 * image's descriptors from its row offset (a multiple of NERO_FEATURES_TILE; rows past an image's count are zero).
 * tiles [T, 5] int: (a_off, a_rows, b_off, b_rows, out): rows a_off .. a_off + 128 of image a against image b's b_rows
 * rows; best [out + r, 3] int = (column index of the nearest, its squared distance d1, the second-nearest's d2) for each of
 * the a_rows (<= 128) rows, ties to the lower column; d2 = 2^31 - 1 without a second column.  The dot products are exact
 * (u8 x u8 -> s32 wgmma), so the distances are exact integers. */
int nero_features_match(const unsigned char* desc, const int* norms, const int* tiles, int T, int* best, void* stream);

/* Matches that pass the ratio test den d1 < num d2, d1 <= max_d1 and the mutual test, over the forward tiles
 * fwd [T, 4] int = (fwd_best, bwd_best, rows, row0): row r < rows of the tile reads best[fwd_best + r] = (c, d1, d2) and is
 * kept when best[bwd_best + c][0] == row0 + r.  matches [cap, 2] uint32 = (row0 + r, c) in tile order, then row order;
 * blk_count [T] int, blk_off [T] int64 (the tile's first match) and *total (DEVICE int64) as in nero_features_extrema. */
int nero_features_mutual(const int* best, const int* fwd, int T, int num, int den, int max_d1, int* blk_count, long long* blk_off,
                         long long* total, unsigned int* matches, long long cap, void* stream);

/* RANSAC per pair, one block each: pts [M, 4] fp64 (x1, y1, x2, y2) of every pair's matches, pair p owning rows
 * off[p] .. off[p + 1] (off [P + 1] int64).  `hypotheses` 8-point fundamental matrices, each from 8 distinct matches drawn
 * by the hash of (seed, p, hypothesis, draw), solved in fp64 on Hartley-normalised points with the rank-2 constraint;
 * inliers have a squared Sampson distance <= max_err2.  The largest inlier count wins (ties: the lower hypothesis), its
 * inliers are refit once, and the refit's inliers are final.  F [P, 9] fp64 (x2^T F x1 = 0, unit Frobenius norm, largest
 * |entry| positive), best [P, 2] int = (winning hypothesis, its count), count [P] int = final inliers, inlier [M] uint8.
 * A pair with fewer than 8 matches gets F = 0, best = (-1, 0), count = 0. */
int nero_features_verify(const double* pts, const long long* off, int P, int hypotheses, unsigned int seed, double max_err2, double* F,
                         int* best, int* count, unsigned char* inlier, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_FEATURES_H_ */
