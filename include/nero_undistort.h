/* libnero_b200 -- C ABI of lens undistortion: the keypoint inversion of COLMAP's SIMPLE_RADIAL model and the resampling
 * of an RGB8 image to the pinhole camera of the undistorted view.
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The camera rule that picks the
 * undistorted camera runs on the host (nero_b200/undistort.py); oracle/nero_oracle_undistort.py restates all of it.
 *
 * Model (SIMPLE_RADIAL, params f, cx, cy, k).  A camera-frame point Y has x = Y_x / Y_z, y = Y_y / Y_z and, with
 * r2 = x x + y y and d = 1 + k r2, the image point u = (f x) d + cx, v = (f y) d + cy.  Pixel (i, j) has its centre at the
 * image point (i + 1/2, j + 1/2).
 *
 * Every fp64 expression below is evaluated as written, left to right, each operation correctly rounded and none contracted
 * (__dadd_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn), so numpy repeats the results bit for bit.
 *
 * Inverse.  For an image point (u, v): xd = (u - cx) / f, yd = (v - cy) / f, rd = sqrt(xd xd + yd yd).  Newton's method on
 * r (1 + k r^2) = rd from r = rd, exactly NERO_UNDISTORT_NEWTON steps of
 *     t = k (r r);  e = r (1 + t) - rd;  r = r - e / (1 + 3 t)
 * then, with t and e recomputed at the final r, the point is valid iff 1 + 3 t > 0 (r is on the monotone branch),
 * |e| <= NERO_UNDISTORT_TOL and r >= 0 (all false for a NaN).  x = xd (r / rd), y = yd (r / rd); x = xd, y = yd when rd = 0.
 *
 * Warp.  Output pixel (i, j) of the pinhole camera (f, cx', cy'): x = (i + 1/2 - cx') / f, y = (j + 1/2 - cy') / f, distorted
 * to (u, v) by the model above; the input is sampled bilinearly at texel point (tx, ty) = (u - 1/2, v - 1/2):
 *     x0 = floor(tx), a = tx - x0, taps x0 and x0 + 1 clamped to [0, w - 1] (x0 first clamped to [-1, w]), likewise y;
 *     c = (1 - b) ((1 - a) p00 + a p01) + b ((1 - a) p10 + a p11)   (p_rc: the tap in row y0 or y1 (r = 0, 1) and column x0 or x1 (c = 0, 1))
 *     byte = min(max(floor(c + 1/2), 0), 255).
 * RGB8 in and out, rows packed (stride 3 w bytes).
 */
#ifndef NERO_UNDISTORT_H_
#define NERO_UNDISTORT_H_

#define NERO_UNDISTORT_BLOCK 256     /* threads per block of both kernels */
#define NERO_UNDISTORT_NEWTON 50     /* Newton steps of the inverse */
#define NERO_UNDISTORT_TOL 1e-12     /* largest |r (1 + k r^2) - rd| of a valid point */

#ifdef __cplusplus
extern "C" {
#endif

/* xy [n,2] fp64 image points of camera (f, cx, cy, k) -> xn [n,2] fp64 undistorted normalised coordinates (x, y) and
 * valid [n] int32 (1 valid, 0 invalid; xn of an invalid point is whatever the iteration reached).  f > 0 and finite,
 * cx, cy, k finite, n >= 0. */
int nero_undistort_points(const double* xy, int n, double f, double cx, double cy, double k, double* xn, int* valid,
                          void* stream);

/* dst [h2, w2, 3] uint8 = src [h, w, 3] uint8 of camera (f, cx, cy, k) resampled to the pinhole camera (f, cx2, cy2) of
 * size w2 x h2.  f > 0 and every parameter finite; 1 <= w, h, w2, h2 and w h, w2 h2 < 2^31. */
int nero_undistort_image(const unsigned char* src, int w, int h, double f, double cx, double cy, double k,
                         unsigned char* dst, int w2, int h2, double cx2, double cy2, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_UNDISTORT_H_ */
