/* libnero_b200 -- C ABI of the environment-light export (the outer light of either stage as an equirectangular HDR map).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 * Plain arguments only (no records).  The protocol is stated in nero_b200/envmap.py.
 *
 * Map conventions (nero_b200/relight.py): the map is `width` x `height` texels stored row 0 at the top, so texel (x, y) has
 * j = height - 1 - y rows below it.  Row r of the MLP input is texel r / ssaa^2 (row-major index y * width + x) and sub-sample
 * k = r % ssaa^2 = b * ssaa + a, which sits at u = (x + (a + 1/2) / ssaa) / width, v = (j + (b + 1/2) / ssaa) / height.
 * Its direction is the inverse of relight's lookup, evaluated in fp64:
 *   phi = (1/2 - u) 2 pi, el = (v - 1/2) pi, d = (cos el cos phi, cos el sin phi, sin el),
 * then d <- frame d (row-major 3x3, fp64, optional) and rounded to fp32 once.
 */
#ifndef NERO_ENVMAP_H_
#define NERO_ENVMAP_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Outer-light MLP input of rows [row0, row0 + n): A[i, 0:72] = IDE(d, kappa_inv) (utils/ref_utils.py, the reference's fp32
 * arithmetic), A[i, 72:lda] = 0 -- except with `sphere`:
 *   1 (stage I, network/field.py:559-561)  A[i, 72:144] = IDE(normalize(offset_points_to_sphere(c) + d t), kappa_inv);
 *   2 (stage II, network/field.py:843-850) A[i, 72:144] = IDE(c' + d t, 0), c' = 0.999 c when |c| > 0.999, not normalised;
 * t = get_sphere_intersection, c = (cx, cy, cz); then A[i, 144:lda] = 0.  frame [9] (device, may be NULL = identity).
 * dirs [n,3] (may be NULL) receives the fp32 directions.  One thread per row; rows are written whole through a per-warp
 * shared-memory tile.  lda is a multiple of 4, at least 72 (144 with `sphere`). */
int nero_env_rows(long long row0, long long n, int width, int height, int ssaa, const double* frame, float kappa_inv, int sphere,
                  float cx, float cy, float cz, float* A, int lda, float* dirs, void* stream);

/* Texels [texel0, texel0 + ntex): env[t, c] = sum_k w_k L_k[c] / sum_k w_k over the ssaa^2 sub-samples k (in order), w_k =
 * cos(elevation of sub-sample k), summed in fp64 and rounded to fp32.  rad [ntex * ssaa^2, ld] holds the radiance of the
 * sub-samples of texel0 onwards (row i * ssaa^2 + k); env [width * height, 3].  One thread per texel, so a texel's value
 * does not depend on how the map was split into launches. */
int nero_env_resolve(const float* rad, int ld, long long texel0, long long ntex, int width, int height, int ssaa, float* env,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_ENVMAP_H_ */
