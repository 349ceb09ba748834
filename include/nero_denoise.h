/* libnero_b200 -- C ABI of the relit-frame denoiser: first-hit feature buffers from the path tracer and an edge-avoiding
 * a-trous wavelet filter on albedo-demodulated radiance (Dammertz et al. 2010; the spatial filter of SVGF, Schied et al. 2017).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 * The sequence is stated in nero_b200/denoise.py; oracle/nero_oracle_denoise.py restates it in fp64.
 *
 * Feature sums.  aov [h*w, NERO_DENOISE_AOV] fp32, added to (the caller zeroes it before the first launch), per pixel, over
 * the camera samples that hit the mesh, in sample order with __fadd_rn (so any split of the samples over launches gives the
 * same bits, as for accum).  For sample s with first hit (albedo a, metallic m, camera-facing face normal n, point x, depth z
 * along the camera's optical axis) and path radiance L_s:
 *   g_s = (1 - m) a + 0.04 (1 - m) + m a        guide albedo: diffuse plus normal-incidence specular reflectance
 *   D_s = L_s / (g_s + NERO_DENOISE_DEMOD_EPS)  albedo-demodulated radiance, per channel
 *   aov[0:3]   += D_s        aov[3]  += lum(D_s)^2   (lum = 0.2126 r + 0.7152 g + 0.0722 b)
 *   aov[4:7]   += g_s        aov[7]  unused (left as it is)
 *   aov[8:11]  += n          aov[11] unused
 *   aov[12:15] += x          aov[15] += z
 *
 * Filter.  With hits = accum.w and alpha = hits / spp, per pixel:
 *   prep    demodulated colour c = aov[0:3] / hits and the luminance variance of that mean,
 *           var = max(0, aov[3] / hits - lum(c)^2) / (hits - 1) in fp64 (NERO_DENOISE_VAR_NONE where hits < 2);
 *           guides: albedo g = aov[4:7] / hits, unit normal n = aov[8:11] / |aov[8:11]|, point x = aov[12:15] / hits,
 *           footprint fp = (aov[15] / hits) / focal, the size of one pixel at the pixel's mean depth.  A pixel with no hit
 *           gets zeros and var = NERO_DENOISE_VAR_NONE.
 *           col [h*w,4] = (c, var);  feat [h*w,12] = (g, alpha, n, 0, x, fp).
 *   iterate at level i (step 2^i): B3-spline taps h = 1/16 [1 4 6 4 1] (x) the same at offsets step * {-2..2}; taps outside
 *           the image are skipped.  Var'_p = the 3x3 Gaussian 1/16 [1 2 1] (x) [1 2 1] of var, each neighbour's weight times
 *           its alpha, normalised by the weights' sum.  For a tap q != p:
 *             w_q = h_q alpha_q exp(-|l_p - l_q| / (sigma_l sqrt(Var'_p) + eps)) max(0, n_p . n_q)^sigma_n
 *                   exp(-|x_p - x_q|^2 / (sigma_x fp_p step)^2)
 *           (sigma_x in pixel footprints, so one setting serves every image size); the centre tap has w_p = h_p.
 *           c' = sum w c_q / sum w,  var' = sum w^2 var_q / (sum w)^2.  Uncovered pixels (alpha 0) contribute nothing to
 *           any other pixel and keep their own (c, var).
 *   finish  out [h*w,4] = (c (g + NERO_DENOISE_DEMOD_EPS) alpha, alpha): remodulated and premultiplied by the pixel's own
 *           coverage, the layout Relighter.render returns.
 */
#ifndef NERO_DENOISE_H_
#define NERO_DENOISE_H_

#include "nero_b200.h"

#define NERO_DENOISE_AOV 16               /* floats per pixel of the feature sums */
#define NERO_DENOISE_DEMOD_EPS 1e-3f      /* demodulation guard: D = L / (g + eps) */
#define NERO_DENOISE_VAR_NONE 1e20f       /* variance of a pixel with fewer than 2 hits: no luminance stop */
#define NERO_DENOISE_MAX_LEVEL 7          /* iterate levels 0..7: at most 8 iterations, step 128 */
/* defaults, restated in nero_b200/denoise.py */
#define NERO_DENOISE_ITERATIONS 5
#define NERO_DENOISE_SIGMA_L 4.0f
#define NERO_DENOISE_SIGMA_N 64.0f
#define NERO_DENOISE_SIGMA_X 1.4f
#define NERO_DENOISE_EPS 1e-3f

#ifdef __cplusplus
extern "C" {
#endif

/* nero_relight_render / nero_relight_render_textured (include/nero_relight_tex.h) that also add the feature sums of each
 * sample into aov.  q->accum is written bit for bit as the plain entry points write it.  Returns 1 also for NULL aov. */
int nero_relight_render_aov(const nero_relight_params* q, float* aov, void* stream);
int nero_relight_render_textured_aov(const nero_relight_params* q, const float* vt, const int* ft, int n_uv, const float* tex,
                                     int tex_w, int tex_h, float* aov, void* stream);

/* accum [h*w,4] and aov [h*w,16] sums of spp samples per pixel -> col [h*w,4], feat [h*w,12].  focal: pixels (K[0][0]).
 * Returns 1 for NULL buffers, width, height or spp < 1, or focal <= 0. */
int nero_denoise_prep(const float* accum, const float* aov, int spp, int width, int height, float focal, float* col, float* feat,
                      void* stream);
/* one a-trous iteration at level in [0, NERO_DENOISE_MAX_LEVEL]: col_in -> col_out (distinct buffers).  Returns 1 for NULL
 * buffers, col_in == col_out, sizes < 1, a level outside that range, or a sigma or eps that is not positive. */
int nero_denoise_iterate(const float* col_in, const float* feat, int width, int height, int level, float sigma_l, float sigma_n,
                         float sigma_x, float eps, float* col_out, void* stream);
/* col, feat -> out [h*w,4].  Returns 1 for NULL buffers or sizes < 1. */
int nero_denoise_finish(const float* col, const float* feat, int width, int height, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_DENOISE_H_ */
