/* libnero_b200 -- C ABI of the image metrics (quantisation, exact PSNR sums, SSIM of uint8 images).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 * Plain arguments only (no records).  The definitions are stated in nero_b200/metrics.py.
 *
 * Images are uint8 [B, H, W, C], row-major with the channel fastest (the layout of a numpy / torch image batch).
 */
#ifndef NERO_METRICS_H_
#define NERO_METRICS_H_

#ifdef __cplusplus
extern "C" {
#endif

/* out[i] = color_map_backward(x[i]) for i < n: v = x * 255 as one fp32 multiply, clipped to [0, 255] and truncated;
 * NaN -> 0, +inf -> 255, -inf -> 0. */
int nero_metrics_quantize(const float* x, long long n, unsigned char* out, void* stream);

/* sse[b * C + c] = sum over pixels of (gt - pr)^2 in channel c of image b, as exact integers (so independent of order). */
int nero_metrics_sse(const unsigned char* gt, const unsigned char* pr, int B, int H, int W, int C, long long* sse, void* stream);

/* SSIM with a win x win uniform window (win odd, 3 <= win <= min(H, W)).  Per (image, channel), all in uncontracted fp64:
 *   ux, uy, uxx, uyy, uxy = uniform_filter of X, Y, X X, Y Y, X Y (axis 0, then axis 1; 'reflect' boundary; running sums)
 *   vx = cov_norm (uxx - ux ux), vy, vxy likewise;  S = ((2 ux) uy + C1)(2 vxy + C2) / ((ux ux + uy uy + C1)(vx + vy + C2))
 *   ssim[b * C + c] = sum of S over the map with a (win - 1) / 2 border cropped (each row left to right, rows in order) / count.
 * work: 5 B H W C + B C H doubles (the five vertically filtered planes, then the cropped row sums).  smap [B, H, W, C] fp64
 * (may be NULL) receives S.  Nothing is accumulated across threads, so the result is bit-identical from run to run and does
 * not depend on the other images of the batch. */
int nero_metrics_ssim(const unsigned char* gt, const unsigned char* pr, int B, int H, int W, int C, int win, double cov_norm,
                      double C1, double C2, double* work, double* smap, double* ssim, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_METRICS_H_ */
