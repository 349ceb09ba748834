// Image metrics of uint8 images: quantisation, exact squared-error sums (PSNR) and SSIM.  The definitions are stated once in
// nero_b200/metrics.py, the ABI in include/nero_metrics.h.
//
//   quantize  one thread per value: fp32 x * 255 rounded to nearest, clipped and truncated (NaN -> 0).
//   sse       blocks of 192 threads over a contiguous range of one image's bytes; 192 is a multiple of every channel count
//             1..4, so each thread keeps to one channel.  Integer sums, one 64-bit atomic per (block, channel): exact, so the
//             result does not depend on the order.
//   ssim      pass 1: one thread per (image, column, channel) walks down its column keeping running sums of X, Y, XX, YY, XY
//             over the window ('reflect' boundary) and stores the five vertically filtered planes; neighbouring threads read
//             neighbouring bytes.  pass 2: one thread per (image, row, channel) walks along its row the same way, forms S,
//             optionally stores it and sums the cropped row left to right.  finish: one thread per (image, channel) adds
//             the row sums in row order.
//
// Every fp64 operation of the SSIM chain is an explicit round-to-nearest intrinsic (no contraction), so the S map is the
// numpy / scipy expression bit for bit, and nothing is accumulated across threads.
#include "common.cuh"
#include "../../include/nero_metrics.h"

namespace nero {
namespace {

constexpr int kQuantBlock = 256;
constexpr int kSseBlock = 192;           // a multiple of C for C = 1, 2, 3, 4
constexpr int kSseIters = 64;            // bytes per thread per block: 64 * 255^2 < 2^32
constexpr int kSsimBlock = 128;

__global__ void __launch_bounds__(kQuantBlock) quantize_kernel(const float* __restrict__ x, long long n, unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kQuantBlock + threadIdx.x;
  if (i >= n) return;
  const float v = __fmul_rn(x[i], 255.0f);
  // !(v > 0) is true for NaN as well; v >= 255 catches +inf
  out[i] = !(v > 0.0f) ? 0 : v >= 255.0f ? 255 : (unsigned char)(int)v;
}

__global__ void __launch_bounds__(kSseBlock) sse_kernel(const unsigned char* __restrict__ gt, const unsigned char* __restrict__ pr,
                                                        long long per_image, int C, unsigned long long* __restrict__ sse) {
  __shared__ unsigned long long s_acc[kSseBlock];
  const int b = blockIdx.y;
  const long long base = (long long)b * per_image;
  const long long e0 = (long long)blockIdx.x * (kSseBlock * kSseIters) + threadIdx.x;
  unsigned int acc = 0;
#pragma unroll 4
  for (int j = 0; j < kSseIters; ++j) {
    const long long e = e0 + (long long)j * kSseBlock;
    if (e < per_image) {
      const int d = int(gt[base + e]) - int(pr[base + e]);
      acc += unsigned(d * d);
    }
  }
  s_acc[threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.x < C) {
    unsigned long long t = 0;
    for (int k = threadIdx.x; k < kSseBlock; k += C) t += s_acc[k];
    atomicAdd(sse + (size_t)b * C + threadIdx.x, t);
  }
}

// index of position i of a line of length n extended by half-sample reflection (d c b a | a b c d | d c b a); |overhang| <= n
__device__ __forceinline__ int reflect(int i, int n) { return i < 0 ? -i - 1 : i >= n ? 2 * n - 1 - i : i; }

// pass 1: thread (b, q = x * C + c) runs down column q of image b
__global__ void __launch_bounds__(kSsimBlock) ssim_cols_kernel(const unsigned char* __restrict__ gt, const unsigned char* __restrict__ pr,
                                                               int B, int H, int WC, int win, double* __restrict__ work) {
  const long long t = (long long)blockIdx.x * kSsimBlock + threadIdx.x;
  if (t >= (long long)B * WC) return;
  const int b = int(t / WC), q = int(t - (long long)b * WC), r = win / 2;
  const size_t img = (size_t)b * H * WC + q, plane = (size_t)B * H * WC;
  const unsigned char* g = gt + img;
  const unsigned char* p = pr + img;
  const double dwin = double(win);
  double s[5];
  for (int j = 0; j < win; ++j) {
    const int yy = reflect(j - r, H);
    const double x = double(g[(size_t)yy * WC]), y = double(p[(size_t)yy * WC]);
    const double v[5] = {x, y, __dmul_rn(x, x), __dmul_rn(y, y), __dmul_rn(x, y)};
    for (int k = 0; k < 5; ++k) s[k] = j == 0 ? v[k] : __dadd_rn(s[k], v[k]);
  }
  double* w = work + img;
  for (int k = 0; k < 5; ++k) w[k * plane] = __ddiv_rn(s[k], dwin);
  for (int yo = 1; yo < H; ++yo) {
    const int ye = reflect(yo + r, H), yl = reflect(yo - 1 - r, H);
    const double xe = double(g[(size_t)ye * WC]), ys = double(p[(size_t)ye * WC]);
    const double xl = double(g[(size_t)yl * WC]), yl_ = double(p[(size_t)yl * WC]);
    const double ve[5] = {xe, ys, __dmul_rn(xe, xe), __dmul_rn(ys, ys), __dmul_rn(xe, ys)};
    const double vl[5] = {xl, yl_, __dmul_rn(xl, xl), __dmul_rn(yl_, yl_), __dmul_rn(xl, yl_)};
    double* wo = w + (size_t)yo * WC;
    for (int k = 0; k < 5; ++k) {
      s[k] = __dadd_rn(s[k], __dsub_rn(ve[k], vl[k]));
      wo[k * plane] = __ddiv_rn(s[k], dwin);
    }
  }
}

// pass 2: thread (b, y, c) runs along row y of channel c of image b
__global__ void __launch_bounds__(kSsimBlock) ssim_rows_kernel(int B, int H, int W, int C, int win, double cov_norm, double C1, double C2,
                                                               double* __restrict__ work, double* __restrict__ smap) {
  const long long t = (long long)blockIdx.x * kSsimBlock + threadIdx.x;
  if (t >= (long long)B * H * C) return;
  const int c = int(t % C);
  const long long by = t / C;                       // b * H + y
  const int y = int(by % H), b = int(by / H), r = win / 2;
  const size_t row = (size_t)by * W * C + c, plane = (size_t)B * H * W * C;
  const double* f = work + row;
  const double dwin = double(win);
  double s[5];
  for (int j = 0; j < win; ++j) {
    const size_t o = (size_t)reflect(j - r, W) * C;
    for (int k = 0; k < 5; ++k) s[k] = j == 0 ? f[k * plane + o] : __dadd_rn(s[k], f[k * plane + o]);
  }
  const bool in_rows = y >= r && y < H - r;
  double acc = 0.0;
  for (int x = 0; x < W; ++x) {
    if (x > 0) {
      const size_t oe = (size_t)reflect(x + r, W) * C, ol = (size_t)reflect(x - 1 - r, W) * C;
      for (int k = 0; k < 5; ++k) s[k] = __dadd_rn(s[k], __dsub_rn(f[k * plane + oe], f[k * plane + ol]));
    }
    const double ux = __ddiv_rn(s[0], dwin), uy = __ddiv_rn(s[1], dwin);
    const double uxx = __ddiv_rn(s[2], dwin), uyy = __ddiv_rn(s[3], dwin), uxy = __ddiv_rn(s[4], dwin);
    const double vx = __dmul_rn(cov_norm, __dsub_rn(uxx, __dmul_rn(ux, ux)));
    const double vy = __dmul_rn(cov_norm, __dsub_rn(uyy, __dmul_rn(uy, uy)));
    const double vxy = __dmul_rn(cov_norm, __dsub_rn(uxy, __dmul_rn(ux, uy)));
    const double A1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1);
    const double A2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
    const double B1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
    const double B2 = __dadd_rn(__dadd_rn(vx, vy), C2);
    const double S = __ddiv_rn(__dmul_rn(A1, A2), __dmul_rn(B1, B2));
    if (smap) smap[row + (size_t)x * C] = S;
    if (in_rows && x >= r && x < W - r) acc = x == r ? S : __dadd_rn(acc, S);
  }
  if (in_rows) work[5 * plane + ((size_t)b * C + c) * H + y] = acc;
}

__global__ void ssim_finish_kernel(const double* __restrict__ rowsum, int BC, int H, int W, int win, double* __restrict__ ssim) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= BC) return;
  const int r = win / 2;
  const double* rs = rowsum + (size_t)t * H;
  double acc = rs[r];
  for (int y = r + 1; y < H - r; ++y) acc = __dadd_rn(acc, rs[y]);
  ssim[t] = __ddiv_rn(acc, double((long long)(H - 2 * r) * (W - 2 * r)));
}

}  // namespace

extern "C" {

int nero_metrics_quantize(const float* x, long long n, unsigned char* out, void* stream) {
  if (n < 0 || (n > 0 && (!x || !out))) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  const long long nblk = (n + kQuantBlock - 1) / kQuantBlock;
  if (nblk > 0x7fffffffLL) return NERO_ERR_ARG;
  quantize_kernel<<<unsigned(nblk), kQuantBlock, 0, (cudaStream_t)stream>>>(x, n, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_metrics_sse(const unsigned char* gt, const unsigned char* pr, int B, int H, int W, int C, long long* sse, void* stream) {
  if (!gt || !pr || !sse || B < 1 || B > 65535 || H < 1 || W < 1 || C < 1 || C > 4) return NERO_ERR_ARG;
  const long long per_image = (long long)H * W * C;
  const long long nblk = (per_image + kSseBlock * kSseIters - 1) / (kSseBlock * kSseIters);
  if (nblk > 0x7fffffffLL) return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(sse, 0, sizeof(long long) * B * C, (cudaStream_t)stream));
  sse_kernel<<<dim3(unsigned(nblk), unsigned(B)), kSseBlock, 0, (cudaStream_t)stream>>>(gt, pr, per_image, C,
                                                                                         reinterpret_cast<unsigned long long*>(sse));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_metrics_ssim(const unsigned char* gt, const unsigned char* pr, int B, int H, int W, int C, int win, double cov_norm,
                      double C1, double C2, double* work, double* smap, double* ssim, void* stream) {
  if (!gt || !pr || !work || !ssim || B < 1 || C < 1 || win < 3 || win % 2 != 1 || H < win || W < win) return NERO_ERR_ARG;
  const long long ncol = (long long)B * W * C, nrow = (long long)B * H * C;
  if ((long long)W * C > 0x7fffffffLL || (ncol + kSsimBlock - 1) / kSsimBlock > 0x7fffffffLL ||
      (nrow + kSsimBlock - 1) / kSsimBlock > 0x7fffffffLL || (long long)B * C > 0x7fffffffLL)
    return NERO_ERR_ARG;
  cudaStream_t s = (cudaStream_t)stream;
  ssim_cols_kernel<<<unsigned((ncol + kSsimBlock - 1) / kSsimBlock), kSsimBlock, 0, s>>>(gt, pr, B, H, W * C, win, work);
  NERO_LAUNCH_CHECK();
  ssim_rows_kernel<<<unsigned((nrow + kSsimBlock - 1) / kSsimBlock), kSsimBlock, 0, s>>>(B, H, W, C, win, cov_norm, C1, C2, work, smap);
  NERO_LAUNCH_CHECK();
  const int bc = B * C;
  ssim_finish_kernel<<<(bc + 127) / 128, 128, 0, s>>>(work + (size_t)5 * B * H * W * C, bc, H, W, win, ssim);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
