// SIFT features: the GPU replacement of COLMAP's feature_extractor in the custom-object workflow.  The protocol is stated in
// nero_b200/features.py, the ABI in include/nero_features.h.
//
//   blur        one thread per sample and pass (horizontal into tmp, vertical into dst); taps in shared memory.
//   dog         one thread per sample.
//   decimate    one thread per output sample.
//   extrema     count -> block_offsets -> emit over the samples of an octave's interior DoG levels: the candidates come out
//               in (level, row, column) order whatever the scheduling.
//   refine      one thread per candidate, fp64.
//   describe    one thread per keypoint: its orientation histogram and up to two descriptors accumulate in the thread's own
//               column of shared memory ([bin][thread]), so every sum runs in a fixed order without atomics.
//
// The scale space (blur, dog, decimate) is a fixed sequence of correctly rounded fp32 operations that
// oracle/nero_oracle_features.py repeats bit for bit; the orientation and descriptor use the fp32 library functions
// (atan2f, expf, __sinf, __cosf), so the oracle agrees with them to rounding.
#include <cmath>

#include "common.cuh"
#include "compact.cuh"
#include "../../include/nero_features.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_FEATURES_BLOCK;
constexpr int kMaxR = NERO_FEATURES_MAX_RADIUS;
constexpr int kBorder = NERO_FEATURES_BORDER;
constexpr int kKp = NERO_FEATURES_KP;
constexpr int kOriBins = 36;
constexpr int kDescThreads = 64;
constexpr float kTwoPi = 6.283185307179586f;

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

inline unsigned nblocks(long long n, int b = kBlock) { return unsigned((n + b - 1) / b); }

// one separable pass: acc = t0 x0, then acc + t_k (x_-k + x_+k); vertical == 1 runs along columns
template <int kVertical>
__global__ void __launch_bounds__(kBlock) blur_kernel(const float* __restrict__ src, int w, int h, const float* __restrict__ taps,
                                                      int radius, float* __restrict__ dst) {
  __shared__ float t[kMaxR + 1];
  if (threadIdx.x <= radius) t[threadIdx.x] = taps[threadIdx.x];
  __syncthreads();
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)w * h) return;
  const int x = int(i % w), y = int(i / w);
  float acc;
  if (kVertical) {
    acc = fm(t[0], __ldg(src + i));
    for (int k = 1; k <= radius; ++k)
      acc = fa(acc, fm(t[k], fa(__ldg(src + (size_t)clampi(y - k, 0, h - 1) * w + x), __ldg(src + (size_t)clampi(y + k, 0, h - 1) * w + x))));
  } else {
    const float* row = src + (size_t)y * w;
    acc = fm(t[0], __ldg(row + x));
    for (int k = 1; k <= radius; ++k) acc = fa(acc, fm(t[k], fa(__ldg(row + clampi(x - k, 0, w - 1)), __ldg(row + clampi(x + k, 0, w - 1)))));
  }
  dst[i] = acc;
}

__global__ void __launch_bounds__(kBlock) dog_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float* __restrict__ d) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i < n) d[i] = __fsub_rn(b[i], a[i]);
}

__global__ void __launch_bounds__(kBlock) decimate_kernel(const float* __restrict__ src, int w, int wo, int ho, float* __restrict__ dst) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= (long long)wo * ho) return;
  const int x = int(i % wo), y = int(i / wo);
  dst[i] = src[(size_t)(2 * y) * w + 2 * x];
}

// sample i of the interior levels (level 1 + i / (h w)) is a candidate
__device__ __forceinline__ bool is_extremum(const float* __restrict__ dog, int w, int h, long long i, float thr, int* px, int* py, int* pl) {
  const long long plane = (long long)w * h;
  const int l = 1 + int(i / plane);
  const long long r = i % plane;
  const int x = int(r % w), y = int(r / w);
  *px = x; *py = y; *pl = l;
  if (x < kBorder || y < kBorder || x >= w - kBorder || y >= h - kBorder) return false;
  const float* c = dog + l * plane + (long long)y * w + x;
  const float v = *c;
  if (!(fabsf(v) > thr)) return false;
  bool mx = true, mn = true;
  for (int dl = -1; dl <= 1; ++dl)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        if (!dl && !dy && !dx) continue;
        const float u = c[dl * plane + (long long)dy * w + dx];
        mx = mx && v > u;
        mn = mn && v < u;
      }
  return mx || mn;
}

__global__ void __launch_bounds__(kBlock) extrema_count_kernel(const float* __restrict__ dog, int w, int h, long long n, float thr,
                                                               int* __restrict__ cnt) {
  __shared__ int s_w[kBlock / 32];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  int x, y, l;
  const int f = i < n && is_extremum(dog, w, h, i, thr, &x, &y, &l);
  int tot;
  block_scan<kBlock>(f, s_w, &tot);
  if (threadIdx.x == 0) cnt[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kBlock) extrema_emit_kernel(const float* __restrict__ dog, int w, int h, long long n, float thr,
                                                              const long long* __restrict__ off, int* __restrict__ cand, long long cap) {
  __shared__ int s_w[kBlock / 32];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  int x = 0, y = 0, l = 0;
  const int f = i < n && is_extremum(dog, w, h, i, thr, &x, &y, &l);
  int tot;
  const long long k = off[blockIdx.x] + block_scan<kBlock>(f, s_w, &tot);
  if (f && k < cap) {
    cand[3 * k] = x;
    cand[3 * k + 1] = y;
    cand[3 * k + 2] = l;
  }
}

// b = -H^-1 g by Cramer's rule (H symmetric); false when H is singular
__device__ __forceinline__ bool solve3(double h00, double h01, double h02, double h11, double h12, double h22, const double g[3], double b[3]) {
  const double c00 = h11 * h22 - h12 * h12, c01 = h02 * h12 - h01 * h22, c02 = h01 * h12 - h02 * h11;
  const double det = h00 * c00 + h01 * c01 + h02 * c02;
  if (!(fabs(det) > 1e-300)) return false;
  const double c11 = h00 * h22 - h02 * h02, c12 = h01 * h02 - h00 * h12, c22 = h00 * h11 - h01 * h01;
  b[0] = -(c00 * g[0] + c01 * g[1] + c02 * g[2]) / det;
  b[1] = -(c01 * g[0] + c11 * g[1] + c12 * g[2]) / det;
  b[2] = -(c02 * g[0] + c12 * g[1] + c22 * g[2]) / det;
  return true;
}

__global__ void __launch_bounds__(kBlock) refine_kernel(const float* __restrict__ dog, int w, int h, int levels, const int* __restrict__ cand,
                                                        int n, int octave, double sigma0, double peak, double edge, float* __restrict__ kp) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const long long plane = (long long)w * h;
  int x = cand[3 * i], y = cand[3 * i + 1];
  const int l = cand[3 * i + 2];
  double b[3] = {0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0}, H[3][3], D = 0.0;
  bool ok = true;
  for (int it = 0; it <= 5; ++it) {
    const float* c = dog + l * plane + (long long)y * w + x;
#define AT(dl, dy, dx) ((double)c[(dl) * plane + (long long)(dy) * w + (dx)])
    D = AT(0, 0, 0);
    g[0] = 0.5 * (AT(0, 0, 1) - AT(0, 0, -1));
    g[1] = 0.5 * (AT(0, 1, 0) - AT(0, -1, 0));
    g[2] = 0.5 * (AT(1, 0, 0) - AT(-1, 0, 0));
    H[0][0] = AT(0, 0, 1) + AT(0, 0, -1) - 2.0 * D;
    H[1][1] = AT(0, 1, 0) + AT(0, -1, 0) - 2.0 * D;
    H[2][2] = AT(1, 0, 0) + AT(-1, 0, 0) - 2.0 * D;
    H[0][1] = H[1][0] = 0.25 * (AT(0, 1, 1) - AT(0, 1, -1) - AT(0, -1, 1) + AT(0, -1, -1));
    H[0][2] = H[2][0] = 0.25 * (AT(1, 0, 1) - AT(1, 0, -1) - AT(-1, 0, 1) + AT(-1, 0, -1));
    H[1][2] = H[2][1] = 0.25 * (AT(1, 1, 0) - AT(1, -1, 0) - AT(-1, 1, 0) + AT(-1, -1, 0));
#undef AT
    if (!solve3(H[0][0], H[0][1], H[0][2], H[1][1], H[1][2], H[2][2], g, b)) {
      ok = false;
      break;
    }
    if (it == 5) break;
    const int dx = (b[0] > 0.6 && x < w - kBorder - 1) ? 1 : ((b[0] < -0.6 && x > kBorder) ? -1 : 0);
    const int dy = (b[1] > 0.6 && y < h - kBorder - 1) ? 1 : ((b[1] < -0.6 && y > kBorder) ? -1 : 0);
    if (!dx && !dy) break;
    x += dx;
    y += dy;
  }
  const double val = D + 0.5 * (g[0] * b[0] + g[1] * b[1] + g[2] * b[2]);
  const double tr = H[0][0] + H[1][1], det = H[0][0] * H[1][1] - H[0][1] * H[0][1];
  ok = ok && fabs(b[0]) < 1.5 && fabs(b[1]) < 1.5 && fabs(b[2]) < 1.5 && fabs(val) >= peak && det > 0.0 &&
       tr * tr * edge < (edge + 1.0) * (edge + 1.0) * det;
  const double s = (double)l + b[2];
  float* o = kp + (size_t)kKp * i;
  o[0] = (float)((double)x + b[0]);
  o[1] = (float)((double)y + b[1]);
  o[2] = (float)(sigma0 * exp2(s / (double)(levels - 2)));
  o[3] = (float)val;
  o[4] = (float)octave;
  o[5] = (float)l;
  o[6] = (float)s;
  o[7] = ok ? 1.0f : 0.0f;
}

// central-difference gradient of sample (x, y) (1 <= x < w - 1, 1 <= y < h - 1): magnitude and angle in [0, 2 pi)
__device__ __forceinline__ void gradient(const float* __restrict__ img, int w, int x, int y, float* mag, float* ang) {
  const float* p = img + (size_t)y * w + x;
  const float gx = 0.5f * (p[1] - p[-1]), gy = 0.5f * (p[w] - p[-w]);
  *mag = sqrtf(gx * gx + gy * gy);
  float a = atan2f(gy, gx);
  if (a < 0.0f) a += kTwoPi;
  *ang = a;
}

__global__ void __launch_bounds__(kDescThreads) describe_kernel(const float* __restrict__ kp, int n, const long long* __restrict__ gauss,
                                                                const int* __restrict__ oct_wh, int levels, float* __restrict__ angle,
                                                                unsigned char* __restrict__ desc, int* __restrict__ nori) {
  __shared__ float sh[(kOriBins + NERO_FEATURES_DIM) * kDescThreads];
  const int t = threadIdx.x;
  float* hist = sh + t;                                   // bin b at hist[b * kDescThreads]
  float* dh = sh + kOriBins * kDescThreads + t;
  const int i = blockIdx.x * kDescThreads + t;
  if (i >= n) return;
  const float* k = kp + (size_t)kKp * i;
  const float x = k[0], y = k[1], sigma = k[2];
  const int o = (int)k[4], l = (int)k[5];
  const int w = oct_wh[2 * o], h = oct_wh[2 * o + 1];
  const float* img = (const float*)gauss[o] + (size_t)l * w * h;
  const int xi = (int)floorf(x + 0.5f), yi = (int)floorf(y + 0.5f);
  // orientation histogram
  const float sw = 1.5f * sigma;
  const int R = max(1, (int)floorf(3.0f * sw));
  for (int b = 0; b < kOriBins; ++b) hist[b * kDescThreads] = 0.0f;
  for (int yy = max(1, yi - R); yy <= min(h - 2, yi + R); ++yy)
    for (int xx = max(1, xi - R); xx <= min(w - 2, xi + R); ++xx) {
      const float dx = (float)xx - x, dy = (float)yy - y, r2 = dx * dx + dy * dy;
      if (r2 >= (float)(R * R) + 0.6f) continue;
      float m, a;
      gradient(img, w, xx, yy, &m, &a);
      int b = (int)floorf((float)kOriBins * a / kTwoPi);
      b = b >= kOriBins ? b - kOriBins : b;
      hist[b * kDescThreads] += m * expf(-r2 / (2.0f * sw * sw));
    }
  for (int it = 0; it < 6; ++it) {
    float prev = hist[(kOriBins - 1) * kDescThreads];
    const float first = hist[0];
    for (int b = 0; b < kOriBins; ++b) {
      const float cur = hist[b * kDescThreads];
      const float next = b + 1 < kOriBins ? hist[(b + 1) * kDescThreads] : first;
      hist[b * kDescThreads] = (prev + cur + next) / 3.0f;
      prev = cur;
    }
  }
  float hmax = 0.0f;
  for (int b = 0; b < kOriBins; ++b) hmax = fmaxf(hmax, hist[b * kDescThreads]);
  float p0 = -1.0f, p1 = -1.0f, th0 = 0.0f, th1 = 0.0f;   // the two highest peaks, descending (ties: lower bin)
  for (int b = 0; b < kOriBins; ++b) {
    const float h0 = hist[b * kDescThreads];
    const float hm = hist[((b + kOriBins - 1) % kOriBins) * kDescThreads], hp = hist[((b + 1) % kOriBins) * kDescThreads];
    if (!(h0 > hm && h0 > hp && h0 >= 0.8f * hmax)) continue;
    const float di = -0.5f * (hp - hm) / (hp + hm - 2.0f * h0);
    const float th = kTwoPi * ((float)b + di + 0.5f) / (float)kOriBins;
    if (h0 > p0) {
      p1 = p0; th1 = th0;
      p0 = h0; th0 = th;
    } else if (h0 > p1) {
      p1 = h0; th1 = th;
    }
  }
  const int no = p0 < 0.0f ? 0 : (p1 < 0.0f ? 1 : 2);
  nori[i] = no;
  angle[2 * i] = th0;
  angle[2 * i + 1] = th1;
  // descriptors
  const float sbp = 3.0f * sigma;
  const int W = (int)floorf(1.4142135623730951f * sbp * 2.5f + 0.5f);
  for (int a = 0; a < 2; ++a) {
    unsigned char* out = desc + ((size_t)2 * i + a) * NERO_FEATURES_DIM;
    if (a >= no) {
      for (int b = 0; b < NERO_FEATURES_DIM; ++b) out[b] = 0;
      continue;
    }
    const float th = a ? th1 : th0;
    const float s = __sinf(th), c = __cosf(th);   // th in [0, 2 pi): no range reduction needed
    for (int b = 0; b < NERO_FEATURES_DIM; ++b) dh[b * kDescThreads] = 0.0f;
    for (int yy = max(1, yi - W); yy <= min(h - 2, yi + W); ++yy)
      for (int xx = max(1, xi - W); xx <= min(w - 2, xi + W); ++xx) {
        const float dx = (float)xx - x, dy = (float)yy - y;
        const float nx = (c * dx + s * dy) / sbp, ny = (-s * dx + c * dy) / sbp;
        const float bx = nx + 1.5f, by = ny + 1.5f;
        if (!(bx > -1.0f && bx < 4.0f && by > -1.0f && by < 4.0f)) continue;
        float m, ang;
        gradient(img, w, xx, yy, &m, &ang);
        float rel = ang - th;
        rel = rel < 0.0f ? rel + kTwoPi : rel;
        rel = rel >= kTwoPi ? rel - kTwoPi : rel;
        const float nt = 8.0f * rel / kTwoPi;
        const float v = m * expf(-(nx * nx + ny * ny) / 8.0f);
        const float x0 = floorf(bx), y0 = floorf(by), t0 = floorf(nt);
        const float fx = bx - x0, fy = by - y0, ft = nt - t0;
        const int ix = (int)x0, iy = (int)y0, it = (int)t0;
        for (int ey = 0; ey < 2; ++ey) {
          const int yb = iy + ey;
          if (yb < 0 || yb > 3) continue;
          const float wy = ey ? fy : 1.0f - fy;
          for (int ex = 0; ex < 2; ++ex) {
            const int xb = ix + ex;
            if (xb < 0 || xb > 3) continue;
            const float wxy = wy * (ex ? fx : 1.0f - fx);
            for (int et = 0; et < 2; ++et) {
              const int tb = (it + et) & 7;
              dh[((yb * 4 + xb) * 8 + tb) * kDescThreads] += v * wxy * (et ? ft : 1.0f - ft);
            }
          }
        }
      }
    float n2 = 0.0f;
    for (int b = 0; b < NERO_FEATURES_DIM; ++b) n2 += dh[b * kDescThreads] * dh[b * kDescThreads];
    const float inv = n2 > 0.0f ? 1.0f / sqrtf(n2) : 0.0f;
    float m2 = 0.0f;
    for (int b = 0; b < NERO_FEATURES_DIM; ++b) {
      const float v = fminf(dh[b * kDescThreads] * inv, 0.2f);
      dh[b * kDescThreads] = v;
      m2 += v * v;
    }
    const float inv2 = m2 > 0.0f ? 1.0f / sqrtf(m2) : 0.0f;
    float l1 = 0.0f;
    for (int b = 0; b < NERO_FEATURES_DIM; ++b) l1 += dh[b * kDescThreads] * inv2;
    const float inv1 = l1 > 0.0f ? 1.0f / l1 : 0.0f;
    for (int b = 0; b < NERO_FEATURES_DIM; ++b) {
      const float v = sqrtf(dh[b * kDescThreads] * inv2 * inv1);
      out[b] = (unsigned char)fminf(255.0f, floorf(512.0f * v + 0.5f));
    }
  }
}

}  // namespace

extern "C" {

int nero_features_blur(const float* src, int w, int h, const float* taps, int radius, float* tmp, float* dst, void* stream) {
  if (!src || !taps || !tmp || !dst || w < 1 || h < 1 || (long long)w * h > 0x7fffffffLL || radius < 1 || radius > kMaxR || src == tmp ||
      tmp == dst)
    return NERO_ERR_ARG;
  const unsigned g = nblocks((long long)w * h);
  blur_kernel<0><<<g, kBlock, 0, (cudaStream_t)stream>>>(src, w, h, taps, radius, tmp);
  blur_kernel<1><<<g, kBlock, 0, (cudaStream_t)stream>>>(tmp, w, h, taps, radius, dst);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_dog(const float* a, const float* b, long long n, float* dog, void* stream) {
  if (!a || !b || !dog || n < 1) return NERO_ERR_ARG;
  dog_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(a, b, n, dog);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_decimate(const float* src, int w, int h, float* dst, void* stream) {
  if (!src || !dst || w < 2 || h < 2 || (long long)w * h > 0x7fffffffLL) return NERO_ERR_ARG;
  const int wo = w / 2, ho = h / 2;
  decimate_kernel<<<nblocks((long long)wo * ho), kBlock, 0, (cudaStream_t)stream>>>(src, w, wo, ho, dst);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_extrema(const float* dog, int w, int h, int levels, float threshold, int* blk_count, long long* blk_off,
                          long long* total, int* cand, long long cap, void* stream) {
  if (!dog || !blk_count || !blk_off || !total || (cap > 0 && !cand) || cap < 0 || w < 1 || h < 1 || levels < 3 ||
      (long long)w * h * levels > 0x7fffffffLL || !(threshold >= 0.0f))
    return NERO_ERR_ARG;
  const long long n = (long long)(levels - 2) * w * h;
  const unsigned g = nblocks(n);
  cudaStream_t st = (cudaStream_t)stream;
  extrema_count_kernel<<<g, kBlock, 0, st>>>(dog, w, h, n, threshold, blk_count);
  block_offsets<1>(blk_count, blk_off, total, g, st);
  extrema_emit_kernel<<<g, kBlock, 0, st>>>(dog, w, h, n, threshold, blk_off, cand, cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_refine(const float* dog, int w, int h, int levels, const int* cand, int n, int octave, double sigma0,
                         double peak, double edge, float* kp, void* stream) {
  if (!dog || (n > 0 && (!cand || !kp)) || n < 0 || w < 2 * kBorder + 1 || h < 2 * kBorder + 1 || levels < 3 || octave < 0 ||
      octave >= NERO_FEATURES_MAX_OCTAVES || !(sigma0 > 0.0) || !(peak >= 0.0) || !(edge > 0.0))
    return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  refine_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(dog, w, h, levels, cand, n, octave, sigma0, peak, edge, kp);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_describe(const float* kp, int n, const long long* gauss, const int* oct_wh, int O, int levels, float* angle,
                           unsigned char* desc, int* nori, void* stream) {
  if (n < 0 || (n > 0 && (!kp || !gauss || !oct_wh || !angle || !desc || !nori)) || O < 1 || O > NERO_FEATURES_MAX_OCTAVES || levels < 1)
    return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  describe_kernel<<<nblocks(n, kDescThreads), kDescThreads, 0, (cudaStream_t)stream>>>(kp, n, gauss, oct_wh, levels, angle, desc, nori);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
