// Relit-frame denoiser (include/nero_denoise.h): prep turns the path tracer's per-pixel sums into means, each a-trous
// iteration is an edge-avoiding 5x5 B3-spline filter of the albedo-demodulated colour at step 2^level guided by the first-hit
// albedo, normal and position and by the colour's own variance, and finish remodulates and re-premultiplies.
//
// One thread per output pixel, taps in a fixed order and no atomics, so the output is a pure function of the input bits.
#include "common.cuh"
#include "../../include/nero_denoise.h"

namespace nero {

namespace {

__device__ __forceinline__ float lum(float r, float g, float b) { return 0.2126f * r + 0.7152f * g + 0.0722f * b; }

__global__ void __launch_bounds__(256) prep_kernel(const float4* __restrict__ accum, const float4* __restrict__ aov, int spp, int n,
                                                   float focal, float4* __restrict__ col, float4* __restrict__ feat) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  const float hits = accum[p].w;
  if (!(hits > 0.f)) {
    col[p] = make_float4(0.f, 0.f, 0.f, NERO_DENOISE_VAR_NONE);
    feat[3 * p] = feat[3 * p + 1] = feat[3 * p + 2] = make_float4(0.f, 0.f, 0.f, 0.f);
    return;
  }
  const float4 dem = aov[4 * p], alb = aov[4 * p + 1], nrm = aov[4 * p + 2], pos = aov[4 * p + 3];
  const double inv = 1.0 / double(hits);
  const double c[3] = {dem.x * inv, dem.y * inv, dem.z * inv};
  const double l = 0.2126 * c[0] + 0.7152 * c[1] + 0.0722 * c[2];
  // E[l^2] - E[l]^2 in fp64: in fp32 the two terms cancel to noise wherever the variance is small against the mean
  const float var = hits < 2.f ? NERO_DENOISE_VAR_NONE : float(fmax(double(dem.w) * inv - l * l, 0.0) / (double(hits) - 1.0));
  col[p] = make_float4(float(c[0]), float(c[1]), float(c[2]), var);
  const double nl = sqrt(double(nrm.x) * nrm.x + double(nrm.y) * nrm.y + double(nrm.z) * nrm.z);
  const double ni = nl > 0.0 ? 1.0 / nl : 0.0;
  feat[3 * p] = make_float4(float(alb.x * inv), float(alb.y * inv), float(alb.z * inv), float(double(hits) / double(spp)));
  feat[3 * p + 1] = make_float4(float(nrm.x * ni), float(nrm.y * ni), float(nrm.z * ni), 0.f);
  feat[3 * p + 2] = make_float4(float(pos.x * inv), float(pos.y * inv), float(pos.z * inv), float(pos.w * inv / double(focal)));
}

__global__ void __launch_bounds__(128) iterate_kernel(const float4* __restrict__ col, const float4* __restrict__ feat, int W, int H,
                                                      int step, float sigma_l, float sigma_n, float sigma_x, float eps,
                                                      float4* __restrict__ out) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 8 + (threadIdx.x >> 4);
  if (x >= W || y >= H) return;
  const int p = y * W + x;
  const float4 cp = col[p];
  const float4 ap = feat[3 * p];
  if (!(ap.w > 0.f)) {           // uncovered: nothing to filter, and no neighbour reads it
    out[p] = cp;
    return;
  }
  const float4 np_ = feat[3 * p + 1], xp = feat[3 * p + 2];
  // variance prefilter: 3x3 Gaussian, neighbours weighted by their coverage
  const float g3[3] = {0.25f, 0.5f, 0.25f};
  float vs = 0.f, vw = 0.f;
  #pragma unroll
  for (int dy = -1; dy <= 1; ++dy) {
    const int qy = y + dy;
    if (qy < 0 || qy >= H) continue;
    #pragma unroll
    for (int dx = -1; dx <= 1; ++dx) {
      const int qx = x + dx;
      if (qx < 0 || qx >= W) continue;
      const int q = qy * W + qx;
      const float k = g3[dx + 1] * g3[dy + 1] * ((dx | dy) ? feat[3 * q].w : 1.0f);
      vs += k * col[q].w;
      vw += k;
    }
  }
  const float lp = lum(cp.x, cp.y, cp.z);
  const float l_scale = 1.0f / (sigma_l * sqrtf(vs / vw) + eps);
  const float xs = sigma_x * xp.w * float(step);
  const float x_scale = 1.0f / (xs * xs);
  const float h5[5] = {1.f / 16, 4.f / 16, 6.f / 16, 4.f / 16, 1.f / 16};
  float sr = 0.f, sg = 0.f, sb = 0.f, sv = 0.f, sw = 0.f;
  #pragma unroll
  for (int j = -2; j <= 2; ++j) {
    const int qy = y + j * step;
    if (qy < 0 || qy >= H) continue;
    #pragma unroll
    for (int i = -2; i <= 2; ++i) {
      const int qx = x + i * step;
      if (qx < 0 || qx >= W) continue;
      const int q = qy * W + qx;
      float w = h5[i + 2] * h5[j + 2];
      const float4 cq = col[q];
      if (i | j) {
        const float aq = feat[3 * q].w;
        if (!(aq > 0.f)) continue;
        const float4 nq = feat[3 * q + 1], xq = feat[3 * q + 2];
        const float dl = fabsf(lp - lum(cq.x, cq.y, cq.z));
        const float ex = xp.x - xq.x, ey = xp.y - xq.y, ez = xp.z - xq.z;
        const float nd = fmaxf(np_.x * nq.x + np_.y * nq.y + np_.z * nq.z, 0.f);
        w *= aq * powf(nd, sigma_n) * expf(-dl * l_scale - (ex * ex + ey * ey + ez * ez) * x_scale);
      }
      sr += w * cq.x;
      sg += w * cq.y;
      sb += w * cq.z;
      sv += w * w * cq.w;
      sw += w;
    }
  }
  const float iw = 1.0f / sw;
  out[p] = make_float4(sr * iw, sg * iw, sb * iw, sv * iw * iw);
}

__global__ void __launch_bounds__(256) finish_kernel(const float4* __restrict__ col, const float4* __restrict__ feat, int n,
                                                     float4* __restrict__ out) {
  const int p = blockIdx.x * 256 + threadIdx.x;
  if (p >= n) return;
  const float4 c = col[p], g = feat[3 * p];
  out[p] = make_float4(c.x * (g.x + NERO_DENOISE_DEMOD_EPS) * g.w, c.y * (g.y + NERO_DENOISE_DEMOD_EPS) * g.w,
                       c.z * (g.z + NERO_DENOISE_DEMOD_EPS) * g.w, g.w);
}

}  // namespace

extern "C" int nero_denoise_prep(const float* accum, const float* aov, int spp, int width, int height, float focal, float* col,
                                 float* feat, void* stream) {
  if (!accum || !aov || !col || !feat || spp < 1 || width < 1 || height < 1 || !(focal > 0.f)) return NERO_ERR_ARG;
  const int n = width * height;
  prep_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(accum),
                                                                  reinterpret_cast<const float4*>(aov), spp, n, focal,
                                                                  reinterpret_cast<float4*>(col), reinterpret_cast<float4*>(feat));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_denoise_iterate(const float* col_in, const float* feat, int width, int height, int level, float sigma_l,
                                    float sigma_n, float sigma_x, float eps, float* col_out, void* stream) {
  if (!col_in || !feat || !col_out || col_in == col_out || width < 1 || height < 1 || level < 0 || level > NERO_DENOISE_MAX_LEVEL ||
      !(sigma_l > 0.f) || !(sigma_n > 0.f) || !(sigma_x > 0.f) || !(eps > 0.f))
    return NERO_ERR_ARG;
  const dim3 grid((width + 15) / 16, (height + 7) / 8);
  iterate_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(col_in), reinterpret_cast<const float4*>(feat),
                                                         width, height, 1 << level, sigma_l, sigma_n, sigma_x, eps,
                                                         reinterpret_cast<float4*>(col_out));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_denoise_finish(const float* col, const float* feat, int width, int height, float* out, void* stream) {
  if (!col || !feat || !out || width < 1 || height < 1) return NERO_ERR_ARG;
  const int n = width * height;
  finish_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(col),
                                                                    reinterpret_cast<const float4*>(feat), n,
                                                                    reinterpret_cast<float4*>(out));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
