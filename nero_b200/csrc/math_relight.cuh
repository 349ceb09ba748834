// Per-sample math of the relighting path tracer (k_relight.cu): the counter-based random numbers, the equirectangular
// environment mapping and its table search, the lobe choice, the BRDF sampling pdfs and NeRO's stage-II BRDF.  Host+device
// so that tests/hostcheck compiles the same expressions for the CPU; oracle/nero_oracle_relight.py restates them in numpy.
// The microfacet terms are those of math_mc.cuh (the model the materials were fitted under, network/field.py:916-930).
#pragma once
#include <cmath>
#include <cstdint>

#include "common.cuh"
#include "hash.cuh"
#include "math_mc.cuh"

namespace nero {

constexpr float kRelightEps = 1e-4f;      // offset of spawned rays along the side normal
constexpr float kRelightMinAlpha = 1e-3f; // GGX sampling floor of alpha (the BRDF itself uses the unclamped alpha)

// uniform in [0, 1) with 24 random bits, a pure function of (seed, pixel, sample, bounce, dim)
NERO_HD float rl_uniform(uint32_t seed, uint32_t pixel, uint32_t sample, uint32_t bounce, uint32_t dim) {
  uint32_t h = rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u);
  h = rl_mix(h ^ pixel);
  h = rl_mix(h ^ sample);
  h = rl_mix(h ^ ((bounce << 8) | dim));
  return float(h >> 8) * (1.0f / 16777216.0f);
}

// index j in [0, n) with cdf[j] <= u < cdf[j+1]  (cdf[0] = 0, cdf[n] = 1, non-decreasing): empty bins are never returned
NERO_HD int rl_search(const float* cdf, int n, float u) {
  int lo = 0, hi = n;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (cdf[mid] <= u) lo = mid; else hi = mid;
  }
  return lo;
}

// equirectangular mapping (z up): u = 0.5 - atan2(y, x) / 2pi, v = 0.5 + atan2(z, hypot(x, y)) / pi, v = 0 at the bottom row.
// Returns the unit direction and cos(elevation) (= sin of the polar angle).
NERO_HD float rl_env_dir(float u, float v, float* d) {
  const float phi = (0.5f - u) * (2.0f * kPi), el = (v - 0.5f) * kPi;
  const float ce = cosf(el);
  d[0] = ce * cosf(phi); d[1] = ce * sinf(phi); d[2] = sinf(el);
  return ce;
}
NERO_HD void rl_env_uv(const float* d, float* u, float* v) {
  *u = 0.5f - atan2f(d[1], d[0]) * (0.5f / kPi);
  *v = 0.5f + atan2f(d[2], sqrtf(d[0] * d[0] + d[1] * d[1])) * (1.0f / kPi);
}
NERO_HD int rl_texel(float u, float v, int W, int H) {   // row-major index, rows bottom-up
  int i = int(u * float(W)), j = int(v * float(H));
  i = i < 0 ? 0 : (i > W - 1 ? W - 1 : i);
  j = j < 0 ? 0 : (j > H - 1 ? H - 1 : j);
  return j * W + i;
}
// solid-angle pdf of the environment sampler for a direction in texel `p_texel` (probability of the texel), cos(elevation) ce
NERO_HD float rl_env_pdf(float p_texel, int W, int H, float ce) {
  return p_texel * float(W) * float(H) / (2.0f * kPi * kPi * fmaxf(ce, 1e-12f));
}

NERO_HD float rl_dot(const float* a, const float* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
NERO_HD float rl_luminance(const float* c) { return 0.2126f * c[0] + 0.7152f * c[1] + 0.0722f * c[2]; }

// probability of the GGX lobe: the specular share of (diffuse albedo, F0) luminance, at least 1/4 while the diffuse lobe is nonzero
NERO_HD float rl_spec_prob(const float* albedo, float metallic) {
  const float m1 = 1.0f - metallic;
  const float f0[3] = {0.04f * m1 + metallic * albedo[0], 0.04f * m1 + metallic * albedo[1], 0.04f * m1 + metallic * albedo[2]};
  const float kd = rl_luminance(albedo) * m1, ks = rl_luminance(f0);
  if (!(kd > 0.f)) return 1.0f;
  return fmaxf(ks / (kd + ks), 0.25f);
}

// cosine-weighted direction around n
NERO_HD void rl_sample_diffuse(const float* n, float r1, float r2, float* l) {
  float x[3], y[3];
  mc_frame(n, x, y);
  const float phi = 2.0f * kPi * r1, st = sqrtf(r2), ct = sqrtf(1.0f - r2);
  const float cp = cosf(phi) * st, sp = sinf(phi) * st;
  for (int k = 0; k < 3; ++k) l[k] = cp * x[k] + sp * y[k] + ct * n[k];
}
// half vector from the exact GGX NDF (alpha floored at kRelightMinAlpha) reflected about it
NERO_HD void rl_sample_ggx(const float* n, const float* v, float alpha, float r1, float r2, float* l) {
  const float a = fmaxf(alpha, kRelightMinAlpha), a2 = a * a;
  float x[3], y[3];
  mc_frame(n, x, y);
  const float phi = 2.0f * kPi * r1;
  const float ct = sqrtf((1.0f - r2) / (1.0f + (a2 - 1.0f) * r2)), st = sqrtf(fmaxf(1.0f - ct * ct, 0.f));
  const float cp = cosf(phi) * st, sp = sinf(phi) * st;
  float h[3];
  for (int k = 0; k < 3; ++k) h[k] = cp * x[k] + sp * y[k] + ct * n[k];
  const float vh = rl_dot(v, h);
  for (int k = 0; k < 3; ++k) l[k] = 2.0f * vh * h[k] - v[k];
}

// solid-angle pdf of the BRDF sampler (lobe mixture) for direction l; 0 below the surface
NERO_HD float rl_bsdf_pdf(const float* n, const float* v, const float* l, float alpha, float ps) {
  const float NoL = rl_dot(n, l);
  if (!(NoL > 0.f)) return 0.f;
  float h[3] = {v[0] + l[0], v[1] + l[1], v[2] + l[2]};
  normalize3(h, h);
  const float NoH = fminf(fmaxf(rl_dot(n, h), 0.f), 1.0f), VoH = fmaxf(rl_dot(v, h), 1e-12f);
  const float a = fmaxf(alpha, kRelightMinAlpha), a2 = a * a;
  const float den = NoH * NoH * (a2 - 1.0f) + 1.0f;
  const float D = a2 / (kPi * den * den);
  return (1.0f - ps) * NoL * (1.0f / kPi) + ps * D * NoH / (4.0f * VoH);
}

// NeRO's stage-II BRDF (field.py:941-984 as a closed form): albedo (1-m)/pi + F D G / (4 NoV NoL), F0 = 0.04 (1-m) + m albedo,
// Schlick F, D with its +1e-4 (mc_ggx_d), G per ggx_smith (mc_geometry).  Zero unless both NoV and NoL are positive.
NERO_HD void rl_brdf(const float* n, const float* v, const float* l, const float* albedo, float metallic, float alpha, int ggx_smith,
                     float* f) {
  const float NoV = rl_dot(n, v), NoL = rl_dot(n, l);
  if (!(NoV > 0.f) || !(NoL > 0.f)) { f[0] = f[1] = f[2] = 0.f; return; }
  float h[3] = {v[0] + l[0], v[1] + l[1], v[2] + l[2]};
  normalize3(h, h);
  const float NoH = fminf(fmaxf(rl_dot(n, h), 0.f), 1.0f), VoH = fminf(fmaxf(rl_dot(v, h), 0.f), 1.0f);
  const float nov = fminf(NoV, 1.0f), nol = fminf(NoL, 1.0f);
  const float D = mc_ggx_d(NoH, alpha);
  const float G = mc_geometry(nov, nol, alpha, ggx_smith);
  const float spec = D * G / (4.0f * nov * nol);
  const float f5 = t_pow5(1.0f - VoH);
  const float m1 = 1.0f - metallic;
  for (int k = 0; k < 3; ++k) {
    const float f0 = 0.04f * m1 + metallic * albedo[k];
    f[k] = albedo[k] * m1 * (1.0f / kPi) + (f0 + (1.0f - f0) * f5) * spec;
  }
}

}  // namespace nero
