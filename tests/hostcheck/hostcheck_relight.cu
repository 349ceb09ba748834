// CPU harness (TEST INFRASTRUCTURE): runs the host+device functions of nero_b200/csrc/math_relight.cuh on the HOST so that
// tests/test_relight_host.py can compare them with the numpy oracle (oracle/nero_oracle_relight.py) without a GPU.
#include "../../nero_b200/csrc/math_relight.cuh"
using namespace nero;

extern "C" {
void hc_rl_uniform(int n, unsigned seed, const int* pixel, const int* sample, const int* bounce, const int* dim, float* out) {
  for (int i = 0; i < n; ++i) out[i] = rl_uniform(seed, uint32_t(pixel[i]), uint32_t(sample[i]), uint32_t(bounce[i]), uint32_t(dim[i]));
}
void hc_rl_search(const float* cdf, int m, int n, const float* u, int* out) {
  for (int i = 0; i < n; ++i) out[i] = rl_search(cdf, m, u[i]);
}
// (u, v) -> direction, cos(elevation) -> (u, v) and texel index on a W x H map
void hc_rl_env(int n, const float* u, const float* v, int W, int H, float* d, float* ce, float* uv, int* tx) {
  for (int i = 0; i < n; ++i) {
    ce[i] = rl_env_dir(u[i], v[i], d + 3 * i);
    rl_env_uv(d + 3 * i, uv + 2 * i, uv + 2 * i + 1);
    tx[i] = rl_texel(uv[2 * i], uv[2 * i + 1], W, H);
  }
}
void hc_rl_lobe(int n, const float* albedo, const float* metallic, float* ps) {
  for (int i = 0; i < n; ++i) ps[i] = rl_spec_prob(albedo + 3 * i, metallic[i]);
}
// spec[i] != 0: GGX sample, else cosine sample; returns the direction and the mixture pdf with lobe probability ps[i]
void hc_rl_sample(int n, const float* nrm, const float* view, const float* alpha, const float* r1, const float* r2, const int* spec,
                  const float* ps, float* l, float* pdf) {
  for (int i = 0; i < n; ++i) {
    if (spec[i]) rl_sample_ggx(nrm + 3 * i, view + 3 * i, alpha[i], r1[i], r2[i], l + 3 * i);
    else rl_sample_diffuse(nrm + 3 * i, r1[i], r2[i], l + 3 * i);
    normalize3(l + 3 * i, l + 3 * i);
    pdf[i] = rl_bsdf_pdf(nrm + 3 * i, view + 3 * i, l + 3 * i, alpha[i], ps[i]);
  }
}
void hc_rl_brdf(int n, const float* nrm, const float* view, const float* l, const float* albedo, const float* metallic,
                const float* alpha, int ggx, float* f) {
  for (int i = 0; i < n; ++i)
    rl_brdf(nrm + 3 * i, view + 3 * i, l + 3 * i, albedo + 3 * i, metallic[i], alpha[i], ggx, f + 3 * i);
}
}
