// Relighting path tracer (the GPU replacement of the reference's Blender Cycles render, relight.py /
// blender_backend/relight_backend.py): a triangle mesh with per-vertex NeRO materials under an equirectangular environment map.
//
// One thread per pixel loops over the sample indices [spp0, spp0 + spp) in order and adds each camera path's radiance into a
// per-pixel fp32 running sum (rgb, hit count).  Every random number is a hash of (seed, pixel, sample, bounce, dim)
// (math_relight.cuh), so the image does not depend on how the host splits the samples over launches.
// Per path: jittered camera ray -> closest hit; at each hit, next-event estimation from the importance-sampled environment
// with an any-hit shadow ray, and a BRDF sample (diffuse or GGX lobe) that continues the path; the two are combined with
// the power heuristic.  No Russian roulette: at most 1 + 2 * max_bounces rays per path.
#include "bvh_traverse.cuh"
#include "common.cuh"
#include "math_relight.cuh"

namespace nero {

namespace {

struct SurfHit {
  float p[3], n[3];     // hit point, unit normal facing the incoming ray
  float albedo[3], metallic, alpha;
};

__device__ __forceinline__ void surface(const nero_relight_params& q, const BvhHit& h, const float* o, const float* d, SurfHit& s) {
  const float4* tris = reinterpret_cast<const float4*>(q.tris);
  const float4 e1 = __ldg(tris + 3 * h.tri + 1), e2 = __ldg(tris + 3 * h.tri + 2);
  // marching-cubes meshes are wound with cross(e1, e2) pointing into the solid: the outward normal is its negation
  float n[3] = {-(e1.y * e2.z - e1.z * e2.y), -(e1.z * e2.x - e1.x * e2.z), -(e1.x * e2.y - e1.y * e2.x)};
  normalize3(n, n);
  if (rl_dot(n, d) > 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }   // two-sided
  for (int k = 0; k < 3; ++k) { s.p[k] = o[k] + h.t * d[k]; s.n[k] = n[k]; }
  const int f = __ldg(q.tri_ids + h.tri);
  const float w0 = 1.0f - h.u - h.v;
  const float4* vm = reinterpret_cast<const float4*>(q.vmat);
  float4 a[3], b[3];
  for (int c = 0; c < 3; ++c) {
    const int vi = __ldg(q.faces + 3 * f + c);
    a[c] = __ldg(vm + 2 * vi);
    b[c] = __ldg(vm + 2 * vi + 1);
  }
  s.albedo[0] = w0 * a[0].x + h.u * a[1].x + h.v * a[2].x;
  s.albedo[1] = w0 * a[0].y + h.u * a[1].y + h.v * a[2].y;
  s.albedo[2] = w0 * a[0].z + h.u * a[1].z + h.v * a[2].z;
  s.metallic = w0 * a[0].w + h.u * a[1].w + h.v * a[2].w;
  const float r = w0 * b[0].x + h.u * b[1].x + h.v * b[2].x;
  s.alpha = r * r;
}

__device__ __forceinline__ float mis(float a, float b) {   // power heuristic a^2 / (a^2 + b^2)
  const float a2 = a * a;
  return a2 / (a2 + b * b);
}

__global__ void __launch_bounds__(128) relight_kernel(const nero_relight_params q) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 8 + (threadIdx.x >> 4);
  if (x >= q.width || y >= q.height) return;
  const uint32_t pix = uint32_t(y) * uint32_t(q.width) + uint32_t(x);
  const float4* n4 = reinterpret_cast<const float4*>(q.nodes);
  const float4* tris = reinterpret_cast<const float4*>(q.tris);
  const float4* env = reinterpret_cast<const float4*>(q.env);
  const int W = q.env_w, H = q.env_h;
  const float* R = q.pose;
  float4 acc = reinterpret_cast<float4*>(q.accum)[pix];
  unsigned long long rays = 0;
  for (int s = q.spp0; s < q.spp0 + q.spp; ++s) {
    const uint32_t si = uint32_t(s);
    // camera ray: OpenCV pinhole, pose = world -> camera [R | t]; box-filtered pixel sample
    const float px = float(x) + rl_uniform(q.seed, pix, si, 0, 0), py = float(y) + rl_uniform(q.seed, pix, si, 0, 1);
    const float cx = (px - q.K[2]) / q.K[0], cy = (py - q.K[3]) / q.K[1];
    float d[3], o[3];
    for (int k = 0; k < 3; ++k) {
      d[k] = R[k] * cx + R[4 + k] * cy + R[8 + k];
      o[k] = -(R[k] * R[3] + R[4 + k] * R[7] + R[8 + k] * R[11]);
    }
    normalize3(d, d);
    ++rays;
    BvhHit h = bvh_traverse<false>(n4, tris, o[0], o[1], o[2], d[0], d[1], d[2], 1e30f);
    if (h.tri < 0) continue;                      // transparent film: background seen directly contributes nothing
    float L[3] = {0.f, 0.f, 0.f}, thr[3] = {1.f, 1.f, 1.f};
    for (int b = 0; b < q.max_bounces; ++b) {
      SurfHit sh;
      surface(q, h, o, d, sh);
      const float v[3] = {-d[0], -d[1], -d[2]};
      float po[3];
      for (int k = 0; k < 3; ++k) po[k] = sh.p[k] + kRelightEps * sh.n[k];
      const uint32_t bb = uint32_t(b);
      const float ps = rl_spec_prob(sh.albedo, sh.metallic);
      // next-event estimation from the environment
      {
        const int j = rl_search(q.cdf_rows, H, rl_uniform(q.seed, pix, si, bb, 2));
        const int i = rl_search(q.cdf_cols + size_t(j) * (W + 1), W, rl_uniform(q.seed, pix, si, bb, 3));
        const float uu = (float(i) + rl_uniform(q.seed, pix, si, bb, 4)) / float(W);
        const float vv = (float(j) + rl_uniform(q.seed, pix, si, bb, 5)) / float(H);
        float l[3];
        const float ce = rl_env_dir(uu, vv, l);
        const float pl = rl_env_pdf(__ldg(q.env_p + size_t(j) * W + i), W, H, ce);
        const float NoL = rl_dot(sh.n, l);
        if (NoL > 0.f && pl > 0.f) {
          float f[3];
          rl_brdf(sh.n, v, l, sh.albedo, sh.metallic, sh.alpha, q.ggx_smith, f);
          ++rays;
          if (bvh_traverse<true>(n4, tris, po[0], po[1], po[2], l[0], l[1], l[2], 1e30f).tri < 0) {
            const float pb = rl_bsdf_pdf(sh.n, v, l, sh.alpha, ps);
            const float w = mis(pl, pb) * NoL / pl;
            const float4 le = __ldg(env + size_t(j) * W + i);
            L[0] += thr[0] * f[0] * le.x * w;
            L[1] += thr[1] * f[1] * le.y * w;
            L[2] += thr[2] * f[2] * le.z * w;
          }
        }
      }
      // BRDF sample: continues the path
      float l[3];
      const float r1 = rl_uniform(q.seed, pix, si, bb, 7), r2 = rl_uniform(q.seed, pix, si, bb, 8);
      if (rl_uniform(q.seed, pix, si, bb, 6) < ps) rl_sample_ggx(sh.n, v, sh.alpha, r1, r2, l);
      else rl_sample_diffuse(sh.n, r1, r2, l);
      normalize3(l, l);
      const float pb = rl_bsdf_pdf(sh.n, v, l, sh.alpha, ps);
      if (!(pb > 0.f)) break;
      float f[3];
      rl_brdf(sh.n, v, l, sh.albedo, sh.metallic, sh.alpha, q.ggx_smith, f);
      const float NoL = rl_dot(sh.n, l);
      for (int k = 0; k < 3; ++k) thr[k] *= f[k] * NoL / pb;
      ++rays;
      h = bvh_traverse<false>(n4, tris, po[0], po[1], po[2], l[0], l[1], l[2], 1e30f);
      if (h.tri < 0) {                            // escapes: environment radiance, MIS-weighted against the light sampler
        float uu, vv;
        rl_env_uv(l, &uu, &vv);
        const int tx = rl_texel(uu, vv, W, H);
        const float pl = rl_env_pdf(__ldg(q.env_p + tx), W, H, sqrtf(l[0] * l[0] + l[1] * l[1]));
        const float w = mis(pb, pl);
        const float4 le = __ldg(env + tx);
        L[0] += thr[0] * le.x * w;
        L[1] += thr[1] * le.y * w;
        L[2] += thr[2] * le.z * w;
        break;
      }
      for (int k = 0; k < 3; ++k) { o[k] = po[k]; d[k] = l[k]; }
    }
    // running sums in sample order; __fadd_rn keeps the additions from being contracted, so any split of the samples over
    // launches gives the same bits
    acc.x = __fadd_rn(acc.x, L[0]);
    acc.y = __fadd_rn(acc.y, L[1]);
    acc.z = __fadd_rn(acc.z, L[2]);
    acc.w = __fadd_rn(acc.w, 1.0f);
  }
  reinterpret_cast<float4*>(q.accum)[pix] = acc;
  if (q.rays) atomicAdd(q.rays, rays);
}

}  // namespace

extern "C" int nero_relight_render(const nero_relight_params* p, void* stream) {
  if (!p) return NERO_ERR_ARG;
  const nero_relight_params& q = *p;
  if (!q.nodes || !q.tris || !q.tri_ids || !q.faces || !q.vmat || !q.env || !q.env_p || !q.cdf_rows || !q.cdf_cols || !q.accum)
    return NERO_ERR_ARG;
  if (q.env_w < 1 || q.env_h < 1 || q.width < 1 || q.height < 1 || q.spp0 < 0 || q.spp < 0 || q.max_bounces < 1) return NERO_ERR_ARG;
  if (q.spp == 0) return NERO_OK;
  const dim3 grid((q.width + 15) / 16, (q.height + 7) / 8);
  relight_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
