// Relighting path tracer (the GPU replacement of the reference's Blender Cycles render, relight.py /
// blender_backend/relight_backend.py): a triangle mesh with per-vertex or UV-textured NeRO materials under an equirectangular
// environment map.  The two material sources differ only in surface(); relight_kernel is one path loop instantiated for each.
//
// One thread per pixel loops over the sample indices [spp0, spp0 + spp) in order and adds each camera path's radiance into a
// per-pixel fp32 running sum (rgb, hit count).  Every random number is a hash of (seed, pixel, sample, bounce, dim)
// (math_relight.cuh), so the image does not depend on how the host splits the samples over launches.
// Per path: jittered camera ray -> closest hit; at each hit, next-event estimation from the importance-sampled environment
// with an any-hit shadow ray, and a BRDF sample (diffuse or GGX lobe) that continues the path; the two are combined with
// the power heuristic.  No Russian roulette: at most 1 + 2 * max_bounces rays per path.
// The kAov instances also add each hitting sample's first-hit guides and demodulated radiance into the feature sums the
// denoiser reads (include/nero_denoise.h); they only read values the colour path computes, so accum keeps its bits.
#include "bvh_traverse.cuh"
#include "common.cuh"
#include "math_relight.cuh"
#include "../../include/nero_denoise.h"
#include "../../include/nero_relight_tex.h"

namespace nero {

namespace {

struct SurfHit {
  float p[3], n[3];     // hit point, unit normal facing the incoming ray
  float albedo[3], metallic, alpha;
};

// hit point and flat normal, shared by both material sources
__device__ __forceinline__ void hit_geometry(const nero_relight_params& q, const BvhHit& h, const float* o, const float* d, SurfHit& s) {
  const float4* tris = reinterpret_cast<const float4*>(q.tris);
  const float4 e1 = __ldg(tris + 3 * h.tri + 1), e2 = __ldg(tris + 3 * h.tri + 2);
  // marching-cubes meshes are wound with cross(e1, e2) pointing into the solid: the outward normal is its negation
  float n[3] = {-(e1.y * e2.z - e1.z * e2.y), -(e1.z * e2.x - e1.x * e2.z), -(e1.x * e2.y - e1.y * e2.x)};
  normalize3(n, n);
  if (rl_dot(n, d) > 0.f) { n[0] = -n[0]; n[1] = -n[1]; n[2] = -n[2]; }   // two-sided
  for (int k = 0; k < 3; ++k) { s.p[k] = o[k] + h.t * d[k]; s.n[k] = n[k]; }
}

struct VertexMaterials {};          // q.vmat [V,8] rows, interpolated barycentrically
struct TexMaterials {              // include/nero_relight_tex.h: vt [n_uv,2], ft [T,3], tex [h,w,8]
  const float2* vt; const int* ft; const float4* tex; int w, h;
};

__device__ __forceinline__ void surface(const nero_relight_params& q, VertexMaterials, const BvhHit& h, const float* o, const float* d,
                                        SurfHit& s) {
  hit_geometry(q, h, o, d, s);
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

__device__ __forceinline__ int wrap(int i, int n) {   // positive modulo: the repeat address mode
  i %= n;
  return i < 0 ? i + n : i;
}

// Textured materials: uv interpolated like the per-vertex rows, then a bilinear, wrapping fetch of the [h,w,8] texel rows with
// v = 0 at the bottom image row (row h-1).  alpha is the filtered roughness itself: the texture export stores the rescaled
// roughness NeRO's shading takes, not its square root.
__device__ __forceinline__ void surface(const nero_relight_params& q, const TexMaterials& m, const BvhHit& h, const float* o,
                                        const float* d, SurfHit& s) {
  hit_geometry(q, h, o, d, s);
  const int f = __ldg(q.tri_ids + h.tri);
  const float w0 = 1.0f - h.u - h.v;
  float2 t[3];
  for (int c = 0; c < 3; ++c) t[c] = __ldg(m.vt + __ldg(m.ft + 3 * f + c));
  const float uvx = w0 * t[0].x + h.u * t[1].x + h.v * t[2].x;
  const float uvy = w0 * t[0].y + h.u * t[1].y + h.v * t[2].y;
  const float sx = uvx * float(m.w) - 0.5f, sy = (1.0f - uvy) * float(m.h) - 0.5f;
  const float x0 = floorf(sx), y0 = floorf(sy);
  const float fx = sx - x0, fy = sy - y0;
  const int ix = wrap(int(x0), m.w), iy = wrap(int(y0), m.h);
  const int ix1 = ix + 1 == m.w ? 0 : ix + 1, iy1 = iy + 1 == m.h ? 0 : iy + 1;
  const size_t r0 = size_t(iy) * m.w, r1 = size_t(iy1) * m.w;
  const size_t tap[4] = {r0 + ix, r0 + ix1, r1 + ix, r1 + ix1};
  float4 a[4];
  float r[4];
  for (int k = 0; k < 4; ++k) {
    a[k] = __ldg(m.tex + 2 * tap[k]);
    r[k] = __ldg(reinterpret_cast<const float*>(m.tex + 2 * tap[k] + 1));
  }
  auto lerp = [](float p, float q_, float w) { return p + w * (q_ - p); };
  auto bilerp = [&](float c00, float c10, float c01, float c11) { return lerp(lerp(c00, c10, fx), lerp(c01, c11, fx), fy); };
  s.albedo[0] = bilerp(a[0].x, a[1].x, a[2].x, a[3].x);
  s.albedo[1] = bilerp(a[0].y, a[1].y, a[2].y, a[3].y);
  s.albedo[2] = bilerp(a[0].z, a[1].z, a[2].z, a[3].z);
  s.metallic = bilerp(a[0].w, a[1].w, a[2].w, a[3].w);
  s.alpha = bilerp(r[0], r[1], r[2], r[3]);
}

__device__ __forceinline__ float mis(float a, float b) {   // power heuristic a^2 / (a^2 + b^2)
  const float a2 = a * a;
  return a2 / (a2 + b * b);
}

template <class Materials, bool kAov>
__global__ void __launch_bounds__(128) relight_kernel(const nero_relight_params q, const Materials mat, float4* aov) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 8 + (threadIdx.x >> 4);
  if (x >= q.width || y >= q.height) return;
  const uint32_t pix = uint32_t(y) * uint32_t(q.width) + uint32_t(x);
  const float4* n4 = reinterpret_cast<const float4*>(q.nodes);
  const float4* tris = reinterpret_cast<const float4*>(q.tris);
  const float4* env = reinterpret_cast<const float4*>(q.env);
  const int W = q.env_w, H = q.env_h;
  const float* R = q.pose;
  float4 acc = reinterpret_cast<float4*>(q.accum)[pix];
  float4 f_dem, f_alb, f_nrm, f_pos;   // feature sums (kAov only)
  if (kAov) {
    f_dem = aov[4 * pix]; f_alb = aov[4 * pix + 1]; f_nrm = aov[4 * pix + 2]; f_pos = aov[4 * pix + 3];
  }
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
    float g[3], n0[3], p0[3], z0;        // first-hit guides (kAov only)
    if (kAov) {
      // Taken from a surface() of their own before the bounce loop, of a copy of the hit the compiler cannot see through,
      // and written with _rn intrinsics, which are never fused: a branch or a select on the bounce index inside the loop, or
      // a surface() the compiler can merge with the loop's first one, changes how it splits and fuses the colour path's
      // multiplies and adds, and so accum's bits.
      BvhHit h0 = h;
      asm("" : "+r"(h0.tri), "+f"(h0.t), "+f"(h0.u), "+f"(h0.v));
      SurfHit s0;
      surface(q, mat, h0, o, d, s0);
      const float m = s0.metallic, m1 = __fsub_rn(1.0f, m), f0 = __fmul_rn(0.04f, m1);
      for (int k = 0; k < 3; ++k) {
        g[k] = __fadd_rn(__fadd_rn(__fmul_rn(m1, s0.albedo[k]), f0), __fmul_rn(m, s0.albedo[k]));
        n0[k] = s0.n[k];
        p0[k] = s0.p[k];
      }
      z0 = __fmul_rn(h0.t, __fadd_rn(__fadd_rn(__fmul_rn(R[8], d[0]), __fmul_rn(R[9], d[1])), __fmul_rn(R[10], d[2])));
    }
    for (int b = 0; b < q.max_bounces; ++b) {
      SurfHit sh;
      surface(q, mat, h, o, d, sh);
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
    if (kAov) {
      float D[3];
      for (int k = 0; k < 3; ++k) D[k] = __fdiv_rn(L[k], __fadd_rn(g[k], NERO_DENOISE_DEMOD_EPS));
      const float l = __fadd_rn(__fadd_rn(__fmul_rn(0.2126f, D[0]), __fmul_rn(0.7152f, D[1])), __fmul_rn(0.0722f, D[2]));
      f_dem.x = __fadd_rn(f_dem.x, D[0]); f_dem.y = __fadd_rn(f_dem.y, D[1]); f_dem.z = __fadd_rn(f_dem.z, D[2]);
      f_dem.w = __fadd_rn(f_dem.w, __fmul_rn(l, l));
      f_alb.x = __fadd_rn(f_alb.x, g[0]); f_alb.y = __fadd_rn(f_alb.y, g[1]); f_alb.z = __fadd_rn(f_alb.z, g[2]);
      f_nrm.x = __fadd_rn(f_nrm.x, n0[0]); f_nrm.y = __fadd_rn(f_nrm.y, n0[1]); f_nrm.z = __fadd_rn(f_nrm.z, n0[2]);
      f_pos.x = __fadd_rn(f_pos.x, p0[0]); f_pos.y = __fadd_rn(f_pos.y, p0[1]); f_pos.z = __fadd_rn(f_pos.z, p0[2]);
      f_pos.w = __fadd_rn(f_pos.w, z0);
    }
  }
  reinterpret_cast<float4*>(q.accum)[pix] = acc;
  if (kAov) {
    aov[4 * pix] = f_dem; aov[4 * pix + 1] = f_alb; aov[4 * pix + 2] = f_nrm; aov[4 * pix + 3] = f_pos;
  }
  if (q.rays) atomicAdd(q.rays, rays);
}

// every check of a launch except those of the material source
bool scene_ok(const nero_relight_params& q) {
  if (!q.nodes || !q.tris || !q.tri_ids || !q.faces || !q.env || !q.env_p || !q.cdf_rows || !q.cdf_cols || !q.accum) return false;
  return q.env_w >= 1 && q.env_h >= 1 && q.width >= 1 && q.height >= 1 && q.spp0 >= 0 && q.spp >= 0 && q.max_bounces >= 1;
}

template <bool kAov, class Materials>
int launch(const nero_relight_params& q, const Materials& m, float* aov, void* stream) {
  if (q.spp == 0) return NERO_OK;
  const dim3 grid((q.width + 15) / 16, (q.height + 7) / 8);
  relight_kernel<Materials, kAov><<<grid, 128, 0, (cudaStream_t)stream>>>(q, m, reinterpret_cast<float4*>(aov));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace

extern "C" int nero_relight_render(const nero_relight_params* p, void* stream) {
  if (!p || !p->vmat || !scene_ok(*p)) return NERO_ERR_ARG;
  return launch<false>(*p, VertexMaterials{}, nullptr, stream);
}

extern "C" int nero_relight_render_textured(const nero_relight_params* p, const float* vt, const int* ft, int n_uv, const float* tex,
                                            int tex_w, int tex_h, void* stream) {
  if (!p || p->vmat || !scene_ok(*p) || !vt || !ft || !tex || n_uv < 1 || tex_w < 1 || tex_h < 1) return NERO_ERR_ARG;
  const TexMaterials m{reinterpret_cast<const float2*>(vt), ft, reinterpret_cast<const float4*>(tex), tex_w, tex_h};
  return launch<false>(*p, m, nullptr, stream);
}

extern "C" int nero_relight_render_aov(const nero_relight_params* p, float* aov, void* stream) {
  if (!p || !p->vmat || !scene_ok(*p) || !aov) return NERO_ERR_ARG;
  return launch<true>(*p, VertexMaterials{}, aov, stream);
}

extern "C" int nero_relight_render_textured_aov(const nero_relight_params* p, const float* vt, const int* ft, int n_uv,
                                                const float* tex, int tex_w, int tex_h, float* aov, void* stream) {
  if (!p || p->vmat || !scene_ok(*p) || !vt || !ft || !tex || n_uv < 1 || tex_w < 1 || tex_h < 1 || !aov) return NERO_ERR_ARG;
  const TexMaterials m{reinterpret_cast<const float2*>(vt), ft, reinterpret_cast<const float4*>(tex), tex_w, tex_h};
  return launch<true>(*p, m, aov, stream);
}

}  // namespace nero
