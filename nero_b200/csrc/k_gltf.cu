// glTF 2.0 export of a textured mesh: the per-element stages whose work scales with the mesh or the atlas.  The formulas,
// orders and fallbacks are stated once in include/nero_gltf.h.
//
//   weld_count / weld_emit  one thread per position vertex: the distinct uv indices of its corners in corner-walk order,
//                           placed by the ordered scan of compact.cuh.
//   tangents                one thread per welded vertex: angle-weighted, projected face tangents of its own corners.
//   tangent_space           one thread per covered texel: the object-space normal solved in the interpolated frame.
//   metal_rough             one thread per texel: two table lookups.
// No atomics and no shared state decides a value, so every output is bit-identical from run to run.
#include "common.cuh"
#include "compact.cuh"
#include "texel_bary.cuh"
#include "../../include/nero_gltf.h"

namespace nero {

namespace {

constexpr int kWeldThreads = 256;

__device__ __forceinline__ float gl_dot(const float a[3], const float b[3]) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
}

__device__ __forceinline__ void gl_cross(const float a[3], const float b[3], float c[3]) {
  c[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
  c[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
  c[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
}

// s / sqrt(dot(s, s)); false (s unchanged) when the length is zero
__device__ __forceinline__ bool gl_normalize(float s[3]) {
  const float l2 = gl_dot(s, s);
  if (!(l2 > 0.f)) return false;
  const float l = __fsqrt_rn(l2);
  for (int k = 0; k < 3; ++k) s[k] = __fdiv_rn(s[k], l);
  return true;
}

// s - n dot(n, s)
__device__ __forceinline__ void gl_project(const float n[3], float s[3]) {
  const float d = gl_dot(n, s);
  for (int k = 0; k < 3; ++k) s[k] = __fsub_rn(s[k], __fmul_rn(n[k], d));
}

__device__ __forceinline__ unsigned char gl_encode(float n) {
  const float k = floorf(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(n, 0.5f), 0.5f), 255.0f), 0.5f));
  return (unsigned char)(k <= 0.f ? 0 : (k >= 255.f ? 255 : int(k)));
}

// The corner walk of position vertex p (include/nero_gltf.h): f(t, s) for each corner, in order.  f returns false to stop.
template <class F>
__device__ __forceinline__ void corner_walk(int p, const int* __restrict__ tris, const int* __restrict__ vt_ptr,
                                            const int* __restrict__ vt_tri, F f) {
  int prev = -1;
  for (int j = __ldg(vt_ptr + p), e = __ldg(vt_ptr + p + 1); j < e; ++j) {
    const int t = __ldg(vt_tri + j);
    if (t == prev) continue;
    prev = t;
    for (int s = 0; s < 3; ++s)
      if (__ldg(tris + 3 * t + s) == p && !f(t, s)) return;
  }
}

// the first corner of p's walk before corner (t, s) with uv index k, as 3 t' + s'; -1 if there is none
__device__ __forceinline__ int first_with_uv(int p, int k, int t, int s, const int* __restrict__ tris, const int* __restrict__ ft,
                                             const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri) {
  int found = -1;
  corner_walk(p, tris, vt_ptr, vt_tri, [&](int t2, int s2) {
    if (t2 == t && s2 == s) return false;
    if (__ldg(ft + 3 * t2 + s2) == k) {
      found = 3 * t2 + s2;
      return false;
    }
    return true;
  });
  return found;
}

__device__ __forceinline__ int distinct_uvs(int p, const int* __restrict__ tris, const int* __restrict__ ft, const int* __restrict__ vt_ptr,
                                            const int* __restrict__ vt_tri) {
  int c = 0;
  corner_walk(p, tris, vt_ptr, vt_tri, [&](int t, int s) {
    c += first_with_uv(p, __ldg(ft + 3 * t + s), t, s, tris, ft, vt_ptr, vt_tri) < 0 ? 1 : 0;
    return true;
  });
  return c;
}

__global__ void __launch_bounds__(kWeldThreads) weld_count_kernel(const int* __restrict__ tris, const int* __restrict__ ft, int V,
                                                                  const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                                  int* __restrict__ blk_cnt) {
  __shared__ int s_w[kWeldThreads / 32];
  const int p = blockIdx.x * kWeldThreads + threadIdx.x;
  const int c = p < V ? distinct_uvs(p, tris, ft, vt_ptr, vt_tri) : 0;
  int total;
  block_scan<kWeldThreads>(c, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

// wf is written and, for a corner whose uv index appeared earlier in the walk, read back by the same thread: plain loads
__global__ void __launch_bounds__(kWeldThreads) weld_emit_kernel(const int* __restrict__ tris, const int* __restrict__ ft, int V,
                                                                 const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                                 const long long* __restrict__ blk_off, int* __restrict__ wv,
                                                                 int* __restrict__ wt, int* wf) {
  __shared__ int s_w[kWeldThreads / 32];
  const int p = blockIdx.x * kWeldThreads + threadIdx.x;
  const int c = p < V ? distinct_uvs(p, tris, ft, vt_ptr, vt_tri) : 0;
  int total;
  const int before = block_scan<kWeldThreads>(c, s_w, &total);
  if (p >= V) return;
  int next = int(blk_off[blockIdx.x] + before);
  corner_walk(p, tris, vt_ptr, vt_tri, [&](int t, int s) {
    const int k = __ldg(ft + 3 * t + s);
    const int first = first_with_uv(p, k, t, s, tris, ft, vt_ptr, vt_tri);
    if (first < 0) {
      wv[next] = p;
      wt[next] = k;
      wf[3 * t + s] = next++;
    } else {
      wf[3 * t + s] = wf[first];
    }
    return true;
  });
}

__global__ void __launch_bounds__(128) tangents_kernel(const float* __restrict__ verts, const int* __restrict__ tris,
                                                       const float* __restrict__ vt, const int* __restrict__ ft,
                                                       const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                       const float* __restrict__ normals, const int* __restrict__ wv,
                                                       const int* __restrict__ wt, int W, float* __restrict__ wnormal,
                                                       float* __restrict__ wtangent) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= W) return;
  const int p = __ldg(wv + i), k = __ldg(wt + i);
  float n[3] = {__ldg(normals + 3 * size_t(p)), __ldg(normals + 3 * size_t(p) + 1), __ldg(normals + 3 * size_t(p) + 2)};
  float T[3] = {1.f, 0.f, 0.f};
  float w = 1.f;
  if (!(gl_dot(n, n) > 0.f)) {
    n[0] = n[1] = 0.f;
    n[2] = 1.f;
  } else {
    float S[3] = {0.f, 0.f, 0.f}, h = 0.f;
    bool any = false;
    corner_walk(p, tris, vt_ptr, vt_tri, [&](int t, int s) {
      if (__ldg(ft + 3 * t + s) != k) return true;
      int c[3], u[3];
      for (int j = 0; j < 3; ++j) {
        c[j] = __ldg(tris + 3 * t + (s + j) % 3);
        u[j] = __ldg(ft + 3 * t + (s + j) % 3);
      }
      float e1[3], e2[3];
      for (int q = 0; q < 3; ++q) {
        const float p0 = __ldg(verts + 3 * size_t(c[0]) + q);
        e1[q] = __fsub_rn(__ldg(verts + 3 * size_t(c[1]) + q), p0);
        e2[q] = __fsub_rn(__ldg(verts + 3 * size_t(c[2]) + q), p0);
      }
      const float d1u = __fsub_rn(__ldg(vt + 2 * size_t(u[1])), __ldg(vt + 2 * size_t(u[0])));
      const float d1v = __fsub_rn(__ldg(vt + 2 * size_t(u[1]) + 1), __ldg(vt + 2 * size_t(u[0]) + 1));
      const float d2u = __fsub_rn(__ldg(vt + 2 * size_t(u[2])), __ldg(vt + 2 * size_t(u[0])));
      const float d2v = __fsub_rn(__ldg(vt + 2 * size_t(u[2]) + 1), __ldg(vt + 2 * size_t(u[0]) + 1));
      const float det = __fsub_rn(__fmul_rn(d1u, d2v), __fmul_rn(d2u, d1v));
      if (det == 0.f) return true;
      float tf[3], bf[3], tp[3], a1[3], a2[3];
      for (int q = 0; q < 3; ++q) {
        tf[q] = __fdiv_rn(__fsub_rn(__fmul_rn(d2v, e1[q]), __fmul_rn(d1v, e2[q])), det);
        bf[q] = __fdiv_rn(__fsub_rn(__fmul_rn(d1u, e2[q]), __fmul_rn(d2u, e1[q])), det);
        tp[q] = tf[q];
        a1[q] = e1[q];
        a2[q] = e2[q];
      }
      gl_project(n, tp);
      if (!gl_normalize(a1) || !gl_normalize(a2) || !gl_normalize(tp)) return true;
      const float a = acosf(fminf(fmaxf(gl_dot(a1, a2), -1.f), 1.f));
      float nt[3];
      gl_cross(n, tf, nt);
      for (int q = 0; q < 3; ++q) S[q] = __fadd_rn(S[q], __fmul_rn(a, tp[q]));
      h = gl_dot(nt, bf) < 0.f ? __fsub_rn(h, a) : __fadd_rn(h, a);
      any = true;
      return true;
    });
    bool ok = false;
    if (any) {
      gl_project(n, S);
      ok = gl_normalize(S);
    }
    if (ok) {
      for (int q = 0; q < 3; ++q) T[q] = S[q];
      w = h < 0.f ? -1.f : 1.f;
    } else {
      const float m0 = fabsf(n[0]), m1 = fabsf(n[1]), m2 = fabsf(n[2]);
      const int ax = (m0 <= m1 && m0 <= m2) ? 0 : (m1 <= m2 ? 1 : 2);
      const float a[3] = {ax == 0 ? 1.f : 0.f, ax == 1 ? 1.f : 0.f, ax == 2 ? 1.f : 0.f};
      gl_cross(a, n, T);
      gl_normalize(T);
    }
  }
  for (int q = 0; q < 3; ++q) {
    wnormal[3 * size_t(i) + q] = n[q];
    wtangent[4 * size_t(i) + q] = T[q];
  }
  wtangent[4 * size_t(i) + 3] = w;
}

// ((b0 r0 + b1 r1) + b2 r2) per component of three rows with the given stride
__device__ __forceinline__ void gl_blend(const float b[3], const float* r0, const float* r1, const float* r2, float out[3]) {
  for (int k = 0; k < 3; ++k)
    out[k] = __fadd_rn(__fadd_rn(__fmul_rn(b[0], __ldg(r0 + k)), __fmul_rn(b[1], __ldg(r1 + k))), __fmul_rn(b[2], __ldg(r2 + k)));
}

__device__ __forceinline__ bool gl_finite3(const float a[3]) {
  return isfinite(a[0]) && isfinite(a[1]) && isfinite(a[2]);
}

__global__ void __launch_bounds__(128) tangent_space_kernel(const unsigned* __restrict__ owner, int width, int height,
                                                            const int* __restrict__ texel, long long n, const float* __restrict__ atlas,
                                                            const int* __restrict__ faces, const int* __restrict__ wf,
                                                            const float* __restrict__ wnormal, const float* __restrict__ wtangent,
                                                            const unsigned char* __restrict__ omap, unsigned char* __restrict__ img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int L = __ldg(texel + i);
  const int t = int(__ldg(owner + L));
  float b[3];
  texel_bary(atlas, faces, t, L, width, height, b);
  int v[3];
  for (int j = 0; j < 3; ++j) v[j] = __ldg(wf + 3 * t + j);
  float N[3], T[3], B[3], c[3][3];
  gl_blend(b, wnormal + 3 * size_t(v[0]), wnormal + 3 * size_t(v[1]), wnormal + 3 * size_t(v[2]), N);
  float t4[3][4];
  for (int j = 0; j < 3; ++j) {
    for (int q = 0; q < 4; ++q) t4[j][q] = __ldg(wtangent + 4 * size_t(v[j]) + q);
    const float nj[3] = {__ldg(wnormal + 3 * size_t(v[j])), __ldg(wnormal + 3 * size_t(v[j]) + 1), __ldg(wnormal + 3 * size_t(v[j]) + 2)};
    gl_cross(nj, t4[j], c[j]);
    for (int q = 0; q < 3; ++q) c[j][q] = __fmul_rn(t4[j][3], c[j][q]);
  }
  for (int q = 0; q < 3; ++q) {
    T[q] = __fadd_rn(__fadd_rn(__fmul_rn(b[0], t4[0][q]), __fmul_rn(b[1], t4[1][q])), __fmul_rn(b[2], t4[2][q]));
    B[q] = __fadd_rn(__fadd_rn(__fmul_rn(b[0], c[0][q]), __fmul_rn(b[1], c[1][q])), __fmul_rn(b[2], c[2][q]));
  }
  gl_normalize(N);
  gl_normalize(T);
  gl_normalize(B);
  float m[3];
  for (int q = 0; q < 3; ++q) m[q] = __fsub_rn(__fdiv_rn(float(2 * int(__ldg(omap + 3 * size_t(L) + q))), 255.f), 1.f);
  float x[3] = {0.f, 0.f, 1.f};
  if (gl_normalize(m)) {
    float bn[3], nt[3], tb[3];
    gl_cross(B, N, bn);
    gl_cross(N, T, nt);
    gl_cross(T, B, tb);
    const float det = gl_dot(T, bn);
    float y[3] = {__fdiv_rn(gl_dot(m, bn), det), __fdiv_rn(gl_dot(m, nt), det), __fdiv_rn(gl_dot(m, tb), det)};
    if (det != 0.f && isfinite(det) && gl_finite3(y) && gl_normalize(y) && gl_finite3(y))
      for (int q = 0; q < 3; ++q) x[q] = y[q];
  }
  unsigned char* px = img + 5 * size_t(L);
  for (int q = 0; q < 3; ++q) px[q] = gl_encode(x[q]);
}

__global__ void __launch_bounds__(256) metal_rough_kernel(const unsigned char* __restrict__ metallic,
                                                          const unsigned char* __restrict__ roughness, long long n,
                                                          const unsigned char* __restrict__ lut_m, const unsigned char* __restrict__ lut_r,
                                                          unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  out[3 * i] = 255;
  out[3 * i + 1] = __ldg(lut_r + __ldg(roughness + i));
  out[3 * i + 2] = __ldg(lut_m + __ldg(metallic + i));
}

}  // namespace

extern "C" {

int nero_gltf_weld_count(const int* tris, const int* ft, int T, int V, const int* vt_ptr, const int* vt_tri, int* blk_cnt,
                         long long* blk_off, long long* total, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (V < 0 || T < 0 || V > 0x7fffffff - kWeldThreads || !total || (V > 0 && (!vt_ptr || !blk_cnt || !blk_off)) ||
      (V > 0 && T > 0 && (!tris || !ft || !vt_tri)))
    return NERO_ERR_ARG;
  if (V == 0) {
    NERO_CUDA_TRY(cudaMemsetAsync(total, 0, sizeof(long long), st));
    return NERO_OK;
  }
  const int nblk = (V + kWeldThreads - 1) / kWeldThreads;
  weld_count_kernel<<<nblk, kWeldThreads, 0, st>>>(tris, ft, V, vt_ptr, vt_tri, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nblk, st);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_gltf_weld_emit(const int* tris, const int* ft, int T, int V, const int* vt_ptr, const int* vt_tri, const long long* blk_off,
                        long long W, int* wv, int* wt, int* wf, void* stream) {
  if (V < 0 || T < 0 || V > 0x7fffffff - kWeldThreads || W < 0 || W > 3LL * T) return NERO_ERR_ARG;
  if (V == 0 || T == 0) return NERO_OK;
  if (!tris || !ft || !vt_ptr || !vt_tri || !blk_off || !wv || !wt || !wf) return NERO_ERR_ARG;
  weld_emit_kernel<<<(V + kWeldThreads - 1) / kWeldThreads, kWeldThreads, 0, (cudaStream_t)stream>>>(tris, ft, V, vt_ptr, vt_tri, blk_off,
                                                                                                      wv, wt, wf);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_gltf_tangents(const float* verts, const int* tris, const float* vt, const int* ft, const int* vt_ptr, const int* vt_tri,
                       const float* normals, const int* wv, const int* wt, int W, float* wnormal, float* wtangent, void* stream) {
  if (W < 0) return NERO_ERR_ARG;
  if (W == 0) return NERO_OK;
  if (!verts || !tris || !vt || !ft || !vt_ptr || !vt_tri || !normals || !wv || !wt || !wnormal || !wtangent) return NERO_ERR_ARG;
  tangents_kernel<<<(W + 127) / 128, 128, 0, (cudaStream_t)stream>>>(verts, tris, vt, ft, vt_ptr, vt_tri, normals, wv, wt, W, wnormal,
                                                                      wtangent);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_gltf_tangent_space(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* atlas,
                            const int* faces, const int* wf, const float* wnormal, const float* wtangent, const unsigned char* omap,
                            unsigned char* img, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (!owner || !img || width < 1 || height < 1) return NERO_ERR_ARG;
  const long long N = (long long)width * height;
  if (N > 0x7fffffffLL || n < 0 || n > N) return NERO_ERR_ARG;
  if (n > 0 && (!texel || !atlas || !faces || !wf || !wnormal || !wtangent || !omap)) return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(img, 0, size_t(N) * 5, st));
  if (n == 0) return NERO_OK;
  tangent_space_kernel<<<unsigned((n + 127) / 128), 128, 0, st>>>(owner, width, height, texel, n, atlas, faces, wf, wnormal, wtangent,
                                                                   omap, img);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_gltf_metal_rough(const unsigned char* metallic, const unsigned char* roughness, long long n, const unsigned char* lut_m,
                          const unsigned char* lut_r, unsigned char* out, void* stream) {
  if (n < 0 || (n > 0 && (!metallic || !roughness || !lut_m || !lut_r || !out))) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  metal_rough_kernel<<<unsigned((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(metallic, roughness, n, lut_m, lut_r, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
