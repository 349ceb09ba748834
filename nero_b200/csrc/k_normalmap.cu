// Normal-map bake: the fine mesh's vertex normals, found by one cage ray per covered texel of the simplified mesh's atlas.
// The convention, the formulas and the byte encoding are stated once in include/nero_normalmap.h.
//
//   vertex_normals  one thread per vertex: the outward area vectors of its triangles summed in ascending triangle order
//                   (the CSR of nero_b200.simplify._vertex_triangles), then normalised; fp32 _rn throughout.
//   bake            one thread per covered texel: the texel's point and barycentrics (texel_bary.cuh, as the texture export
//                   computes them), the cage direction from the low mesh's vertex normals, one closest-hit ray on the detail
//                   BVH (bvh_traverse.cuh) and the interpolated detail normal, encoded to bytes.
// No atomics and no shared state between threads, so every output is bit-identical from run to run.
#include "bvh_traverse.cuh"
#include "common.cuh"
#include "texel_bary.cuh"
#include "../../include/nero_normalmap.h"

namespace nero {

namespace {

// s / |s| with |s| = sqrt((x x + y y) + z z), each operation rounded; a zero vector stays zero
__device__ __forceinline__ void nm_normalize(float s[3]) {
  const float l2 = __fadd_rn(__fadd_rn(__fmul_rn(s[0], s[0]), __fmul_rn(s[1], s[1])), __fmul_rn(s[2], s[2]));
  if (l2 > 0.f) {
    const float l = __fsqrt_rn(l2);
    for (int k = 0; k < 3; ++k) s[k] = __fdiv_rn(s[k], l);
  } else {
    s[0] = s[1] = s[2] = 0.f;
  }
}

// ((a0 x0 + a1 x1) + a2 x2) per component of three fp32 [*,3] rows
__device__ __forceinline__ void nm_blend(const float w[3], const float* r0, const float* r1, const float* r2, float out[3]) {
  for (int k = 0; k < 3; ++k)
    out[k] = __fadd_rn(__fadd_rn(__fmul_rn(w[0], __ldg(r0 + k)), __fmul_rn(w[1], __ldg(r1 + k))), __fmul_rn(w[2], __ldg(r2 + k)));
}

__device__ __forceinline__ unsigned char nm_encode(float n) {
  const float k = floorf(__fadd_rn(__fmul_rn(__fadd_rn(__fmul_rn(n, 0.5f), 0.5f), 255.0f), 0.5f));
  return (unsigned char)(k <= 0.f ? 0 : (k >= 255.f ? 255 : int(k)));
}

__global__ void __launch_bounds__(256) vertex_normals_kernel(const float* __restrict__ verts, int V, const int* __restrict__ tris,
                                                             const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                             float* __restrict__ normals) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  float s[3] = {0.f, 0.f, 0.f};
  for (int j = __ldg(vt_ptr + v), e = __ldg(vt_ptr + v + 1); j < e; ++j) {
    const int t = __ldg(vt_tri + j);
    const float* p0 = verts + 3 * size_t(__ldg(tris + 3 * t));
    const float* p1 = verts + 3 * size_t(__ldg(tris + 3 * t + 1));
    const float* p2 = verts + 3 * size_t(__ldg(tris + 3 * t + 2));
    float e1[3], e2[3];
    for (int k = 0; k < 3; ++k) {
      e1[k] = __fsub_rn(__ldg(p1 + k), __ldg(p0 + k));
      e2[k] = __fsub_rn(__ldg(p2 + k), __ldg(p0 + k));
    }
    // -cross(e1, e2): the outward area vector (twice the area)
    s[0] = __fadd_rn(s[0], -__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1])));
    s[1] = __fadd_rn(s[1], -__fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2])));
    s[2] = __fadd_rn(s[2], -__fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0])));
  }
  nm_normalize(s);
  for (int k = 0; k < 3; ++k) normals[3 * size_t(v) + k] = s[k];
}

__global__ void __launch_bounds__(128) bake_kernel(const unsigned* __restrict__ owner, int width, int height, const int* __restrict__ texel,
                                                   long long n, const float* __restrict__ vt, const int* __restrict__ ft,
                                                   const float* __restrict__ verts, const int* __restrict__ faces,
                                                   const float* __restrict__ low_normals, const float4* __restrict__ nodes,
                                                   const float4* __restrict__ bvh_tris, const int* __restrict__ tri_ids,
                                                   const int* __restrict__ detail_faces, const float* __restrict__ detail_normals,
                                                   float distance, unsigned char* __restrict__ img, unsigned char* __restrict__ hit,
                                                   float* __restrict__ point, float* __restrict__ cage, float* __restrict__ normal) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int L = __ldg(texel + i);
  const int t = int(__ldg(owner + L));
  float b[3], p[3], c[3], o[3];
  texel_point(vt, ft, verts, faces, t, L, width, height, b, p);
  nm_blend(b, low_normals + 3 * size_t(__ldg(faces + 3 * t)), low_normals + 3 * size_t(__ldg(faces + 3 * t + 1)),
           low_normals + 3 * size_t(__ldg(faces + 3 * t + 2)), c);
  nm_normalize(c);
  for (int k = 0; k < 3; ++k) o[k] = __fadd_rn(p[k], __fmul_rn(distance, c[k]));
  float nrm[3] = {c[0], c[1], c[2]};
  bool got = false;
  if (c[0] != 0.f || c[1] != 0.f || c[2] != 0.f) {
    const BvhHit h = bvh_traverse<false>(nodes, bvh_tris, o[0], o[1], o[2], -c[0], -c[1], -c[2], 2.0f * distance);
    if (h.tri >= 0) {
      got = true;
      const int f = __ldg(tri_ids + h.tri);
      const float w[3] = {__fsub_rn(__fsub_rn(1.0f, h.u), h.v), h.u, h.v};
      nm_blend(w, detail_normals + 3 * size_t(__ldg(detail_faces + 3 * f)), detail_normals + 3 * size_t(__ldg(detail_faces + 3 * f + 1)),
               detail_normals + 3 * size_t(__ldg(detail_faces + 3 * f + 2)), nrm);
      nm_normalize(nrm);
    }
  }
  unsigned char* px = img + 5 * size_t(L);
  for (int k = 0; k < 3; ++k) px[k] = nm_encode(nrm[k]);
  hit[i] = got ? 1 : 0;
  if (point) for (int k = 0; k < 3; ++k) point[3 * i + k] = p[k];
  if (cage) for (int k = 0; k < 3; ++k) cage[3 * i + k] = c[k];
  if (normal) for (int k = 0; k < 3; ++k) normal[3 * i + k] = nrm[k];
}

}  // namespace

extern "C" {

int nero_normalmap_vertex_normals(const float* verts, int V, const int* tris, int T, const int* vt_ptr, const int* vt_tri, float* normals,
                                  void* stream) {
  if (V < 0 || T < 0 || (V > 0 && (!vt_ptr || !normals)) || (V > 0 && T > 0 && (!verts || !tris || !vt_tri))) return NERO_ERR_ARG;
  if (V == 0) return NERO_OK;
  vertex_normals_kernel<<<(V + 255) / 256, 256, 0, (cudaStream_t)stream>>>(verts, V, tris, vt_ptr, vt_tri, normals);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_normalmap_bake(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* vt, const int* ft,
                        const float* verts, const int* faces, const float* low_normals, const float* nodes, const float* bvh_tris,
                        const int* tri_ids, const int* detail_faces, const float* detail_normals, float distance, unsigned char* img,
                        unsigned char* hit, float* point, float* cage, float* normal, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (!owner || !img || width < 1 || height < 1 || !(distance > 0.f) || !(distance < 3.0e38f)) return NERO_ERR_ARG;
  const long long N = (long long)width * height;
  if (N > 0x7fffffffLL || n < 0 || n > N) return NERO_ERR_ARG;
  if (n > 0 && (!texel || !vt || !ft || !verts || !faces || !low_normals || !nodes || !bvh_tris || !tri_ids || !detail_faces ||
                !detail_normals || !hit))
    return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(img, 0, size_t(N) * 5, st));
  if (n == 0) return NERO_OK;
  bake_kernel<<<unsigned((n + 127) / 128), 128, 0, st>>>(owner, width, height, texel, n, vt, ft, verts, faces, low_normals,
                                                          reinterpret_cast<const float4*>(nodes), reinterpret_cast<const float4*>(bvh_tris),
                                                          tri_ids, detail_faces, detail_normals, distance, img, hit, point, cage, normal);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
