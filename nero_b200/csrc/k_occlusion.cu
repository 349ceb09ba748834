// Ambient-occlusion bake: cosine-weighted visibility within a distance, counted per point with short any-hit rays.  The
// convention, the sampler and the byte are stated once in include/nero_occlusion.h.
//
//   texels  one thread per covered texel: the point, flat outward normal and key the count starts from, from the texel's own
//           point (texel_bary.cuh, as the texture export computes it) or from the normal bake's cage ray into a detail mesh.
//   count   one warp per row: lanes stride the N rays of the per-row rotated Hammersley set, each an any-hit ray on the
//           occluder BVH (bvh_traverse.cuh); the unoccluded rays are summed with __reduce_add_sync.
//   bytes   one thread per covered texel: round-half-up of 255 c / N in integers.
// Counts are integers and no thread shares state with another, so every output is bit-identical from run to run.
//
// The cage ray restates bake_kernel of k_normalmap.cu operation for operation (the same texel_point, blend, normalisation and
// closest-hit traversal).  It is not shared through a helper because moving it out of k_normalmap.cu changes the instruction
// schedule of nero_normalmap_bake.
#include "bvh_traverse.cuh"
#include "common.cuh"
#include "math_relight.cuh"
#include "texel_bary.cuh"
#include "../../include/nero_occlusion.h"

namespace nero {

namespace {

constexpr int kMaxRays = 65536;
constexpr int kCountThreads = 128;      // four rows per block

// s / |s| with |s| = sqrt((x x + y y) + z z), each operation rounded; a zero vector stays zero
__device__ __forceinline__ void occ_normalize(float s[3]) {
  const float l2 = __fadd_rn(__fadd_rn(__fmul_rn(s[0], s[0]), __fmul_rn(s[1], s[1])), __fmul_rn(s[2], s[2]));
  if (l2 > 0.f) {
    const float l = __fsqrt_rn(l2);
    for (int k = 0; k < 3; ++k) s[k] = __fdiv_rn(s[k], l);
  } else {
    s[0] = s[1] = s[2] = 0.f;
  }
}

// normalize(-cross(e1, e2)): the flat outward normal of the project's winding
__device__ __forceinline__ void occ_flat_normal(const float e1[3], const float e2[3], float n[3]) {
  n[0] = -__fsub_rn(__fmul_rn(e1[1], e2[2]), __fmul_rn(e1[2], e2[1]));
  n[1] = -__fsub_rn(__fmul_rn(e1[2], e2[0]), __fmul_rn(e1[0], e2[2]));
  n[2] = -__fsub_rn(__fmul_rn(e1[0], e2[1]), __fmul_rn(e1[1], e2[0]));
  occ_normalize(n);
}

__global__ void __launch_bounds__(128) occlusion_texels_kernel(const unsigned* __restrict__ owner, int width, int height,
                                                               const int* __restrict__ texel, long long n, const float* __restrict__ vt,
                                                               const int* __restrict__ ft, const float* __restrict__ verts,
                                                               const int* __restrict__ faces, const float* __restrict__ low_normals,
                                                               const float4* __restrict__ nodes, const float4* __restrict__ bvh_tris,
                                                               float cage_distance, float* __restrict__ points, float* __restrict__ normals,
                                                               unsigned* __restrict__ keys, unsigned char* __restrict__ hit,
                                                               float* __restrict__ surface, float* __restrict__ cage) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int L = __ldg(texel + i);
  const int t = int(__ldg(owner + L));
  float b[3], p[3], c[3] = {0.f, 0.f, 0.f}, q[3], ng[3] = {0.f, 0.f, 0.f};
  texel_point(vt, ft, verts, faces, t, L, width, height, b, p);
  bool got = true;
  for (int k = 0; k < 3; ++k) q[k] = p[k];
  if (nodes == nullptr) {
    const float* p0 = verts + 3 * size_t(__ldg(faces + 3 * t));
    const float* p1 = verts + 3 * size_t(__ldg(faces + 3 * t + 1));
    const float* p2 = verts + 3 * size_t(__ldg(faces + 3 * t + 2));
    float e1[3], e2[3];
    for (int k = 0; k < 3; ++k) {
      e1[k] = __fsub_rn(__ldg(p1 + k), __ldg(p0 + k));
      e2[k] = __fsub_rn(__ldg(p2 + k), __ldg(p0 + k));
    }
    occ_flat_normal(e1, e2, ng);
  } else {
    // the cage ray of k_normalmap.cu's bake_kernel
    const float* n0 = low_normals + 3 * size_t(__ldg(faces + 3 * t));
    const float* n1 = low_normals + 3 * size_t(__ldg(faces + 3 * t + 1));
    const float* n2 = low_normals + 3 * size_t(__ldg(faces + 3 * t + 2));
    for (int k = 0; k < 3; ++k)
      c[k] = __fadd_rn(__fadd_rn(__fmul_rn(b[0], __ldg(n0 + k)), __fmul_rn(b[1], __ldg(n1 + k))), __fmul_rn(b[2], __ldg(n2 + k)));
    occ_normalize(c);
    float o[3];
    for (int k = 0; k < 3; ++k) o[k] = __fadd_rn(p[k], __fmul_rn(cage_distance, c[k]));
    got = false;
    if (c[0] != 0.f || c[1] != 0.f || c[2] != 0.f) {
      const BvhHit h = bvh_traverse<false>(nodes, bvh_tris, o[0], o[1], o[2], -c[0], -c[1], -c[2], 2.0f * cage_distance);
      if (h.tri >= 0) {
        got = true;
        for (int k = 0; k < 3; ++k) q[k] = __fadd_rn(o[k], __fmul_rn(h.t, -c[k]));
        const float4 a = __ldg(bvh_tris + 3 * h.tri + 1), d = __ldg(bvh_tris + 3 * h.tri + 2);
        const float e1[3] = {a.x, a.y, a.z}, e2[3] = {d.x, d.y, d.z};
        occ_flat_normal(e1, e2, ng);
      }
    }
  }
  for (int k = 0; k < 3; ++k) {
    points[3 * i + k] = q[k];
    normals[3 * i + k] = ng[k];
  }
  keys[i] = unsigned(L);
  hit[i] = got ? 1 : 0;
  if (surface) for (int k = 0; k < 3; ++k) surface[3 * i + k] = p[k];
  if (cage) for (int k = 0; k < 3; ++k) cage[3 * i + k] = c[k];
}

__global__ void __launch_bounds__(kCountThreads) occlusion_count_kernel(const float* __restrict__ points, const float* __restrict__ normals,
                                                                        const unsigned* __restrict__ keys, long long n,
                                                                        const float4* __restrict__ nodes, const float4* __restrict__ bvh_tris,
                                                                        int rays, float distance, unsigned seed, int* __restrict__ counts) {
  const long long row = (long long)blockIdx.x * (kCountThreads / 32) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;   // whole warps leave together: the row is per warp
  float ng[3], o[3];
  for (int k = 0; k < 3; ++k) ng[k] = __ldg(normals + 3 * row + k);
  if (ng[0] == 0.f && ng[1] == 0.f && ng[2] == 0.f) {
    if (lane == 0) counts[row] = rays;
    return;
  }
  for (int k = 0; k < 3; ++k) o[k] = __fadd_rn(__ldg(points + 3 * row + k), __fmul_rn(kRelightEps, ng[k]));
  const unsigned key = keys ? __ldg(keys + row) : unsigned(row);
  const float xi1 = rl_uniform(seed, key, 0, 0, 0), xi2 = rl_uniform(seed, key, 0, 0, 1);
  const float two_n = float(2 * rays);
  unsigned clear = 0;
  for (int i = lane; i < rays; i += 32) {
    const float a = __fadd_rn(__fdiv_rn(float(2 * i + 1), two_n), xi1);
    const float b = __fadd_rn(__fmul_rn(float(__brev(unsigned(i)) >> 8), 5.9604644775390625e-8f), xi2);   // x 2^-24
    const float r1 = a < 1.0f ? a : __fsub_rn(a, 1.0f), r2 = b < 1.0f ? b : __fsub_rn(b, 1.0f);
    float l[3];
    rl_sample_diffuse(ng, r1, r2, l);
    const BvhHit h = bvh_traverse<true>(nodes, bvh_tris, o[0], o[1], o[2], l[0], l[1], l[2], distance);
    clear += h.tri < 0 ? 1u : 0u;
  }
  const unsigned total = __reduce_add_sync(0xffffffffu, clear);
  if (lane == 0) counts[row] = int(total);
}

__global__ void __launch_bounds__(256) occlusion_bytes_kernel(const int* __restrict__ texel, long long n, const int* __restrict__ counts,
                                                              int rays, unsigned char* __restrict__ img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long c = __ldg(counts + i);
  const unsigned char k = (unsigned char)((510 * c + rays) / (2 * (long long)rays));
  unsigned char* px = img + 5 * size_t(__ldg(texel + i));
  px[0] = px[1] = px[2] = k;
}

}  // namespace

extern "C" {

int nero_occlusion_points(const float* points, const float* normals, const unsigned int* keys, long long n, const float* nodes,
                          const float* bvh_tris, int rays, float distance, unsigned int seed, int* counts, void* stream) {
  if (n < 0 || rays < 1 || rays > kMaxRays || !(distance > 0.f) || !(distance < 3.0e38f)) return NERO_ERR_ARG;
  if (n > 0 && (!points || !normals || !nodes || !bvh_tris || !counts)) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  const long long rows_per_block = kCountThreads / 32;
  occlusion_count_kernel<<<unsigned((n + rows_per_block - 1) / rows_per_block), kCountThreads, 0, (cudaStream_t)stream>>>(
      points, normals, keys, n, reinterpret_cast<const float4*>(nodes), reinterpret_cast<const float4*>(bvh_tris), rays, distance, seed,
      counts);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_occlusion_texels(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* vt, const int* ft,
                          const float* verts, const int* faces, const float* low_normals, const float* nodes, const float* bvh_tris,
                          float cage_distance, float* points, float* normals, unsigned int* keys, unsigned char* hit, float* surface,
                          float* cage, void* stream) {
  if (!owner || width < 1 || height < 1) return NERO_ERR_ARG;
  const long long N = (long long)width * height;
  if (N > 0x7fffffffLL || n < 0 || n > N) return NERO_ERR_ARG;
  if (nodes && (!bvh_tris || !low_normals || !(cage_distance > 0.f) || !(cage_distance < 3.0e38f))) return NERO_ERR_ARG;
  if (n > 0 && (!texel || !vt || !ft || !verts || !faces || !points || !normals || !keys || !hit)) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  occlusion_texels_kernel<<<unsigned((n + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
      owner, width, height, texel, n, vt, ft, verts, faces, low_normals, reinterpret_cast<const float4*>(nodes),
      reinterpret_cast<const float4*>(bvh_tris), cage_distance, points, normals, keys, hit, surface, cage);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_occlusion_bytes(const int* texel, long long n, const int* counts, int rays, int width, int height, unsigned char* img,
                         void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  if (!img || width < 1 || height < 1 || rays < 1 || rays > kMaxRays) return NERO_ERR_ARG;
  const long long N = (long long)width * height;
  if (N > 0x7fffffffLL || n < 0 || n > N) return NERO_ERR_ARG;
  if (n > 0 && (!texel || !counts)) return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(img, 0, size_t(N) * 5, st));
  if (n == 0) return NERO_OK;
  occlusion_bytes_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(texel, n, counts, rays, img);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
