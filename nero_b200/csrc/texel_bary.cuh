// The texel -> surface point map of the UV atlas, shared by the texture export (k_texmap.cu: raster and texel_emit), the
// normal-map bake (k_normalmap.cu) and the glTF export's tangent-space conversion (k_gltf.cu), so a bake point is the point
// the export stores in raster()['xyz'], bit for bit.
//
// uv is snapped to 1/256 texel (round-half-even of u * width * 256, exact in fp64); coverage uses exact int64 edge functions
// with the top-left rule for either winding; the barycentrics of a covered texel are w_i / area rounded once to fp32, and
// the point is ((b0 p0 + b1 p1) + b2 p2) with every fp32 operation rounded on its own.
#pragma once
#include "common.cuh"

namespace nero {

// uv of triangle t snapped to 1/256 texel
struct SnapTri {
  long long x[3], y[3];
  long long area;   // positive orientation after the sign s
  int s;
};

__device__ __forceinline__ SnapTri snap_tri(const float* __restrict__ vt, const int* __restrict__ ft, int t, int width, int height) {
  SnapTri q;
  for (int i = 0; i < 3; ++i) {
    const int k = __ldg(ft + 3 * t + i);
    q.x[i] = llrint(double(__ldg(vt + 2 * k)) * double(width) * 256.0);
    q.y[i] = llrint(double(__ldg(vt + 2 * k + 1)) * double(height) * 256.0);
  }
  const long long a = (q.x[1] - q.x[0]) * (q.y[2] - q.y[0]) - (q.y[1] - q.y[0]) * (q.x[2] - q.x[0]);
  q.s = a < 0 ? -1 : 1;
  q.area = a < 0 ? -a : a;
  return q;
}

// edge weights w[i] (edge opposite vertex i) at the texel centre (px, py) in 1/256 texel; true if the texel is covered
__device__ __forceinline__ bool tri_cover(const SnapTri& q, long long px, long long py, long long w[3]) {
  bool in = true;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int a = (i + 1) % 3, b = (i + 2) % 3;
    const long long dx = q.x[b] - q.x[a], dy = q.y[b] - q.y[a];
    w[i] = q.s * (dx * (py - q.y[a]) - dy * (px - q.x[a]));
    const long long sdx = q.s * dx, sdy = q.s * dy;
    const bool top_left = sdy < 0 || (sdy == 0 && sdx > 0);
    in = in && (w[i] > 0 || (w[i] == 0 && top_left));
  }
  return in;
}

// barycentrics b [3] of texel L (row-major in a width-wide atlas) owned by triangle t
__device__ __forceinline__ void texel_bary(const float* __restrict__ vt, const int* __restrict__ ft, int t, long long L, int width,
                                           int height, float b[3]) {
  const SnapTri q = snap_tri(vt, ft, t, width, height);
  const long long y = L / width, x = L - y * width;
  long long w[3];
  tri_cover(q, 256 * x + 128, 256 * y + 128, w);
#pragma unroll
  for (int i = 0; i < 3; ++i) b[i] = float(double(w[i]) / double(q.area));
}

// barycentrics b [3] and position p [3] of texel L owned by triangle t
__device__ __forceinline__ void texel_point(const float* __restrict__ vt, const int* __restrict__ ft, const float* __restrict__ verts,
                                            const int* __restrict__ faces, int t, long long L, int width, int height, float b[3],
                                            float p[3]) {
  texel_bary(vt, ft, t, L, width, height, b);
  const float* p0 = verts + 3 * size_t(__ldg(faces + 3 * t));
  const float* p1 = verts + 3 * size_t(__ldg(faces + 3 * t + 1));
  const float* p2 = verts + 3 * size_t(__ldg(faces + 3 * t + 2));
#pragma unroll
  for (int k = 0; k < 3; ++k)
    p[k] = __fadd_rn(__fadd_rn(__fmul_rn(b[0], __ldg(p0 + k)), __fmul_rn(b[1], __ldg(p1 + k))), __fmul_rn(b[2], __ldg(p2 + k)));
}

}  // namespace nero
