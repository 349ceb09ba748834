// Stack traversal of the BVH built by bvh_build_host (k_bvh.cu), shared by the stage-II tracer (bvh_trace_kernel) and the
// relighting path tracer (k_relight.cu).  Nodes are 32-byte records in depth-first order (left child = index + 1), read as
// two float4: (lo, right-or-first) and (hi, count); triangles are (v0, e1, e2) float4 triples in BVH order.
#pragma once
#include "common.cuh"

namespace nero {

struct BvhHit {
  int tri;          // BVH-order triangle index, -1 = no hit
  float t, u, v;    // ray parameter and the Moeller-Trumbore barycentrics of vertices 1 and 2
};

// kAnyHit = false: closest hit with t in (0, t_max).  kAnyHit = true: returns as soon as any triangle is hit with t in
// (0, t_max) (shadow rays); t, u, v are then those of that triangle.
template <bool kAnyHit>
__device__ __forceinline__ BvhHit bvh_traverse(const float4* __restrict__ n4, const float4* __restrict__ tris, float ox, float oy,
                                               float oz, float dx, float dy, float dz, float t_max) {
  const float ix = 1.0f / dx, iy = 1.0f / dy, iz = 1.0f / dz;
  BvhHit h;
  h.tri = -1; h.t = t_max; h.u = 0.f; h.v = 0.f;
  int stack[48];
  int sp = 0;
  int node = 0;
  while (true) {
    const float4 a = __ldg(n4 + 2 * node), b = __ldg(n4 + 2 * node + 1);
    // slab test against [0, best]
    float t0 = (a.x - ox) * ix, t1 = (b.x - ox) * ix;
    float tmin = fminf(t0, t1), tmax = fmaxf(t0, t1);
    t0 = (a.y - oy) * iy; t1 = (b.y - oy) * iy;
    tmin = fmaxf(tmin, fminf(t0, t1)); tmax = fminf(tmax, fmaxf(t0, t1));
    t0 = (a.z - oz) * iz; t1 = (b.z - oz) * iz;
    tmin = fmaxf(tmin, fminf(t0, t1)); tmax = fminf(tmax, fmaxf(t0, t1));
    // conservative margin: a hit computed in fp32 may sit a few ulps outside the box
    const bool overlap = (tmax >= fmaxf(tmin, 0.f) - 1e-6f * (1.0f + fabsf(tmax))) && (tmin <= h.t);
    int next = -1;
    if (overlap) {
      const int cnt = __float_as_int(b.w), first_or_right = __float_as_int(a.w);
      if (cnt > 0) {
        for (int k = 0; k < cnt; ++k) {
          const int ti = first_or_right + k;
          const float4 v0 = __ldg(tris + 3 * ti), e1 = __ldg(tris + 3 * ti + 1), e2 = __ldg(tris + 3 * ti + 2);
          // Moeller-Trumbore
          const float px = dy * e2.z - dz * e2.y, py = dz * e2.x - dx * e2.z, pz = dx * e2.y - dy * e2.x;
          const float det = e1.x * px + e1.y * py + e1.z * pz;
          if (fabsf(det) > 1e-12f) {
            const float inv = 1.0f / det;
            const float tx = ox - v0.x, ty = oy - v0.y, tz = oz - v0.z;
            const float u = (tx * px + ty * py + tz * pz) * inv;
            const float qx = ty * e1.z - tz * e1.y, qy = tz * e1.x - tx * e1.z, qz = tx * e1.y - ty * e1.x;
            const float v = (dx * qx + dy * qy + dz * qz) * inv;
            const float t = (e2.x * qx + e2.y * qy + e2.z * qz) * inv;
            if (u >= 0.f && v >= 0.f && u + v <= 1.f && t > 0.f && t < h.t) {
              h.t = t; h.tri = ti; h.u = u; h.v = v;
              if (kAnyHit) return h;
            }
          }
        }
      } else {
        stack[sp++] = first_or_right;   // right child later
        next = node + 1;                // left child now (depth-first layout)
      }
    }
    if (next < 0) {
      if (sp == 0) break;
      next = stack[--sp];
    }
    node = next;
  }
  return h;
}

}  // namespace nero
