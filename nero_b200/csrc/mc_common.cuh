// What the dense (k_mcubes.cu) and the brick-wise (k_mcsparse.cu) marching cubes share beyond the case tables: the case
// index and the vertex interpolation.  Both paths must produce the same bits, so the expressions live here once.  A corner
// is below iff u <= iso.
#pragma once
#include "mc_tables.cuh"

namespace nero {

constexpr int kMcbThreads = 256;

// case index of a cube from its corner values c[0..7] (corner q = p + (q&1, q>>1&1, q>>2&1))
__device__ __forceinline__ int mc_case(const float* c, float iso) {
  int cs = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) cs |= (c[q] <= iso ? 1 : 0) << q;
  return cs;
}

// position of the vertex on the edge (p, p+e_a) as a fraction of the edge, u0 = u(p), u1 = u(p+e_a)
__device__ __forceinline__ float mc_interp(float iso, float u0, float u1) { return (iso - u0) / (u1 - u0); }

}  // namespace nero
