// What the dense (k_mcubes.cu) and the brick-wise (k_mcsparse.cu) marching cubes share beyond the case tables: the case
// index, the vertex interpolation and the block scans.  Both paths must produce the same bits, so the expressions live here
// once.  A corner is below iff u <= iso.
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

// exclusive prefix of x over the block in thread order; *total = block sum.  s_w: kMcbThreads/32 ints.
__device__ __forceinline__ int mcb_block_scan(int x, int* s_w, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int incl = x;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_w[wid] = incl;
  __syncthreads();
  int before = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < kMcbThreads / 32; ++w) {
    const int v = s_w[w];
    before += w < wid ? v : 0;
    tot += v;
  }
  __syncthreads();
  *total = tot;
  return before + incl - x;
}

__device__ __forceinline__ long long mcb_warp_incl(long long x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += v;
  }
  return x;
}

}  // namespace nero
