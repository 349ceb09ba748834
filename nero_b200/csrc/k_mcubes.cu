// Marching cubes on a dense fp32 grid: the mcubes.marching_cubes call of extract_geometry (network/field.py:1110-1117) and
// extract_mesh.py, as an indexed mesh whose vertex and triangle order is fixed by the input alone.
//
//   u[i,j,k] at index point (i,j,k), C-contiguous [nx,ny,nz]; a corner is below iff u <= iso.
//   One vertex per grid edge (p, p+e_a) whose ends lie on different sides, at p + t e_a, t = (iso-u(p)) / (u(p+e_a)-u(p));
//   vertices are ordered by (linear index of p, a), triangles by the linear index of their cube, then by table order.
//
// Grid points are dealt to blocks in tiles of kMcbTile consecutive linear indices.  count: per-block vertex / triangle counts;
// scan: their exclusive scans in block order (compact.cuh's block_offsets over the two interleaved streams); verts / tris:
// each block recomputes its counts, scans them in point order, writes its rows into shared memory and copies them out as one
// contiguous range (a thread writing its own 12-byte rows would leave partly filled sectors).  No atomics decide where
// anything goes, so the output is bit-identical run to run.  The triangle pass finds the vertex ids of its cube's edges in
// `emap` (edge key 3*L + a -> vertex id), which the vertex pass fills at sign-change edges only.
#include "common.cuh"
#include "compact.cuh"
#include "mc_common.cuh"

namespace nero {
namespace {

constexpr int kMcbSub = 4;
constexpr int kMcbTile = kMcbThreads * kMcbSub;   // keep in step with include/nero_b200.h (nblk)

struct McGrid {
  const float* u;
  int nx, ny, nz;
  long long N, sx;   // sx = ny * nz
  float iso;
};

// The sign-change edges of point L (bit a: edge along axis a) and, if the cube based at L exists, its case index (else -1).
// Also returns the corner values c[0], c[1], c[2], c[4] (the far ends of the three edges) for the interpolation.
template <bool kCube>
__device__ __forceinline__ void mcb_classify(const McGrid& g, long long L, int& i, int& j, int& k, float* c, int& emask, int& cs) {
  const long long ii = L / g.sx;
  const long long r = L - ii * g.sx;
  i = int(ii);
  j = int(r / g.nz);
  k = int(r - (long long)j * g.nz);
  const bool hx = i < g.nx - 1, hy = j < g.ny - 1, hz = k < g.nz - 1;
  const float* p = g.u + L;
  const float iso = g.iso;
  c[0] = __ldg(p);
  c[1] = hx ? __ldg(p + g.sx) : 0.f;
  c[2] = hy ? __ldg(p + g.nz) : 0.f;
  c[4] = hz ? __ldg(p + 1) : 0.f;
  const bool b0 = c[0] <= iso;
  emask = (hx && ((c[1] <= iso) != b0) ? 1 : 0) | (hy && ((c[2] <= iso) != b0) ? 2 : 0) | (hz && ((c[4] <= iso) != b0) ? 4 : 0);
  cs = -1;
  if (kCube && hx && hy && hz) {
    c[3] = __ldg(p + g.sx + g.nz);
    c[5] = __ldg(p + g.sx + 1);
    c[6] = __ldg(p + g.nz + 1);
    c[7] = __ldg(p + g.sx + g.nz + 1);
    cs = mc_case(c, iso);
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcubes_count_kernel(const McGrid g, int* __restrict__ blk_cnt) {
  __shared__ unsigned char s_nt[256];
  __shared__ int s_w[2][kMcbThreads / 32];
  s_nt[threadIdx.x] = kMcNumTri[threadIdx.x];
  __syncthreads();
  const long long base = (long long)blockIdx.x * kMcbTile;
  int nv = 0, nt = 0;
  for (int s = 0; s < kMcbSub; ++s) {
    const long long L = base + s * kMcbThreads + threadIdx.x;
    if (L < g.N) {
      int i, j, k, em, cs;
      float c[8];
      mcb_classify<true>(g, L, i, j, k, c, em, cs);
      nv += __popc(em);
      nt += cs >= 0 ? s_nt[cs] : 0;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    nv += __shfl_xor_sync(0xffffffffu, nv, o);
    nt += __shfl_xor_sync(0xffffffffu, nt, o);
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) { s_w[0][wid] = nv; s_w[1][wid] = nt; }
  __syncthreads();
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int w = 0; w < kMcbThreads / 32; ++w) { a += s_w[0][w]; b += s_w[1][w]; }
    blk_cnt[2 * blockIdx.x] = a;
    blk_cnt[2 * blockIdx.x + 1] = b;
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcubes_verts_kernel(const McGrid g, const long long* __restrict__ blk_off,
                                                                   int* __restrict__ emap, float* __restrict__ verts) {
  __shared__ float s_v[3 * 3 * kMcbThreads];
  __shared__ int s_w[kMcbThreads / 32];
  long long vbase = blk_off[2 * blockIdx.x];
  const long long base = (long long)blockIdx.x * kMcbTile;
  for (int s = 0; s < kMcbSub; ++s) {
    const long long L = base + s * kMcbThreads + threadIdx.x;
    int i = 0, j = 0, k = 0, em = 0, cs;
    float c[8];
    if (L < g.N) mcb_classify<false>(g, L, i, j, k, c, em, cs);
    int total;
    int off = block_scan<kMcbThreads>(__popc(em), s_w, &total);
    if (total == 0) continue;              // uniform across the block
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (em >> a & 1) {
        const float t = mc_interp(g.iso, c[0], c[1 << a]);
        float* row = s_v + 3 * off;
        row[0] = float(i) + (a == 0 ? t : 0.f);
        row[1] = float(j) + (a == 1 ? t : 0.f);
        row[2] = float(k) + (a == 2 ? t : 0.f);
        emap[3 * L + a] = int(vbase + off);
        ++off;
      }
    }
    __syncthreads();
    float* dst = verts + 3 * vbase;
    for (int q = threadIdx.x; q < 3 * total; q += kMcbThreads) dst[q] = s_v[q];
    vbase += total;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcubes_tris_kernel(const McGrid g, const long long* __restrict__ blk_off,
                                                                  const int* __restrict__ emap, int* __restrict__ tris) {
  constexpr int W = 3 * kMcMaxTri;
  __shared__ signed char s_tri[256 * W];
  __shared__ unsigned char s_nt[256];
  __shared__ long long s_ekey[12];          // edge e of the cube at L has key 3 * L + s_ekey[e]
  __shared__ int s_t[W * kMcbThreads];
  __shared__ int s_w[kMcbThreads / 32];
  for (int q = threadIdx.x; q < 256 * W; q += kMcbThreads) s_tri[q] = (&kMcTri[0][0])[q];
  s_nt[threadIdx.x] = kMcNumTri[threadIdx.x];
  if (threadIdx.x < 12) {
    const int c0 = kMcEdgeCorner[threadIdx.x][0];
    s_ekey[threadIdx.x] = 3 * ((c0 & 1) * g.sx + (c0 >> 1 & 1) * g.nz + (c0 >> 2 & 1)) + (threadIdx.x >> 2);
  }
  __syncthreads();
  long long tbase = blk_off[2 * blockIdx.x + 1];
  const long long base = (long long)blockIdx.x * kMcbTile;
  for (int s = 0; s < kMcbSub; ++s) {
    const long long L = base + s * kMcbThreads + threadIdx.x;
    int i, j, k, em, cs = -1;
    float c[8];
    if (L < g.N) mcb_classify<true>(g, L, i, j, k, c, em, cs);
    const int nt = cs >= 0 ? s_nt[cs] : 0;
    int total;
    const int off = block_scan<kMcbThreads>(nt, s_w, &total);
    if (total == 0) continue;              // uniform across the block
    const signed char* tab = s_tri + (cs >= 0 ? cs : 0) * W;
    for (int q = 0; q < 3 * nt; ++q) s_t[3 * off + q] = emap[3 * L + s_ekey[tab[q]]];
    __syncthreads();
    int* dst = tris + 3 * tbase;
    for (int q = threadIdx.x; q < 3 * total; q += kMcbThreads) dst[q] = s_t[q];
    tbase += total;
    __syncthreads();
  }
}

bool mcb_grid(const float* u, int nx, int ny, int nz, float iso, McGrid& g, int& nblk) {
  if (!u || nx < 2 || ny < 2 || nz < 2) return false;
  g = McGrid{u, nx, ny, nz, (long long)nx * ny * nz, (long long)ny * nz, iso};
  const long long nb = (g.N + kMcbTile - 1) / kMcbTile;
  if (nb > 0x7fffffffLL) return false;
  nblk = int(nb);
  return true;
}

}  // namespace

extern "C" {

int nero_mcubes_count(const float* u, int nx, int ny, int nz, float iso, int* blk_cnt, long long* blk_off, long long* totals,
                      void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  McGrid g;
  int nblk;
  if (!mcb_grid(u, nx, ny, nz, iso, g, nblk) || !blk_cnt || !blk_off || !totals) return NERO_ERR_ARG;
  mcubes_count_kernel<<<nblk, kMcbThreads, 0, st>>>(g, blk_cnt);
  block_offsets<2>(blk_cnt, blk_off, totals, nblk, st);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcubes_emit(const float* u, int nx, int ny, int nz, float iso, const long long* blk_off, long long V, long long T, int* emap,
                     float* verts, int* tris, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  McGrid g;
  int nblk;
  if (!mcb_grid(u, nx, ny, nz, iso, g, nblk) || !blk_off) return NERO_ERR_ARG;
  if (V < 0 || T < 0 || V > 0x7fffffffLL || T > 0x7fffffffLL) return NERO_ERR_ARG;
  if (V > 0 && (!emap || !verts)) return NERO_ERR_ARG;
  if (T > 0 && (!emap || !tris || V == 0)) return NERO_ERR_ARG;
  if (V > 0) mcubes_verts_kernel<<<nblk, kMcbThreads, 0, st>>>(g, blk_off, emap, verts);
  if (T > 0) mcubes_tris_kernel<<<nblk, kMcbThreads, 0, st>>>(g, blk_off, emap, tris);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
