// Brick-wise marching cubes on a narrow band of the grid (include/nero_mcsparse.h): the mesh of k_mcubes.cu from field values
// at the points of a list of B^3-cube bricks only, so that the work follows the surface instead of the volume.
//
//   coarse_points  one thread per coarse point (every B-th grid point and the last one per axis): its position, gathered from
//                  the three axis arrays.
//   seed           one thread per brick: the Lipschitz test on its 8 coarse corners -> flag.
//   compact        flags -> per-block counts -> one-block int64 scan -> emit in ascending order (appended to the brick list,
//                  brick -> list entry written to `slot`, flags cleared), with the ordered compaction of compact.cuh.
//   brick_points   one thread per point of a listed brick: (B+1)^3 rows per brick, the high-side apron included, clamped to
//                  the grid (a clamped row repeats a boundary point; its value is never read as a grid point of its own).
//   grow           one block per newly filled brick: a neighbour that is not listed is flagged when a grid edge in the
//                  shared plane of points changes side.  Cubes with a sign change are connected through cube faces that
//                  hold a sign-change edge, so following such faces from brick to brick reaches every cube of a surface
//                  sheet that touches a listed brick.
//   count / emit   one block per brick, its values in shared memory: each brick emits the vertices of the edges and the
//                  triangles of the cubes it owns, with int64 keys (3 L + a; 5 C + s) instead of positions in the output.
//                  Placement comes from scans, not atomics; the caller sorts by key, which gives the order of k_mcubes.cu.
//   lookup         edge key -> vertex id by binary search in the sorted vertex keys.
#include "common.cuh"
#include "compact.cuh"
#include "mc_common.cuh"
#include "../../include/nero_mcsparse.h"

namespace nero {
namespace {

constexpr int kMsTile = NERO_MCSPARSE_TILE;
constexpr int kMsSub = kMsTile / kMcbThreads;
constexpr int kMsMaxP = 17 * 17 * 17;
constexpr int kMsGrowThreads = 128;

struct MsGrid {
  int n[3];      // grid points per axis
  int nb[3];     // bricks per axis
  int B, B1, P;  // cubes per brick edge, points per brick edge, points per brick
  float iso;
};

bool ms_grid(int nx, int ny, int nz, int brick, float iso, MsGrid& g) {
  if (nx < 2 || ny < 2 || nz < 2 || (brick != 4 && brick != 8 && brick != 16)) return false;
  g.n[0] = nx; g.n[1] = ny; g.n[2] = nz;
  for (int a = 0; a < 3; ++a) g.nb[a] = (g.n[a] - 2) / brick + 1;
  if ((long long)g.nb[0] * g.nb[1] * g.nb[2] > 0x7fffffffLL) return false;
  g.B = brick; g.B1 = brick + 1; g.P = g.B1 * g.B1 * g.B1;
  g.iso = iso;
  return true;
}

__device__ __forceinline__ void ms_brick_origin(const MsGrid& g, int b, int* o) {
  const int bz = b % g.nb[2], r = b / g.nb[2];
  o[0] = (r / g.nb[1]) * g.B;
  o[1] = (r % g.nb[1]) * g.B;
  o[2] = bz * g.B;
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_coarse_points_kernel(const float* __restrict__ ax, const float* __restrict__ ay,
                                                                             const float* __restrict__ az, const MsGrid g,
                                                                             long long first, long long count, float* __restrict__ rows) {
  const long long r = (long long)blockIdx.x * kMcbThreads + threadIdx.x;
  if (r >= count) return;
  const long long c = first + r;
  const int cy = g.nb[1] + 1, cz = g.nb[2] + 1;
  const int k = int(c % cz);
  const long long q = c / cz;
  const int j = int(q % cy), i = int(q / cy);
  rows[3 * r] = __ldg(ax + min(i * g.B, g.n[0] - 1));
  rows[3 * r + 1] = __ldg(ay + min(j * g.B, g.n[1] - 1));
  rows[3 * r + 2] = __ldg(az + min(k * g.B, g.n[2] - 1));
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_seed_kernel(const float* __restrict__ cval, const unsigned char* __restrict__ cout,
                                                                    const MsGrid g, float margin, int nbricks,
                                                                    unsigned char* __restrict__ flag) {
  const int b = blockIdx.x * kMcbThreads + threadIdx.x;
  if (b >= nbricks) return;
  const int bz = b % g.nb[2], r = b / g.nb[2], by = r % g.nb[1], bx = r / g.nb[1];
  const long long cy = g.nb[1] + 1, cz = g.nb[2] + 1;
  float mn = INFINITY, mn_abs = INFINITY;
  int n_out = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const long long c = ((bx + (q & 1)) * cy + (by + (q >> 1 & 1))) * cz + (bz + (q >> 2 & 1));
    const float d = __ldg(cval + c) - g.iso;
    mn = fminf(mn, d);
    mn_abs = fminf(mn_abs, fabsf(d));
    if (cout) n_out += __ldg(cout + c) ? 1 : 0;
  }
  flag[b] = (mn_abs <= margin || (n_out > 0 && n_out < 8 && mn <= margin)) ? 1 : 0;
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_flag_count_kernel(const unsigned char* __restrict__ flag, long long n,
                                                                          int* __restrict__ blk_cnt) {
  __shared__ int s_w[kMcbThreads / 32];
  const long long base = (long long)blockIdx.x * kMsTile;
  int c = 0;
  for (int s = 0; s < kMsSub; ++s) {
    const long long i = base + s * kMcbThreads + threadIdx.x;
    c += i < n && flag[i] ? 1 : 0;
  }
  int total;
  block_scan<kMcbThreads>(c, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_flag_emit_kernel(unsigned char* __restrict__ flag, long long n,
                                                                         const long long* __restrict__ blk_off, long long base,
                                                                         int* __restrict__ list, int* __restrict__ slot) {
  __shared__ int s_w[kMcbThreads / 32];
  long long at = base + blk_off[blockIdx.x];
  const long long i0 = (long long)blockIdx.x * kMsTile;
  for (int s = 0; s < kMsSub; ++s) {
    const long long i = i0 + s * kMcbThreads + threadIdx.x;
    const int f = i < n && flag[i] ? 1 : 0;
    int total;
    const int off = block_scan<kMcbThreads>(f, s_w, &total);
    if (f) {
      list[at + off] = int(i);
      slot[i] = int(at + off);
      flag[i] = 0;
    }
    at += total;
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_brick_points_kernel(const float* __restrict__ ax, const float* __restrict__ ay,
                                                                            const float* __restrict__ az, const MsGrid g,
                                                                            const int* __restrict__ list, long long count,
                                                                            float* __restrict__ rows) {
  const long long r = (long long)blockIdx.x * kMcbThreads + threadIdx.x;
  if (r >= count * g.P) return;
  const long long j = r / g.P;
  const int l = int(r - j * g.P);
  int o[3];
  ms_brick_origin(g, __ldg(list + j), o);
  const int dz = l % g.B1, q = l / g.B1;
  rows[3 * r] = __ldg(ax + min(o[0] + q / g.B1, g.n[0] - 1));
  rows[3 * r + 1] = __ldg(ay + min(o[1] + q % g.B1, g.n[1] - 1));
  rows[3 * r + 2] = __ldg(az + min(o[2] + dz, g.n[2] - 1));
}

// the two faces of brick (bx, by, bz) across axis kA: strides sa (across the face), s1, s2 (in its plane)
template <int kA>
__device__ __forceinline__ void ms_grow_faces(const MsGrid& g, const float* u, const int* __restrict__ slot, int bx, int by, int bz,
                                              unsigned char* __restrict__ flag) {
  const int sx = g.B1 * g.B1, sy = g.B1;
  const int sa = kA == 0 ? sx : kA == 1 ? sy : 1, s1 = kA == 0 ? sy : kA == 1 ? 1 : sx, s2 = kA == 0 ? 1 : kA == 1 ? sx : sy;
  const int ba = kA == 0 ? bx : kA == 1 ? by : bz;
  for (int hi = 0; hi < 2; ++hi) {
    const int na = ba + (hi ? 1 : -1);
    if (na < 0 || na >= g.nb[kA]) continue;                 // uniform across the block, like the skip below
    const int nb = ((kA == 0 ? na : bx) * g.nb[1] + (kA == 1 ? na : by)) * g.nb[2] + (kA == 2 ? na : bz);
    if (slot[nb] >= 0) continue;
    const float* pl = u + (hi ? g.B : 0) * sa;
    bool any = false;
    for (int q = threadIdx.x; q < sx; q += kMsGrowThreads) {
      const int s = q / g.B1, t = q % g.B1;
      const float* p = pl + s * s1 + t * s2;
      const bool b0 = __ldg(p) <= g.iso;
      any |= s < g.B && (__ldg(p + s1) <= g.iso) != b0;
      any |= t < g.B && (__ldg(p + s2) <= g.iso) != b0;
    }
    if (__syncthreads_or(any) && threadIdx.x == 0) flag[nb] = 1;
  }
}

__global__ void __launch_bounds__(kMsGrowThreads) mcsparse_grow_kernel(const float* __restrict__ pool, const int* __restrict__ list,
                                                                       long long first, const int* __restrict__ slot, const MsGrid g,
                                                                       unsigned char* __restrict__ flag) {
  const long long j = first + blockIdx.x;
  const int b = list[j];
  const float* u = pool + j * g.P;
  const int bz = b % g.nb[2], r = b / g.nb[2], by = r % g.nb[1], bx = r / g.nb[1];
  ms_grow_faces<0>(g, u, slot, bx, by, bz, flag);
  ms_grow_faces<1>(g, u, slot, bx, by, bz, flag);
  ms_grow_faces<2>(g, u, slot, bx, by, bz, flag);
}

// The sign-change edges (bit a: along axis a) that local point l of the brick at origin o owns, and the case of the cube it
// owns (-1 if none); gp = its grid coordinates.  s_u: the brick's values.
__device__ __forceinline__ void ms_classify(const MsGrid& g, const float* s_u, const int* o, int l, int* gp, int& emask, int& cs,
                                            float* c) {
  const int d[3] = {l / (g.B1 * g.B1), l / g.B1 % g.B1, l % g.B1};
  bool own = true, e[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    gp[a] = o[a] + d[a];
    own = own && gp[a] < g.n[a] && (d[a] < g.B || gp[a] == g.n[a] - 1);
    e[a] = gp[a] < g.n[a] - 1;
  }
  emask = 0;
  cs = -1;
  if (!own) return;
  const int sx = g.B1 * g.B1, sy = g.B1;
  const float* p = s_u + l;
  c[0] = p[0];
  c[1] = e[0] ? p[sx] : 0.f;
  c[2] = e[1] ? p[sy] : 0.f;
  c[4] = e[2] ? p[1] : 0.f;
  const bool b0 = c[0] <= g.iso;
  emask = (e[0] && ((c[1] <= g.iso) != b0) ? 1 : 0) | (e[1] && ((c[2] <= g.iso) != b0) ? 2 : 0) | (e[2] && ((c[4] <= g.iso) != b0) ? 4 : 0);
  if (e[0] && e[1] && e[2]) {
    c[3] = p[sx + sy];
    c[5] = p[sx + 1];
    c[6] = p[sy + 1];
    c[7] = p[sx + sy + 1];
    cs = mc_case(c, g.iso);
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_count_kernel(const float* __restrict__ pool, const int* __restrict__ list,
                                                                     const MsGrid g, int* __restrict__ blk_cnt) {
  __shared__ float s_u[kMsMaxP];
  __shared__ unsigned char s_nt[256];
  __shared__ int s_w[kMcbThreads / 32];
  s_nt[threadIdx.x] = kMcNumTri[threadIdx.x];
  const float* u = pool + (long long)blockIdx.x * g.P;
  for (int l = threadIdx.x; l < g.P; l += kMcbThreads) s_u[l] = __ldg(u + l);
  __syncthreads();
  int o[3];
  ms_brick_origin(g, list[blockIdx.x], o);
  int x = 0;                                                // vertices in the low half, triangles in the high half
  for (int l = threadIdx.x; l < g.P; l += kMcbThreads) {
    int gp[3], em, cs;
    float c[8];
    ms_classify(g, s_u, o, l, gp, em, cs, c);
    x += __popc(em) + ((cs >= 0 ? s_nt[cs] : 0) << 16);
  }
  int total;
  block_scan<kMcbThreads>(x, s_w, &total);                  // at most 3 * 4913 vertices and 5 * 4096 triangles per brick
  if (threadIdx.x == 0) {
    blk_cnt[2 * blockIdx.x] = total & 0xffff;
    blk_cnt[2 * blockIdx.x + 1] = total >> 16;
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_emit_kernel(const float* __restrict__ pool, const int* __restrict__ list,
                                                                    const MsGrid g, const long long* __restrict__ blk_off,
                                                                    long long* __restrict__ vkey, float* __restrict__ vpos,
                                                                    long long* __restrict__ tkey, long long* __restrict__ tedge) {
  constexpr int W = 3 * kMcMaxTri;
  __shared__ float s_u[kMsMaxP];
  __shared__ signed char s_tri[256 * W];
  __shared__ unsigned char s_nt[256];
  __shared__ long long s_ekey[12];          // edge e of the cube at L has key 3 * L + s_ekey[e]
  __shared__ int s_w[kMcbThreads / 32];
  const long long sy = g.n[2], sx = (long long)g.n[1] * g.n[2];
  for (int q = threadIdx.x; q < 256 * W; q += kMcbThreads) s_tri[q] = (&kMcTri[0][0])[q];
  s_nt[threadIdx.x] = kMcNumTri[threadIdx.x];
  if (threadIdx.x < 12) {
    const int c0 = kMcEdgeCorner[threadIdx.x][0];
    s_ekey[threadIdx.x] = 3 * ((c0 & 1) * sx + (c0 >> 1 & 1) * sy + (c0 >> 2 & 1)) + (threadIdx.x >> 2);
  }
  const float* u = pool + (long long)blockIdx.x * g.P;
  for (int l = threadIdx.x; l < g.P; l += kMcbThreads) s_u[l] = __ldg(u + l);
  __syncthreads();
  int o[3];
  ms_brick_origin(g, list[blockIdx.x], o);
  long long vbase = blk_off[2 * blockIdx.x], tbase = blk_off[2 * blockIdx.x + 1];
  for (int l0 = 0; l0 < g.P; l0 += kMcbThreads) {
    const int l = l0 + threadIdx.x;
    int gp[3] = {0, 0, 0}, em = 0, cs = -1;
    float c[8];
    if (l < g.P) ms_classify(g, s_u, o, l, gp, em, cs, c);
    const int nt = cs >= 0 ? s_nt[cs] : 0;
    int total;
    const int off = block_scan<kMcbThreads>(__popc(em) + (nt << 16), s_w, &total);
    const long long L = gp[0] * sx + gp[1] * sy + gp[2];
    long long v = vbase + (off & 0xffff);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (em >> a & 1) {
        const float t = mc_interp(g.iso, c[0], c[1 << a]);
        vkey[v] = 3 * L + a;
        vpos[3 * v] = float(gp[0]) + (a == 0 ? t : 0.f);
        vpos[3 * v + 1] = float(gp[1]) + (a == 1 ? t : 0.f);
        vpos[3 * v + 2] = float(gp[2]) + (a == 2 ? t : 0.f);
        ++v;
      }
    }
    const long long t0 = tbase + (off >> 16);
    const signed char* tab = s_tri + (cs >= 0 ? cs : 0) * W;
    for (int s = 0; s < nt; ++s) {
      tkey[t0 + s] = kMcMaxTri * L + s;
#pragma unroll
      for (int q = 0; q < 3; ++q) tedge[3 * (t0 + s) + q] = 3 * L + s_ekey[tab[3 * s + q]];
    }
    vbase += total & 0xffff;
    tbase += total >> 16;
  }
}

__global__ void __launch_bounds__(kMcbThreads) mcsparse_lookup_kernel(const long long* __restrict__ sorted, long long n_sorted,
                                                                      const long long* __restrict__ key, long long n,
                                                                      int* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kMcbThreads + threadIdx.x;
  if (i >= n) return;
  const long long k = key[i];
  long long lo = 0, hi = n_sorted;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(sorted + mid) < k) lo = mid + 1; else hi = mid;
  }
  out[i] = lo < n_sorted && __ldg(sorted + lo) == k ? int(lo) : -1;
}

bool ms_blocks(long long work, int per_block, int& nblk) {
  const long long nb = (work + per_block - 1) / per_block;
  if (work < 0 || nb > 0x7fffffffLL) return false;
  nblk = int(nb);
  return true;
}

}  // namespace

extern "C" {

int nero_mcsparse_coarse_points(const float* ax, const float* ay, const float* az, int nx, int ny, int nz, int brick,
                                long long first, long long count, float* rows, void* stream) {
  MsGrid g;
  int nblk;
  if (!ms_grid(nx, ny, nz, brick, 0.f, g) || !ax || !ay || !az || !rows || first < 0 || count <= 0) return NERO_ERR_ARG;
  if (first + count > (long long)(g.nb[0] + 1) * (g.nb[1] + 1) * (g.nb[2] + 1) || !ms_blocks(count, kMcbThreads, nblk)) return NERO_ERR_ARG;
  mcsparse_coarse_points_kernel<<<nblk, kMcbThreads, 0, (cudaStream_t)stream>>>(ax, ay, az, g, first, count, rows);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_seed(const float* cval, const unsigned char* coutside, int nx, int ny, int nz, int brick, float iso, float margin,
                       unsigned char* flag, void* stream) {
  MsGrid g;
  if (!ms_grid(nx, ny, nz, brick, iso, g) || !cval || !flag || !(margin >= 0.f)) return NERO_ERR_ARG;
  const int nbricks = g.nb[0] * g.nb[1] * g.nb[2];
  mcsparse_seed_kernel<<<(nbricks + kMcbThreads - 1) / kMcbThreads, kMcbThreads, 0, (cudaStream_t)stream>>>(cval, coutside, g, margin,
                                                                                                          nbricks, flag);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_compact_count(const unsigned char* flag, long long n, int* blk_cnt, long long* blk_off, long long* total,
                                void* stream) {
  int nblk;
  if (!flag || n <= 0 || n > 0x7fffffffLL || !blk_cnt || !blk_off || !total || !ms_blocks(n, kMsTile, nblk)) return NERO_ERR_ARG;
  mcsparse_flag_count_kernel<<<nblk, kMcbThreads, 0, (cudaStream_t)stream>>>(flag, n, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nblk, (cudaStream_t)stream);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_compact_emit(unsigned char* flag, long long n, const long long* blk_off, long long base, int* list, int* slot,
                               void* stream) {
  int nblk;
  if (!flag || n <= 0 || n > 0x7fffffffLL || !blk_off || base < 0 || !list || !slot || !ms_blocks(n, kMsTile, nblk)) return NERO_ERR_ARG;
  mcsparse_flag_emit_kernel<<<nblk, kMcbThreads, 0, (cudaStream_t)stream>>>(flag, n, blk_off, base, list, slot);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_brick_points(const float* ax, const float* ay, const float* az, int nx, int ny, int nz, int brick, const int* list,
                               long long first, long long count, float* rows, void* stream) {
  MsGrid g;
  int nblk;
  if (!ms_grid(nx, ny, nz, brick, 0.f, g) || !ax || !ay || !az || !list || !rows || first < 0 || count <= 0) return NERO_ERR_ARG;
  if (count > 0x7fffffffLL || !ms_blocks(count * g.P, kMcbThreads, nblk)) return NERO_ERR_ARG;
  mcsparse_brick_points_kernel<<<nblk, kMcbThreads, 0, (cudaStream_t)stream>>>(ax, ay, az, g, list + first, count, rows);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_grow(const float* pool, const int* list, long long first, long long count, const int* slot, int nx, int ny, int nz,
                       int brick, float iso, unsigned char* flag, void* stream) {
  MsGrid g;
  if (!ms_grid(nx, ny, nz, brick, iso, g) || !pool || !list || !slot || !flag) return NERO_ERR_ARG;
  if (first < 0 || count <= 0 || count > 0x7fffffffLL) return NERO_ERR_ARG;
  mcsparse_grow_kernel<<<int(count), kMsGrowThreads, 0, (cudaStream_t)stream>>>(pool, list, first, slot, g, flag);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_count(const float* pool, const int* list, long long n_bricks, int nx, int ny, int nz, int brick, float iso,
                        int* blk_cnt, long long* blk_off, long long* totals, void* stream) {
  MsGrid g;
  if (!ms_grid(nx, ny, nz, brick, iso, g) || !pool || !list || !blk_cnt || !blk_off || !totals) return NERO_ERR_ARG;
  if (n_bricks <= 0 || n_bricks > 0x7fffffffLL) return NERO_ERR_ARG;
  mcsparse_count_kernel<<<int(n_bricks), kMcbThreads, 0, (cudaStream_t)stream>>>(pool, list, g, blk_cnt);
  block_offsets<2>(blk_cnt, blk_off, totals, n_bricks, (cudaStream_t)stream);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_emit(const float* pool, const int* list, long long n_bricks, int nx, int ny, int nz, int brick, float iso,
                       const long long* blk_off, long long* vkey, float* vpos, long long* tkey, long long* tedge, void* stream) {
  MsGrid g;
  if (!ms_grid(nx, ny, nz, brick, iso, g) || !pool || !list || !blk_off || !vkey || !vpos || !tkey || !tedge) return NERO_ERR_ARG;
  if (n_bricks <= 0 || n_bricks > 0x7fffffffLL) return NERO_ERR_ARG;
  mcsparse_emit_kernel<<<int(n_bricks), kMcbThreads, 0, (cudaStream_t)stream>>>(pool, list, g, blk_off, vkey, vpos, tkey, tedge);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_mcsparse_lookup(const long long* sorted, long long n_sorted, const long long* key, long long n, int* out, void* stream) {
  int nblk;
  if (!sorted || n_sorted <= 0 || n_sorted > 0x7fffffffLL || !key || n <= 0 || !out || !ms_blocks(n, kMcbThreads, nblk)) return NERO_ERR_ARG;
  mcsparse_lookup_kernel<<<nblk, kMcbThreads, 0, (cudaStream_t)stream>>>(sorted, n_sorted, key, n, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
