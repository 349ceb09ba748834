// Custom-object preparation: the GPU replacement of the CloudCompare steps of the custom-object workflow (crop the object
// out of COLMAP's fused cloud, fit the support plane).  The protocol is stated in nero_b200/objprep.py, the ABI in
// include/nero_objprep.h.
//
//   crop         one thread per point: the sphere / box test of crop.cuh in fp64.
//   compaction   flags -> per-block counts -> one-block int64 scan -> emit in original order (compact.cuh).
//   hypotheses   one thread per hypothesis: counter-based hash -> three kept points -> unit normal and offset in fp64.
//   counts       the hot loop, H x n point-plane tests.  A block keeps 8 points per thread in registers and walks a tile
//                of 256 planes staged in shared memory; each test is a warp ballot, its popcount goes to the lane that owns
//                the plane (lane = plane mod 32), the 8 warps are summed in shared memory and the block adds its int64
//                counts with one integer atomic per plane.  Integer sums, so the counts are exact in any order.
//   moments      fixed 4096-point blocks: per-thread sequential sums, a fixed shared-memory tree, then one thread per
//                sum adds the block partials in block order, so the refit sums are bit-reproducible.
//   above        one thread per point: height over the plane and the packed voxel key.
//   components   union-find over the occupied voxels (sorted keys, union_find.cuh): 13 forward neighbours found by binary
//                search, hooks to the smaller root by CAS, then ceil(log2 m) + 1 rounds of pointer jumping; label = smallest
//                voxel index.
//   select       integer atomics sum each component's points, one block takes the maximum and marks the kept voxels.
//
// Floating-point values are never combined by atomics, so every output is bit-identical from run to run.
#include <climits>
#include <cmath>

#include "common.cuh"
#include "compact.cuh"
#include "crop.cuh"
#include "hash.cuh"
#include "union_find.cuh"
#include "../../include/nero_objprep.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_OBJPREP_BLOCK;
constexpr int kChunk = NERO_OBJPREP_CHUNK;
constexpr int kMom = NERO_OBJPREP_MOMENTS;
constexpr int kPerThread = kChunk / kBlock;        // points per thread of a moments block
constexpr int kSelectThreads = 1024;
constexpr int kTile = 256;                         // planes per shared-memory tile of the counts
constexpr int kPts = 8;                            // points per thread per pass of the counts
constexpr int kCountBlocks = 2048;                 // grid cap of the counts (the result does not depend on it)
constexpr long long kVoxMax = 1LL << 21;
constexpr long long kNoKey = LLONG_MAX;

struct Plane {
  double n[4];
};

// signed distance ((nx x + ny y) + nz z) + d, uncontracted
__device__ __forceinline__ double plane_r(double nx, double ny, double nz, double d, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, x), __dmul_rn(ny, y)), __dmul_rn(nz, z)), d);
}

__global__ void __launch_bounds__(kBlock) crop_kernel(const double* __restrict__ pts, long long n, const Crop q,
                                                      unsigned char* __restrict__ keep) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  keep[i] = inside(q, pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ ordered compaction
__global__ void __launch_bounds__(kBlock) count_kernel(const unsigned char* __restrict__ flag, long long n, int* __restrict__ blk_cnt) {
  __shared__ int s_w[kBlock / 32];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  int total;
  block_scan<kBlock>(i < n && flag[i] ? 1 : 0, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) emit_kernel(const double* __restrict__ pts, const unsigned char* __restrict__ flag, long long n,
                                                      const long long* __restrict__ blk_off, int* __restrict__ idx,
                                                      double* __restrict__ out) {
  __shared__ int s_w[kBlock / 32];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  const bool f = i < n && flag[i];
  int total;
  const int r = block_scan<kBlock>(f ? 1 : 0, s_w, &total);
  if (!f) return;
  const long long pos = blk_off[blockIdx.x] + r;
  idx[pos] = int(i);
  if (out)
    for (int k = 0; k < 3; ++k) out[3 * pos + k] = pts[3 * i + k];
}

// ------------------------------------------------------------------------------------------------ hypotheses
__device__ __forceinline__ uint32_t op_bits(uint32_t seed, uint32_t k, uint32_t d) {
  return rl_mix(rl_mix(rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u) ^ k) ^ d);
}

__device__ __forceinline__ double sq3(double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
}

__global__ void __launch_bounds__(kBlock) hyp_kernel(const double* __restrict__ pts, long long n, int H, uint32_t seed,
                                                     double* __restrict__ planes, int* __restrict__ sample,
                                                     unsigned char* __restrict__ valid) {
  const int k = blockIdx.x * kBlock + threadIdx.x;
  if (k >= H) return;
  double p[3][3];
  for (int d = 0; d < 3; ++d) {
    const long long j = (long long)(((unsigned long long)op_bits(seed, uint32_t(k), uint32_t(d)) * (unsigned long long)n) >> 32);
    sample[3 * k + d] = int(j);
    for (int a = 0; a < 3; ++a) p[d][a] = pts[3 * j + a];
  }
  const double e1x = __dsub_rn(p[1][0], p[0][0]), e1y = __dsub_rn(p[1][1], p[0][1]), e1z = __dsub_rn(p[1][2], p[0][2]);
  const double e2x = __dsub_rn(p[2][0], p[0][0]), e2y = __dsub_rn(p[2][1], p[0][1]), e2z = __dsub_rn(p[2][2], p[0][2]);
  const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
  const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
  const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
  const double c2 = sq3(cx, cy, cz);
  const bool ok = c2 > __dmul_rn(1e-20, __dmul_rn(sq3(e1x, e1y, e1z), sq3(e2x, e2y, e2z)));
  double out[4];
  if (ok) {
    const double nrm = __dsqrt_rn(c2);
    out[0] = __ddiv_rn(cx, nrm); out[1] = __ddiv_rn(cy, nrm); out[2] = __ddiv_rn(cz, nrm);
    out[3] = -__dadd_rn(__dadd_rn(__dmul_rn(out[0], p[0][0]), __dmul_rn(out[1], p[0][1])), __dmul_rn(out[2], p[0][2]));
  } else {
    out[0] = out[1] = out[2] = out[3] = __longlong_as_double(0x7ff8000000000000LL);
  }
  for (int a = 0; a < 4; ++a) planes[4 * k + a] = out[a];
  valid[k] = ok ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ inlier counts
__global__ void __launch_bounds__(kBlock) counts_kernel(const double* __restrict__ pts, long long n, const double* __restrict__ planes,
                                                        int H, double tol, unsigned long long* __restrict__ counts) {
  __shared__ double4 s_pl[kTile];
  __shared__ int s_cnt[kBlock / 32][kTile];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const double qnan = __longlong_as_double(0x7ff8000000000000LL);
  for (int t0 = 0; t0 < H; t0 += kTile) {
    const int nt = min(kTile, H - t0);
    __syncthreads();                                  // the previous tile's s_pl / s_cnt are consumed
    for (int j = threadIdx.x; j < kTile; j += kBlock)
      s_pl[j] = j < nt ? make_double4(planes[4 * (t0 + j)], planes[4 * (t0 + j) + 1], planes[4 * (t0 + j) + 2], planes[4 * (t0 + j) + 3])
                       : make_double4(qnan, qnan, qnan, qnan);
    __syncthreads();
    int acc[kTile / 32];
#pragma unroll
    for (int jj = 0; jj < kTile / 32; ++jj) acc[jj] = 0;
    for (long long base = (long long)blockIdx.x * (kBlock * kPts); base < n; base += (long long)gridDim.x * (kBlock * kPts)) {
      double px[kPts], py[kPts], pz[kPts];
      bool in[kPts];
#pragma unroll
      for (int q = 0; q < kPts; ++q) {
        const long long i = base + q * kBlock + threadIdx.x;
        in[q] = i < n;
        px[q] = in[q] ? pts[3 * i] : 0.0;
        py[q] = in[q] ? pts[3 * i + 1] : 0.0;
        pz[q] = in[q] ? pts[3 * i + 2] : 0.0;
      }
#pragma unroll
      for (int jj = 0; jj < kTile / 32; ++jj) {
#pragma unroll 4
        for (int l = 0; l < 32; ++l) {
          const double4 pl = s_pl[jj * 32 + l];
          int c = 0;
#pragma unroll
          for (int q = 0; q < kPts; ++q)
            c += __popc(__ballot_sync(0xffffffffu, in[q] && fabs(plane_r(pl.x, pl.y, pl.z, pl.w, px[q], py[q], pz[q])) <= tol));
          acc[jj] += lane == l ? c : 0;
        }
      }
    }
#pragma unroll
    for (int jj = 0; jj < kTile / 32; ++jj) s_cnt[wid][jj * 32 + lane] = acc[jj];
    __syncthreads();
    for (int j = threadIdx.x; j < nt; j += kBlock) {
      long long s = 0;
#pragma unroll
      for (int w = 0; w < kBlock / 32; ++w) s += s_cnt[w][j];
      if (s) atomicAdd(counts + t0 + j, (unsigned long long)s);
    }
  }
}

// ------------------------------------------------------------------------------------------------ refit sums
__global__ void __launch_bounds__(kBlock) moments_kernel(const double* __restrict__ pts, long long n, const Plane pl, double tol,
                                                         double cx, double cy, double cz, double* __restrict__ partial) {
  __shared__ double s_m[kMom][kBlock];
  double s[kMom];
#pragma unroll
  for (int q = 0; q < kMom; ++q) s[q] = 0.0;
  for (int j = 0; j < kPerThread; ++j) {
    const long long i = (long long)blockIdx.x * kChunk + j * kBlock + threadIdx.x;
    if (i >= n) break;
    const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
    if (!(fabs(plane_r(pl.n[0], pl.n[1], pl.n[2], pl.n[3], x, y, z)) <= tol)) continue;
    const double dx = __dsub_rn(x, cx), dy = __dsub_rn(y, cy), dz = __dsub_rn(z, cz);
    const double t[kMom] = {1.0, dx, dy, dz, __dmul_rn(dx, dx), __dmul_rn(dx, dy), __dmul_rn(dx, dz), __dmul_rn(dy, dy), __dmul_rn(dy, dz),
                            __dmul_rn(dz, dz)};
#pragma unroll
    for (int q = 0; q < kMom; ++q) s[q] = __dadd_rn(s[q], t[q]);
  }
#pragma unroll
  for (int q = 0; q < kMom; ++q) s_m[q][threadIdx.x] = s[q];
  __syncthreads();
  for (int w = kBlock / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w)
#pragma unroll
      for (int q = 0; q < kMom; ++q) s_m[q][threadIdx.x] = __dadd_rn(s_m[q][threadIdx.x], s_m[q][threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x < kMom) partial[(long long)blockIdx.x * kMom + threadIdx.x] = s_m[threadIdx.x][0];
}

// one thread per sum: the block partials in block order
__global__ void moments_finish_kernel(const double* __restrict__ partial, int nblk, double* __restrict__ out) {
  const int q = threadIdx.x;
  if (q >= kMom) return;
  double s = partial[q];
  for (int b = 1; b < nblk; ++b) s = __dadd_rn(s, partial[(long long)b * kMom + q]);
  out[q] = s;
}

// ------------------------------------------------------------------------------------------------ object isolation
__global__ void __launch_bounds__(kBlock) above_kernel(const double* __restrict__ pts, long long n, const unsigned char* __restrict__ keep,
                                                       const Plane pl, double above, double ox, double oy, double oz, double voxel,
                                                       unsigned char* __restrict__ flag, long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const double x = pts[3 * i], y = pts[3 * i + 1], z = pts[3 * i + 2];
  const bool f = keep[i] && plane_r(pl.n[0], pl.n[1], pl.n[2], pl.n[3], x, y, z) >= above;
  flag[i] = f ? 1 : 0;
  long long key = kNoKey;
  if (f) {
    const long long a = (long long)floor(__ddiv_rn(__dsub_rn(x, ox), voxel));
    const long long b = (long long)floor(__ddiv_rn(__dsub_rn(y, oy), voxel));
    const long long c = (long long)floor(__ddiv_rn(__dsub_rn(z, oz), voxel));
    key = (a << 42) | (b << 21) | c;
  }
  keys[i] = key;
}

// index of key in the ascending ukeys[lo, hi), or -1
__device__ __forceinline__ long long find_key(const long long* __restrict__ ukeys, long long lo, long long hi, long long key) {
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    const long long v = ukeys[mid];
    if (v == key) return mid;
    if (v < key) lo = mid + 1; else hi = mid;
  }
  return -1;
}

// the 13 neighbours (da, db, dc) > (0, 0, 0) in lexicographic order have the larger packed keys, so they lie after v
__global__ void __launch_bounds__(kBlock) vox_hook_kernel(const long long* __restrict__ ukeys, long long m, int* parent) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v >= m) return;
  const long long key = ukeys[v];
  const long long a = key >> 42, b = (key >> 21) & (kVoxMax - 1), c = key & (kVoxMax - 1);
  for (int o = 14; o < 27; ++o) {                     // o = 9 (da + 1) + 3 (db + 1) + (dc + 1); 13 is (0, 0, 0)
    const long long na = a + o / 9 - 1, nb = b + (o / 3) % 3 - 1, nc = c + o % 3 - 1;
    if (na < 0 || na >= kVoxMax || nb < 0 || nb >= kVoxMax || nc < 0 || nc >= kVoxMax) continue;
    const long long u = find_key(ukeys, v + 1, m, (na << 42) | (nb << 21) | nc);
    if (u >= 0) uf_unite(parent, int(v), int(u));
  }
}

__global__ void __launch_bounds__(kBlock) copy_label_kernel(const int* __restrict__ parent, long long m, int* __restrict__ label) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v < m) label[v] = parent[v];
}

__global__ void __launch_bounds__(kBlock) comp_count_kernel(const int* __restrict__ label, const long long* __restrict__ vcount, long long m,
                                                            unsigned long long* __restrict__ comp_count) {
  const long long v = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (v < m) atomicAdd(comp_count + label[v], (unsigned long long)vcount[v]);
}

__global__ void __launch_bounds__(kSelectThreads) comp_select_kernel(const int* __restrict__ label, const long long* __restrict__ comp_count,
                                                                     long long m, double frac, unsigned char* __restrict__ voxel_keep) {
  __shared__ long long s_max[kSelectThreads];
  long long mx = 0;
  for (long long v = threadIdx.x; v < m; v += kSelectThreads) mx = max(mx, comp_count[v]);
  s_max[threadIdx.x] = mx;
  __syncthreads();
  for (int w = kSelectThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s_max[threadIdx.x] = max(s_max[threadIdx.x], s_max[threadIdx.x + w]);
    __syncthreads();
  }
  const double thr = __dmul_rn(frac, double(s_max[0]));
  for (long long v = threadIdx.x; v < m; v += kSelectThreads) voxel_keep[v] = double(comp_count[label[v]]) >= thr ? 1 : 0;
}

__global__ void __launch_bounds__(kBlock) point_keep_kernel(const long long* __restrict__ keys, const unsigned char* __restrict__ flag,
                                                            long long n, const long long* __restrict__ ukeys, long long m,
                                                            const unsigned char* __restrict__ voxel_keep, unsigned char* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  unsigned char k = 0;
  if (flag[i]) {
    const long long v = find_key(ukeys, 0, m, keys[i]);
    k = v >= 0 ? voxel_keep[v] : 0;
  }
  out[i] = k;
}

inline unsigned nblocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

bool finite_n(const double* x, int k) {
  for (int a = 0; a < k; ++a)
    if (!std::isfinite(x[a])) return false;
  return true;
}

// a plane from the host: finite, with a unit normal to within 1e-6
bool plane_ok(const double* p) {
  if (!p || !finite_n(p, 4)) return false;
  const double nn = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
  return std::fabs(nn - 1.0) <= 1e-6;
}

constexpr long long kMaxN = 0x7fffffffLL;

}  // namespace

extern "C" {

int nero_objprep_crop(const double* pts, long long n, const double* sphere, const double* box, unsigned char* keep, void* stream) {
  if (!pts || !keep || n < 1 || n > kMaxN) return NERO_ERR_ARG;
  Crop q;
  if (!make_crop(sphere, box, q)) return NERO_ERR_ARG;
  crop_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(pts, n, q, keep);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_compact_count(const unsigned char* flag, long long n, int* blk_cnt, long long* blk_off, long long* total, void* stream) {
  if (!flag || !blk_cnt || !blk_off || !total || n < 1 || n > kMaxN) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int nb = int(nblocks(n));
  count_kernel<<<nb, kBlock, 0, s>>>(flag, n, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nb, s);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_compact_emit(const double* pts, const unsigned char* flag, long long n, const long long* blk_off, long long m, int* idx,
                              double* out, void* stream) {
  if (!flag || !blk_off || n < 1 || n > kMaxN || m < 0 || m > n || (m > 0 && !idx) || (out && !pts)) return NERO_ERR_ARG;
  if (m > 0) emit_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(pts, flag, n, blk_off, idx, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_hypotheses(const double* pts, long long n, int H, unsigned int seed, double* planes, int* sample, unsigned char* valid,
                            void* stream) {
  if (!pts || !planes || !sample || !valid || n < 3 || n > kMaxN || H < 1) return NERO_ERR_ARG;
  hyp_kernel<<<nblocks(H), kBlock, 0, (cudaStream_t)stream>>>(pts, n, H, seed, planes, sample, valid);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_counts(const double* pts, long long n, const double* planes, int H, double tol, long long* counts, void* stream) {
  if (!pts || !planes || !counts || n < 1 || n > kMaxN || H < 1 || !(tol >= 0.0) || !std::isfinite(tol)) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  NERO_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(long long) * (size_t)H, s));
  const long long chunks = (n + kBlock * kPts - 1) / (kBlock * kPts);
  counts_kernel<<<unsigned(chunks < kCountBlocks ? chunks : kCountBlocks), kBlock, 0, s>>>(pts, n, planes, H, tol,
                                                                                           (unsigned long long*)counts);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_moments(const double* pts, long long n, const double* plane, double tol, const double* center, double* partial, double* out,
                         void* stream) {
  if (!pts || !partial || !out || n < 1 || n > kMaxN || !plane_ok(plane) || !(tol >= 0.0) || !std::isfinite(tol) || !center ||
      !finite_n(center, 3))
    return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int nblk = int((n + kChunk - 1) / kChunk);
  Plane pl;
  for (int a = 0; a < 4; ++a) pl.n[a] = plane[a];
  moments_kernel<<<nblk, kBlock, 0, s>>>(pts, n, pl, tol, center[0], center[1], center[2], partial);
  moments_finish_kernel<<<1, 32, 0, s>>>(partial, nblk, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_above(const double* pts, long long n, const unsigned char* keep, const double* plane, double above, const double* origin,
                       double voxel, unsigned char* flag, long long* keys, void* stream) {
  if (!pts || !keep || !flag || !keys || n < 1 || n > kMaxN || !plane_ok(plane) || !std::isfinite(above) || !origin || !finite_n(origin, 3) ||
      !(voxel > 0.0) || !std::isfinite(voxel))
    return NERO_ERR_ARG;
  Plane pl;
  for (int a = 0; a < 4; ++a) pl.n[a] = plane[a];
  above_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(pts, n, keep, pl, above, origin[0], origin[1], origin[2], voxel, flag, keys);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_voxel_components(const long long* ukeys, long long m, int* parent, int* label, void* stream) {
  if (!ukeys || !parent || !label || m < 1 || m > kMaxN) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  uf_init(parent, m, s);
  vox_hook_kernel<<<nblocks(m), kBlock, 0, s>>>(ukeys, m, parent);
  uf_flatten(parent, m, s);
  copy_label_kernel<<<nblocks(m), kBlock, 0, s>>>(parent, m, label);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_component_select(const int* label, const long long* vcount, long long m, double frac, long long* comp_count,
                                  unsigned char* voxel_keep, void* stream) {
  if (!label || !vcount || !comp_count || !voxel_keep || m < 1 || m > kMaxN || !(frac >= 0.0 && frac <= 1.0)) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  NERO_CUDA_TRY(cudaMemsetAsync(comp_count, 0, sizeof(long long) * (size_t)m, s));
  comp_count_kernel<<<nblocks(m), kBlock, 0, s>>>(label, vcount, m, (unsigned long long*)comp_count);
  comp_select_kernel<<<1, kSelectThreads, 0, s>>>(label, comp_count, m, frac, voxel_keep);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_objprep_point_keep(const long long* keys, const unsigned char* flag, long long n, const long long* ukeys, long long m,
                            const unsigned char* voxel_keep, unsigned char* out, void* stream) {
  if (!keys || !flag || !ukeys || !voxel_keep || !out || n < 1 || n > kMaxN || m < 1) return NERO_ERR_ARG;
  point_keep_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(keys, flag, n, ukeys, m, voxel_keep, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
