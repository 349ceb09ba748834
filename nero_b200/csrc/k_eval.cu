// Shape evaluation: the GPU replacement of the reference's eval_synthetic_shape.py / eval_real_shape.py (Chamfer distance of
// a mesh against ground-truth depth maps or a point cloud).  The protocol is stated once in nero_b200/evaluate.py.
//
//   depth_render  one thread per pixel: closest hit of the ray through the pixel centre (bvh_traverse.cuh), depth as the
//                 reference's nvdiffrast call produces it with w = 1 (screen-space linear): sum b_i z_i^2 / sum b_i z_i,
//                 0 on a miss or outside [near, far].
//   depth_points  ordered compaction of the pixels with lo < depth < hi over a stack of views, unprojected at integer pixel
//                 coordinates and moved to world space in fp64: count -> exclusive scan -> emit, as in k_mcubes.cu.
//   voxel_keys    Open3D's VoxelDownSample voxel index floor((p - min_bound) / voxel) in fp64, packed 21 bits per axis.
//   voxel_mean    per voxel (segments of the key-sorted order) the mean of its points, summed in input order in fp64.
//   nearest_dist  exact brute-force nearest distance: one thread per 4 queries, target tiles staged in shared memory,
//                 squared distance ((dx*dx + dy*dy) + dz*dz) with round-to-nearest, uncontracted operations.
//
// Nothing here uses atomics to place or combine values, so every output is bit-identical from run to run.
#include "bvh_traverse.cuh"
#include "common.cuh"

namespace nero {

namespace {

// ------------------------------------------------------------------------------------------------ depth maps
__global__ void __launch_bounds__(128) depth_render_kernel(const nero_depth_params q) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 8 + (threadIdx.x >> 4);
  if (x >= q.width || y >= q.height) return;
  const float* R = q.pose;
  // pinhole ray through the pixel centre (x + 1/2, y + 1/2): the point nvdiffrast samples for pixel (x, y)
  const float cx = (float(x) + 0.5f - q.K[2]) / q.K[0], cy = (float(y) + 0.5f - q.K[5]) / q.K[4];
  float d[3], o[3];
  for (int k = 0; k < 3; ++k) {
    d[k] = R[k] * cx + R[4 + k] * cy + R[8 + k];
    o[k] = -(R[k] * R[3] + R[4 + k] * R[7] + R[8 + k] * R[11]);
  }
  const BvhHit h = bvh_traverse<false>(reinterpret_cast<const float4*>(q.nodes), reinterpret_cast<const float4*>(q.tris), o[0], o[1],
                                       o[2], d[0], d[1], d[2], 1e30f);
  float depth = 0.f;
  if (h.tri >= 0) {
    // camera depths of the triangle's input vertices (not the BVH's v0 + e1 reconstruction)
    const int f = __ldg(q.tri_ids + h.tri);
    float z[3];
    for (int c = 0; c < 3; ++c) {
      const float* v = q.verts + 3 * size_t(__ldg(q.faces + 3 * f + c));
      z[c] = R[8] * __ldg(v) + R[9] * __ldg(v + 1) + R[10] * __ldg(v + 2) + R[11];
    }
    const float b0 = 1.0f - h.u - h.v;
    // screen-space barycentrics are b_i z_i / sum b_j z_j, so the linearly interpolated depth is sum b_i z_i^2 / sum b_i z_i
    const float num = b0 * z[0] * z[0] + h.u * z[1] * z[1] + h.v * z[2] * z[2];
    const float den = b0 * z[0] + h.u * z[1] + h.v * z[2];
    const float dz = num / den;
    if (dz >= q.near_z && dz <= q.far_z) depth = dz;   // clipping keeps depths in [near, far] only
  }
  q.depth[size_t(y) * q.width + x] = depth;
}

// ------------------------------------------------------------------------------------------------ ordered compaction
constexpr int kEvThreads = 256;
constexpr int kEvSub = 4;
constexpr int kEvTile = kEvThreads * kEvSub;   // keep in step with include/nero_b200.h (nblk)
constexpr int kEvScanThreads = 1024;

// exclusive prefix of x over the block in thread order; *total = block sum.  s_w: kEvThreads/32 ints.
__device__ __forceinline__ int ev_block_scan(int x, int* s_w, int* total) {
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
  for (int w = 0; w < kEvThreads / 32; ++w) {
    const int v = s_w[w];
    before += w < wid ? v : 0;
    tot += v;
  }
  __syncthreads();
  *total = tot;
  return before + incl - x;
}

__device__ __forceinline__ bool ev_keep(const float* depth, long long L, long long N, float lo, float hi) {
  if (L >= N) return false;
  const float d = __ldg(depth + L);
  return d > lo && d < hi;
}

__global__ void __launch_bounds__(kEvThreads) points_count_kernel(const float* __restrict__ depth, long long N, float lo, float hi,
                                                                  int* __restrict__ blk_cnt) {
  __shared__ int s_w[kEvThreads / 32];
  const long long base = (long long)blockIdx.x * kEvTile;
  int n = 0;
  for (int s = 0; s < kEvSub; ++s) n += ev_keep(depth, base + s * kEvThreads + threadIdx.x, N, lo, hi) ? 1 : 0;
  int total;
  ev_block_scan(n, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__device__ __forceinline__ long long ev_warp_incl(long long x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += v;
  }
  return x;
}

// one block: exclusive scan of the block counts in block order (chunks of 1024 with a 64-bit carry), and the total.
// k_mcubes.cu scans interleaved (vertex, triangle) pairs; this one scans a single count per block.
__global__ void __launch_bounds__(kEvScanThreads) points_scan_kernel(const int* __restrict__ blk_cnt, long long* __restrict__ blk_off,
                                                                     long long* __restrict__ total, int nblk) {
  __shared__ long long s_w[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long carry = 0;
  for (int c0 = 0; c0 < nblk; c0 += kEvScanThreads) {
    const int b = c0 + threadIdx.x;
    const long long v = b < nblk ? blk_cnt[b] : 0;
    const long long iv = ev_warp_incl(v, lane);
    if (lane == 31) s_w[wid] = iv;
    __syncthreads();
    if (wid == 0) s_w[lane] = ev_warp_incl(s_w[lane], lane);
    __syncthreads();
    if (b < nblk) blk_off[b] = carry + (wid ? s_w[wid - 1] : 0) + iv - v;
    carry += s_w[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) *total = carry;
}

// cams [n_views,16] fp64: camera -> world rotation (row-major 3x3), camera centre, fx, fy, cx, cy
__global__ void __launch_bounds__(kEvThreads) points_emit_kernel(const float* __restrict__ depth, long long N, long long hw, int width,
                                                                 float lo, float hi, const double* __restrict__ cams,
                                                                 const long long* __restrict__ blk_off, float* __restrict__ pts) {
  __shared__ float s_p[3 * kEvThreads];
  __shared__ int s_w[kEvThreads / 32];
  long long pbase = blk_off[blockIdx.x];
  const long long base = (long long)blockIdx.x * kEvTile;
  for (int s = 0; s < kEvSub; ++s) {
    const long long L = base + s * kEvThreads + threadIdx.x;
    const bool keep = ev_keep(depth, L, N, lo, hi);
    int total;
    const int off = ev_block_scan(keep ? 1 : 0, s_w, &total);
    if (total == 0) continue;              // uniform across the block
    if (keep) {
      const long long view = L / hw, r = L - view * hw;
      const long long py = r / width, px = r - py * width;
      const double* c = cams + 16 * view;
      const double dd = double(__ldg(depth + L));
      // mask_depth_to_pts: inv(K) (x d, y d, d) at the integer pixel coordinates (x, y)
      const double xc = (double(px) - c[14]) * dd / c[12], yc = (double(py) - c[15]) * dd / c[13];
#pragma unroll
      for (int k = 0; k < 3; ++k) s_p[3 * off + k] = float(c[3 * k] * xc + c[3 * k + 1] * yc + c[3 * k + 2] * dd + c[9 + k]);
    }
    __syncthreads();
    float* dst = pts + 3 * pbase;
    for (int q = threadIdx.x; q < 3 * total; q += kEvThreads) dst[q] = s_p[q];
    pbase += total;
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ voxel down-sampling
constexpr long long kVoxMax = 1LL << 21;

__global__ void voxel_keys_kernel(const double* __restrict__ pts, long long n, double mx, double my, double mz, double voxel,
                                  long long* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  // Open3D: ref_coord = (p - voxel_min_bound) / voxel_size, voxel_index = floor(ref_coord); fp64, no contraction possible
  const long long a = (long long)floor(__ddiv_rn(__dsub_rn(pts[3 * i], mx), voxel));
  const long long b = (long long)floor(__ddiv_rn(__dsub_rn(pts[3 * i + 1], my), voxel));
  const long long c = (long long)floor(__ddiv_rn(__dsub_rn(pts[3 * i + 2], mz), voxel));
  keys[i] = (a << 42) | (b << 21) | c;
}

// one thread per voxel: points order[ends[v-1] .. ends[v]) in input order; mean = (sum in that order) / count
__global__ void voxel_mean_kernel(const double* __restrict__ pts, const long long* __restrict__ order, const long long* __restrict__ ends,
                                  long long m, double* __restrict__ out) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= m) return;
  const long long e = ends[v], b = v ? ends[v - 1] : 0;
  double sx = 0.0, sy = 0.0, sz = 0.0;
  for (long long j = b; j < e; ++j) {
    const double* p = pts + 3 * order[j];
    sx = __dadd_rn(sx, p[0]);
    sy = __dadd_rn(sy, p[1]);
    sz = __dadd_rn(sz, p[2]);
  }
  const double cnt = double(e - b);
  out[3 * v] = __ddiv_rn(sx, cnt);
  out[3 * v + 1] = __ddiv_rn(sy, cnt);
  out[3 * v + 2] = __ddiv_rn(sz, cnt);
}

// ------------------------------------------------------------------------------------------------ nearest distance
constexpr int kNnThreads = 128;
constexpr int kNnQ = 4;                      // queries per thread: one shared-memory load feeds kNnQ distance evaluations
constexpr int kNnTile = 1024;                // targets per shared-memory tile (16 KB)

__global__ void __launch_bounds__(kNnThreads) nearest_kernel(const float* __restrict__ qp, long long n, const float* __restrict__ tp,
                                                             long long m, float* __restrict__ dist) {
  __shared__ float4 s_t[kNnTile];
  const long long q0 = (long long)blockIdx.x * (kNnThreads * kNnQ) + threadIdx.x;
  float qx[kNnQ], qy[kNnQ], qz[kNnQ], best[kNnQ];
#pragma unroll
  for (int k = 0; k < kNnQ; ++k) {
    const long long i = min(q0 + k * kNnThreads, n - 1);   // out-of-range slots repeat the last query and are not stored
    qx[k] = __ldg(qp + 3 * i); qy[k] = __ldg(qp + 3 * i + 1); qz[k] = __ldg(qp + 3 * i + 2);
    best[k] = __int_as_float(0x7f800000);
  }
  for (long long t0 = 0; t0 < m; t0 += kNnTile) {
    const int cnt = int(min((long long)kNnTile, m - t0));
    __syncthreads();
    for (int j = threadIdx.x; j < cnt; j += kNnThreads) {
      const float* p = tp + 3 * (t0 + j);
      s_t[j] = make_float4(__ldg(p), __ldg(p + 1), __ldg(p + 2), 0.f);
    }
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < cnt; ++j) {
      const float4 p = s_t[j];
#pragma unroll
      for (int k = 0; k < kNnQ; ++k) {
        const float dx = __fsub_rn(qx[k], p.x), dy = __fsub_rn(qy[k], p.y), dz = __fsub_rn(qz[k], p.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        best[k] = fminf(best[k], d2);
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kNnQ; ++k) {
    const long long i = q0 + k * kNnThreads;
    if (i < n) dist[i] = __fsqrt_rn(best[k]);
  }
}

bool ev_grid(int n_views, int height, int width, long long& N, int& nblk) {
  if (n_views < 1 || height < 1 || width < 1) return false;
  N = (long long)n_views * height * width;
  const long long nb = (N + kEvTile - 1) / kEvTile;
  if (nb > 0x7fffffffLL) return false;
  nblk = int(nb);
  return true;
}

}  // namespace

extern "C" {

int nero_depth_render(const nero_depth_params* p, void* stream) {
  if (!p) return NERO_ERR_ARG;
  const nero_depth_params& q = *p;
  if (!q.nodes || !q.tris || !q.tri_ids || !q.faces || !q.verts || !q.depth || q.width < 1 || q.height < 1) return NERO_ERR_ARG;
  // pinhole intrinsics only: zero skew, last row (0, 0, 1), non-zero focal lengths
  if (q.K[1] != 0.f || q.K[3] != 0.f || q.K[6] != 0.f || q.K[7] != 0.f || q.K[8] != 1.f || q.K[0] == 0.f || q.K[4] == 0.f)
    return NERO_ERR_ARG;
  if (!(q.near_z < q.far_z)) return NERO_ERR_ARG;
  const dim3 grid((q.width + 15) / 16, (q.height + 7) / 8);
  depth_render_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_depth_points_count(const float* depth, int n_views, int height, int width, float lo, float hi, int* blk_cnt,
                            long long* blk_off, long long* total, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  long long N;
  int nblk;
  if (!depth || !blk_cnt || !blk_off || !total || !ev_grid(n_views, height, width, N, nblk)) return NERO_ERR_ARG;
  points_count_kernel<<<nblk, kEvThreads, 0, st>>>(depth, N, lo, hi, blk_cnt);
  points_scan_kernel<<<1, kEvScanThreads, 0, st>>>(blk_cnt, blk_off, total, nblk);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_depth_points_emit(const float* depth, int n_views, int height, int width, float lo, float hi, const double* cams,
                           const long long* blk_off, long long n, float* pts, void* stream) {
  long long N;
  int nblk;
  if (!depth || !cams || !blk_off || n < 0 || !ev_grid(n_views, height, width, N, nblk) || n > N) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!pts) return NERO_ERR_ARG;
  points_emit_kernel<<<nblk, kEvThreads, 0, (cudaStream_t)stream>>>(depth, N, (long long)height * width, width, lo, hi, cams, blk_off, pts);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_voxel_keys(const double* pts, long long n, const double* bounds, double voxel, long long* keys, void* stream) {
  if (!bounds || n < 0 || !(voxel > 0.0) || (n > 0 && (!pts || !keys))) return NERO_ERR_ARG;
  for (int a = 0; a < 3; ++a) {
    // the largest index along each axis, computed as the kernel computes it, must fit 21 bits
    const double hi = floor((bounds[3 + a] - bounds[a]) / voxel);
    if (!(bounds[a] <= bounds[3 + a]) || !(hi < double(kVoxMax))) return NERO_ERR_ARG;
  }
  if (n == 0) return NERO_OK;
  voxel_keys_kernel<<<unsigned((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(pts, n, bounds[0], bounds[1], bounds[2], voxel, keys);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_voxel_mean(const double* pts, const long long* order, const long long* ends, long long m, double* out, void* stream) {
  if (m < 0 || (m > 0 && (!pts || !order || !ends || !out))) return NERO_ERR_ARG;
  if (m == 0) return NERO_OK;
  voxel_mean_kernel<<<unsigned((m + 255) / 256), 256, 0, (cudaStream_t)stream>>>(pts, order, ends, m, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_nearest_dist(const float* q, long long n, const float* t, long long m, float* dist, void* stream) {
  if (n < 0 || m < 1 || !t || (n > 0 && (!q || !dist))) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  const long long nb = (n + kNnThreads * kNnQ - 1) / (kNnThreads * kNnQ);
  if (nb > 0x7fffffffLL) return NERO_ERR_ARG;
  nearest_kernel<<<unsigned(nb), kNnThreads, 0, (cudaStream_t)stream>>>(q, n, t, m, dist);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
