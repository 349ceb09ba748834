// Mesh clean-up and area-uniform surface sampling: the GPU replacement of the MeshLab clean-up and the CloudCompare sampling
// of the real-data shape protocol.  The protocol is stated in nero_b200/evaluate.py, the ABI in include/nero_meshpts.h.
//
//   areas        one thread per triangle: fp64 area from the fp32 vertices (uncontracted), crop test (crop.cuh) of its three
//                vertices.
//   components   union-find over vertex indices (union_find.cuh): hook the larger root to the smaller by CAS (finds halve
//                paths), then ceil(log2 V) + 1 rounds of pointer jumping, which flatten any tree of depth < V; label = root =
//                the smallest vertex index of the component, so the result does not depend on scheduling.
//   comp areas   one warp per component sums its triangles' areas in ascending triangle index (the order of a stable sort
//                by label); one block takes the maximum (exact) and marks the components at or above frac * max.
//   compaction   flags -> per-block counts -> one-block int64 scan -> emit in original order (compact.cuh).
//   cdf          one thread per 256-triangle chunk sums it sequentially; one thread prefixes the chunk sums; one thread per
//                triangle adds its chunk's offset.
//   sample       one thread per sample: counter-based hash, binary search of the cdf, barycentric point in fp64.
//
// Floating-point values are never combined by atomics, so every output is bit-identical from run to run.
#include "common.cuh"
#include "compact.cuh"
#include "crop.cuh"
#include "hash.cuh"
#include "union_find.cuh"
#include "../../include/nero_meshpts.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_MESHPTS_BLOCK;
constexpr int kChunk = NERO_MESHPTS_CHUNK;
constexpr int kSelectThreads = 1024;

__global__ void __launch_bounds__(kBlock) areas_kernel(const float* __restrict__ verts, int V, const int* __restrict__ tris, int T,
                                                       const Crop q, double* __restrict__ area, unsigned char* __restrict__ keep) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  int id[3];
  bool ok = true;
  for (int k = 0; k < 3; ++k) {
    id[k] = __ldg(tris + 3 * (size_t)t + k);
    ok = ok && id[k] >= 0 && id[k] < V;
  }
  double a = 0.0;
  if (ok) {
    double p[3][3];
    for (int k = 0; k < 3; ++k)
      for (int j = 0; j < 3; ++j) p[k][j] = double(__ldg(verts + 3 * (size_t)id[k] + j));
    const double e1x = __dsub_rn(p[1][0], p[0][0]), e1y = __dsub_rn(p[1][1], p[0][1]), e1z = __dsub_rn(p[1][2], p[0][2]);
    const double e2x = __dsub_rn(p[2][0], p[0][0]), e2y = __dsub_rn(p[2][1], p[0][1]), e2z = __dsub_rn(p[2][2], p[0][2]);
    const double cx = __dsub_rn(__dmul_rn(e1y, e2z), __dmul_rn(e1z, e2y));
    const double cy = __dsub_rn(__dmul_rn(e1z, e2x), __dmul_rn(e1x, e2z));
    const double cz = __dsub_rn(__dmul_rn(e1x, e2y), __dmul_rn(e1y, e2x));
    a = __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz))));
    for (int k = 0; k < 3; ++k) ok = ok && inside(q, p[k][0], p[k][1], p[k][2]);
  }
  area[t] = a;
  if (keep) keep[t] = ok ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ components
__global__ void __launch_bounds__(kBlock) uf_hook_kernel(const int* __restrict__ tris, int T, const unsigned char* __restrict__ keep,
                                                         int* parent) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T || !keep[t]) return;
  const int i0 = __ldg(tris + 3 * (size_t)t), i1 = __ldg(tris + 3 * (size_t)t + 1), i2 = __ldg(tris + 3 * (size_t)t + 2);
  uf_unite(parent, i0, i1);
  uf_unite(parent, i0, i2);
}

__global__ void __launch_bounds__(kBlock) uf_label_kernel(const int* __restrict__ tris, int T, const unsigned char* __restrict__ keep,
                                                          const int* __restrict__ parent, int V, int* __restrict__ tri_label) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  tri_label[t] = keep[t] ? parent[__ldg(tris + 3 * (size_t)t)] : V;
}

// ------------------------------------------------------------------------------------------------ component areas
// one warp per component: the lanes gather 32 areas at a time (the next 32 are in flight while these are added) and every
// lane adds them in order, so the sum is the sequential one
__global__ void __launch_bounds__(kBlock) comp_sum_kernel(const double* __restrict__ area, const long long* __restrict__ order,
                                                          const long long* __restrict__ ends, int m, double* __restrict__ comp_area) {
  const long long c = ((long long)blockIdx.x * kBlock + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= m) return;                    // uniform across the warp
  const long long b = c ? ends[c - 1] : 0, e = ends[c];
  double x = b + lane < e ? area[order[b + lane]] : 0.0;
  double s = 0.0;
  for (long long j0 = b; j0 < e; j0 += 32) {
    const long long jn = j0 + 32 + lane;
    const double xn = jn < e ? area[order[jn]] : 0.0;
    const int cnt = int(min(32LL, e - j0));
    for (int k = 0; k < cnt; ++k) {
      const double y = __shfl_sync(0xffffffffu, x, k);
      s = j0 == b && k == 0 ? y : __dadd_rn(s, y);
    }
    x = xn;
  }
  if (lane == 0) comp_area[c] = s;
}

__global__ void __launch_bounds__(kSelectThreads) comp_select_kernel(const double* __restrict__ comp_area, const int* __restrict__ comp_label,
                                                                     int m, double frac, unsigned char* __restrict__ root_keep) {
  __shared__ double s_max[kSelectThreads];
  double mx = 0.0;
  for (int c = threadIdx.x; c < m; c += kSelectThreads) mx = fmax(mx, comp_area[c]);
  s_max[threadIdx.x] = mx;
  __syncthreads();
  for (int w = kSelectThreads / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w) s_max[threadIdx.x] = fmax(s_max[threadIdx.x], s_max[threadIdx.x + w]);
    __syncthreads();
  }
  const double thr = __dmul_rn(frac, s_max[0]);
  for (int c = threadIdx.x; c < m; c += kSelectThreads) root_keep[comp_label[c]] = comp_area[c] >= thr ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ ordered compaction
__global__ void __launch_bounds__(kBlock) flag_kernel(const int* __restrict__ tris, int T, const unsigned char* __restrict__ keep,
                                                      const int* __restrict__ tri_label, const unsigned char* __restrict__ root_keep,
                                                      unsigned char* __restrict__ tri_flag, unsigned char* vert_flag) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  const bool f = keep[t] && root_keep[tri_label[t]];
  tri_flag[t] = f ? 1 : 0;
  if (f)
    for (int k = 0; k < 3; ++k) vert_flag[__ldg(tris + 3 * (size_t)t + k)] = 1;   // every writer stores 1
}

__global__ void __launch_bounds__(kBlock) count_kernel(const unsigned char* __restrict__ flag, int n, int* __restrict__ blk_cnt) {
  __shared__ int s_w[kBlock / 32];
  const int i = blockIdx.x * kBlock + threadIdx.x;
  int total;
  block_scan<kBlock>(i < n && flag[i] ? 1 : 0, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) vert_emit_kernel(const float* __restrict__ verts, int V, const unsigned char* __restrict__ flag,
                                                           const long long* __restrict__ blk_off, int* __restrict__ remap,
                                                           float* __restrict__ out) {
  __shared__ int s_w[kBlock / 32];
  const int v = blockIdx.x * kBlock + threadIdx.x;
  const bool f = v < V && flag[v];
  int total;
  const int r = block_scan<kBlock>(f ? 1 : 0, s_w, &total);
  if (!f) return;
  const long long pos = blk_off[blockIdx.x] + r;
  remap[v] = int(pos);
  for (int k = 0; k < 3; ++k) out[3 * pos + k] = __ldg(verts + 3 * (size_t)v + k);
}

__global__ void __launch_bounds__(kBlock) tri_emit_kernel(const int* __restrict__ tris, int T, const unsigned char* __restrict__ flag,
                                                          const long long* __restrict__ blk_off, const int* __restrict__ remap,
                                                          int* __restrict__ out) {
  __shared__ int s_w[kBlock / 32];
  const int t = blockIdx.x * kBlock + threadIdx.x;
  const bool f = t < T && flag[t];
  int total;
  const int r = block_scan<kBlock>(f ? 1 : 0, s_w, &total);
  if (!f) return;
  const long long pos = blk_off[blockIdx.x] + r;
  for (int k = 0; k < 3; ++k) out[3 * pos + k] = remap[__ldg(tris + 3 * (size_t)t + k)];
}

// ------------------------------------------------------------------------------------------------ cumulative areas
__global__ void __launch_bounds__(kBlock) cdf_chunk_kernel(const double* __restrict__ area, int T, double* __restrict__ chunk,
                                                          double* __restrict__ cdf) {
  const int c = blockIdx.x * kBlock + threadIdx.x;
  const long long t0 = (long long)c * kChunk;
  if (t0 >= T) return;
  const int t1 = int(min((long long)T, t0 + kChunk));
  double s = area[t0];
  cdf[t0] = s;
  for (int t = int(t0) + 1; t < t1; ++t) {
    s = __dadd_rn(s, area[t]);
    cdf[t] = s;
  }
  chunk[c] = s;
}

// one thread: chunk sums -> exclusive offsets, in chunk order
__global__ void cdf_offsets_kernel(double* __restrict__ chunk, int nchunk) {
  double run = 0.0;
  for (int c = 0; c < nchunk; ++c) {
    const double s = chunk[c];
    chunk[c] = run;
    run = __dadd_rn(run, s);
  }
}

__global__ void __launch_bounds__(kBlock) cdf_add_kernel(const double* __restrict__ chunk, int T, double* __restrict__ cdf) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  cdf[t] = __dadd_rn(chunk[t / kChunk], cdf[t]);
}

// ------------------------------------------------------------------------------------------------ sampling
__device__ __forceinline__ uint32_t mp_bits(uint32_t seed, unsigned long long i, uint32_t dim) {
  uint32_t h = rl_mix(seed * 0x9e3779b9u + 0x7f4a7c15u);
  h = rl_mix(h ^ uint32_t(i));
  h = rl_mix(h ^ uint32_t(i >> 32));
  return rl_mix(h ^ dim);
}

__global__ void __launch_bounds__(kBlock) sample_kernel(const float* __restrict__ verts, int V, const int* __restrict__ tris, int T,
                                                        const double* __restrict__ cdf, uint32_t seed, long long i0, long long n,
                                                        double* __restrict__ out) {
  const long long k = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (k >= n) return;
  const unsigned long long i = (unsigned long long)(i0 + k);
  const uint32_t h0 = mp_bits(seed, i, 0), h1 = mp_bits(seed, i, 1), h2 = mp_bits(seed, i, 2), h3 = mp_bits(seed, i, 3);
  const double u0 = __dmul_rn(__dadd_rn(__dmul_rn(double(h0 >> 5), 67108864.0), double(h1 >> 6)), 0x1p-53);
  const double r1 = __dmul_rn(double(h2), 0x1p-32), r2 = __dmul_rn(double(h3), 0x1p-32);
  const double target = __dmul_rn(u0, __ldg(cdf + T - 1));
  int lo = 0, hi = T - 1;                 // first t with cdf[t] > target; T - 1 if there is none
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(cdf + mid) > target) hi = mid; else lo = mid + 1;
  }
  const double s = __dsqrt_rn(r1);
  const double b[3] = {__dsub_rn(1.0, s), __dmul_rn(s, __dsub_rn(1.0, r2)), __dmul_rn(s, r2)};
  double p[3] = {0.0, 0.0, 0.0};
  for (int c = 0; c < 3; ++c) {
    const int v = __ldg(tris + 3 * (size_t)lo + c);
    if (v < 0 || v >= V) {             // only when nothing has area (the caller refuses that): never read out of bounds
      p[0] = p[1] = p[2] = __longlong_as_double(0x7ff8000000000000LL);
      break;
    }
    for (int j = 0; j < 3; ++j) {
      const double x = __dmul_rn(b[c], double(__ldg(verts + 3 * (size_t)v + j)));
      p[j] = c == 0 ? x : __dadd_rn(p[j], x);
    }
  }
  for (int j = 0; j < 3; ++j) out[3 * k + j] = p[j];
}

inline unsigned nblocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

}  // namespace

extern "C" {

int nero_meshpts_areas(const float* verts, int V, const int* tris, int T, const double* sphere, const double* box, double* area,
                       unsigned char* keep, void* stream) {
  if (!verts || !tris || !area || V < 1 || T < 1) return NERO_ERR_ARG;
  Crop q;
  if (!make_crop(sphere, box, q) || ((sphere || box) && !keep)) return NERO_ERR_ARG;
  areas_kernel<<<nblocks(T), kBlock, 0, (cudaStream_t)stream>>>(verts, V, tris, T, q, area, keep);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_components(const int* tris, int T, const unsigned char* keep, int V, int* parent, int* tri_label, void* stream) {
  if (!tris || !keep || !parent || !tri_label || V < 1 || T < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  uf_init(parent, V, s);
  uf_hook_kernel<<<nblocks(T), kBlock, 0, s>>>(tris, T, keep, parent);
  uf_flatten(parent, V, s);
  uf_label_kernel<<<nblocks(T), kBlock, 0, s>>>(tris, T, keep, parent, V, tri_label);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_component_areas(const double* area, const long long* order, const long long* ends, const int* comp_label, int m,
                                 double frac, double* comp_area, unsigned char* root_keep, void* stream) {
  if (!area || !order || !ends || !comp_label || !comp_area || !root_keep || m < 1 || !(frac >= 0.0 && frac <= 1.0)) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  comp_sum_kernel<<<nblocks(32LL * m), kBlock, 0, s>>>(area, order, ends, m, comp_area);
  comp_select_kernel<<<1, kSelectThreads, 0, s>>>(comp_area, comp_label, m, frac, root_keep);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_compact_count(const int* tris, int T, const unsigned char* keep, const int* tri_label, const unsigned char* root_keep,
                               int V, unsigned char* tri_flag, unsigned char* vert_flag, int* blk_cnt, long long* blk_off,
                               long long* totals, void* stream) {
  if (!tris || !keep || !tri_label || !root_keep || !tri_flag || !vert_flag || !blk_cnt || !blk_off || !totals || V < 1 || T < 1)
    return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int nbt = int(nblocks(T)), nbv = int(nblocks(V));
  NERO_CUDA_TRY(cudaMemsetAsync(vert_flag, 0, (size_t)V, s));
  flag_kernel<<<nbt, kBlock, 0, s>>>(tris, T, keep, tri_label, root_keep, tri_flag, vert_flag);
  count_kernel<<<nbt, kBlock, 0, s>>>(tri_flag, T, blk_cnt);
  count_kernel<<<nbv, kBlock, 0, s>>>(vert_flag, V, blk_cnt + nbt);
  block_offsets<1>(blk_cnt, blk_off, totals + 1, nbt, s);
  block_offsets<1>(blk_cnt + nbt, blk_off + nbt, totals, nbv, s);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_compact_emit(const float* verts, int V, const int* tris, int T, const unsigned char* tri_flag,
                              const unsigned char* vert_flag, const long long* blk_off, long long nv, long long nt, int* remap,
                              float* verts_out, int* tris_out, void* stream) {
  if (!verts || !tris || !tri_flag || !vert_flag || !blk_off || !remap || V < 1 || T < 1 || nv < 0 || nv > V || nt < 0 || nt > T)
    return NERO_ERR_ARG;
  if ((nv > 0 && !verts_out) || (nt > 0 && !tris_out)) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int nbt = int(nblocks(T));
  if (nv > 0) vert_emit_kernel<<<nblocks(V), kBlock, 0, s>>>(verts, V, vert_flag, blk_off + nbt, remap, verts_out);
  if (nt > 0) tri_emit_kernel<<<nbt, kBlock, 0, s>>>(tris, T, tri_flag, blk_off, remap, tris_out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_cdf(const double* area, int T, double* chunk, double* cdf, void* stream) {
  if (!area || !chunk || !cdf || T < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  const int nchunk = (T + kChunk - 1) / kChunk;
  cdf_chunk_kernel<<<nblocks(nchunk), kBlock, 0, s>>>(area, T, chunk, cdf);
  cdf_offsets_kernel<<<1, 1, 0, s>>>(chunk, nchunk);
  cdf_add_kernel<<<nblocks(T), kBlock, 0, s>>>(chunk, T, cdf);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_meshpts_sample(const float* verts, int V, const int* tris, int T, const double* cdf, unsigned int seed, long long i0,
                        long long n, double* out, void* stream) {
  if (!verts || !tris || !cdf || !out || V < 1 || T < 1 || i0 < 0 || n < 1) return NERO_ERR_ARG;
  if ((n + kBlock - 1) / kBlock > 0x7fffffffLL) return NERO_ERR_ARG;
  sample_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(verts, V, tris, T, cdf, seed, i0, n, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
