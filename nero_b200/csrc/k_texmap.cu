// UV texture-map export: the GPU replacement of the nvdiffrast raster, scipy morphology and sklearn kd-tree of the
// reference's extract_materials_texture_map.py.  The protocol is stated once in nero_b200/texmap.py.
//
//   raster     one thread per uv triangle over its texel bounding box: uv snapped to 1/256 texel, exact int64 edge functions
//              with the top-left rule (either winding; zero-area triangles own nothing).  owner = atomicMin(triangle id), so
//              the map is deterministic even where triangles overlap; cover counts them.
//   compact    ordered compaction of the covered texels in row-major order: count -> one-block scan -> emit
//              (compact.cuh).  emit interpolates the mesh positions in fp32 with the barycentrics of the same edge functions
//              (texel_bary.cuh, shared with the normal-map bake).
//   encode     linear_to_srgb in fp64 as numpy evaluates it (no contraction), x 255, truncated to uint8.
//   inpaint    search texels (covered, Manhattan distance <= 3 from an uncovered texel or the border), a 16x16 tile map of
//              them, then per uncovered texel a ring-by-ring scan of the radius-32 window for the nearest search texel.
//   downsample 2x, (a + b + c + d + 2) >> 2 per channel: OpenCV's INTER_LINEAR on an exact 2x uint8 shrink.
//
// No atomics combine values except the order-free atomicMin / count of the raster, so every output is bit-identical from
// run to run.
#include "common.cuh"
#include "compact.cuh"
#include "texel_bary.cuh"
#include "../../include/nero_texmap.h"

namespace nero {

namespace {

constexpr unsigned kNoOwner = 0xffffffffu;
constexpr int kInpaintR = 32;      // binary_dilation(iterations=32) with the cross: Manhattan distance <= 32
constexpr int kErodeR = 3;         // binary_erosion(iterations=3)
constexpr int kTile = 16;          // tile of the search-texel occupancy map

__device__ __forceinline__ long long floordiv(long long a, long long b) {
  const long long q = a / b;
  return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q;
}

__global__ void __launch_bounds__(128) raster_kernel(const float* __restrict__ vt, const int* __restrict__ ft, int T, int width, int height,
                                                     unsigned* __restrict__ owner, int* __restrict__ cover) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const SnapTri q = snap_tri(vt, ft, t, width, height);
  if (q.area == 0) return;
  const long long mnx = min(q.x[0], min(q.x[1], q.x[2])), mxx = max(q.x[0], max(q.x[1], q.x[2]));
  const long long mny = min(q.y[0], min(q.y[1], q.y[2])), mxy = max(q.y[0], max(q.y[1], q.y[2]));
  // texels whose centre 256 x + 128 lies in [min, max]
  const long long x0 = max(0LL, floordiv(mnx - 128 + 255, 256)), x1 = min((long long)width - 1, floordiv(mxx - 128, 256));
  const long long y0 = max(0LL, floordiv(mny - 128 + 255, 256)), y1 = min((long long)height - 1, floordiv(mxy - 128, 256));
  for (long long y = y0; y <= y1; ++y) {
    for (long long x = x0; x <= x1; ++x) {
      long long w[3];
      if (tri_cover(q, 256 * x + 128, 256 * y + 128, w)) {
        const long long i = y * width + x;
        atomicMin(owner + i, unsigned(t));
        atomicAdd(cover + i, 1);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ ordered compaction
constexpr int kTxThreads = 256;
constexpr int kTxSub = 4;
constexpr int kTxTile = kTxThreads * kTxSub;   // keep in step with include/nero_texmap.h (nblk)

__device__ __forceinline__ bool tx_covered(const unsigned* owner, long long L, long long N) {
  return L < N && __ldg(owner + L) != kNoOwner;
}

__global__ void __launch_bounds__(kTxThreads) texel_count_kernel(const unsigned* __restrict__ owner, long long N, int* __restrict__ blk_cnt) {
  __shared__ int s_w[kTxThreads / 32];
  const long long base = (long long)blockIdx.x * kTxTile;
  int n = 0;
  for (int s = 0; s < kTxSub; ++s) n += tx_covered(owner, base + s * kTxThreads + threadIdx.x, N) ? 1 : 0;
  int total;
  block_scan<kTxThreads>(n, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kTxThreads) texel_emit_kernel(const unsigned* __restrict__ owner, long long N, int width, int height,
                                                                const float* __restrict__ vt, const int* __restrict__ ft,
                                                                const float* __restrict__ verts, const int* __restrict__ faces,
                                                                const long long* __restrict__ blk_off, int* __restrict__ texel,
                                                                float* __restrict__ xyz) {
  __shared__ int s_w[kTxThreads / 32];
  long long pbase = blk_off[blockIdx.x];
  const long long base = (long long)blockIdx.x * kTxTile;
  for (int s = 0; s < kTxSub; ++s) {
    const long long L = base + s * kTxThreads + threadIdx.x;
    const bool keep = tx_covered(owner, L, N);
    int total;
    const int off = block_scan<kTxThreads>(keep ? 1 : 0, s_w, &total);
    if (keep) {
      float b[3], p[3];
      texel_point(vt, ft, verts, faces, int(__ldg(owner + L)), L, width, height, b, p);
      const long long o = pbase + off;
      texel[o] = int(L);
#pragma unroll
      for (int k = 0; k < 3; ++k) xyz[3 * o + k] = p[k];
    }
    pbase += total;
  }
}

// ------------------------------------------------------------------------------------------------ encode
// utils/raw_utils.py:11-15 on a float64 array, operation by operation (numpy rounds each one; nothing may be contracted)
__device__ __forceinline__ unsigned char encode_srgb8(float v) {
  const double x = double(v);
  double s;
  if (x <= 0.0031308) {
    s = __dmul_rn(323.0 / 25.0, x);
  } else {
    const double p = pow(fmax(1.1920928955078125e-07, x), 5.0 / 12.0);
    s = __ddiv_rn(__dsub_rn(__dmul_rn(211.0, p), 11.0), 200.0);
  }
  const double b = __dmul_rn(s, 255.0);
  return (unsigned char)(b <= 0.0 ? 0 : (b >= 255.0 ? 255 : int(b)));   // astype(uint8) truncates
}

__global__ void encode_kernel(const float* __restrict__ mat, const int* __restrict__ texel, long long n, unsigned char* __restrict__ img) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  unsigned char* o = img + 5 * size_t(__ldg(texel + i));
#pragma unroll
  for (int c = 0; c < 5; ++c) o[c] = encode_srgb8(__ldg(mat + 5 * i + c));
}

// ------------------------------------------------------------------------------------------------ inpaint
__device__ __forceinline__ bool is_covered(const unsigned* owner, int x, int y, int width, int height) {
  return x >= 0 && y >= 0 && x < width && y < height && __ldg(owner + size_t(y) * width + x) != kNoOwner;
}

// search = mask & ~binary_erosion(mask, 3): covered, and some texel within Manhattan distance 3 is uncovered or outside
__global__ void search_kernel(const unsigned* __restrict__ owner, int width, int height, unsigned char* __restrict__ search,
                              int* __restrict__ tile_occ, int tiles_x) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 16 + (threadIdx.x >> 4);
  if (x >= width || y >= height) return;
  bool edge = false;
  if (is_covered(owner, x, y, width, height)) {
    for (int dy = -kErodeR; dy <= kErodeR && !edge; ++dy) {
      const int r = kErodeR - abs(dy);
      for (int dx = -r; dx <= r; ++dx) edge = edge || !is_covered(owner, x + dx, y + dy, width, height);
    }
  }
  search[size_t(y) * width + x] = edge ? 1 : 0;
  if (edge) tile_occ[(y / kTile) * tiles_x + x / kTile] = 1;   // every writer stores the same value
}

__global__ void __launch_bounds__(256) inpaint_kernel(const unsigned char* __restrict__ img, const unsigned* __restrict__ owner, int width,
                                                      int height, const unsigned char* __restrict__ search, const int* __restrict__ tile_occ,
                                                      int tiles_x, int tiles_y, unsigned char* __restrict__ out, int* __restrict__ src) {
  const int x = blockIdx.x * 16 + (threadIdx.x & 15), y = blockIdx.y * 16 + (threadIdx.x >> 4);
  if (x >= width || y >= height) return;
  const size_t me = size_t(y) * width + x;
  int from = -1;
  if (__ldg(owner + me) == kNoOwner) {
    // a covered texel within Manhattan distance 32 implies a search texel within it (the first covered texel on a monotone
    // lattice path), so a window without search tiles holds no inpaint source: background texels leave here
    bool any = false;
    for (int ty = max(0, (y - kInpaintR) / kTile); ty <= min(tiles_y - 1, (y + kInpaintR) / kTile) && !any; ++ty)
      for (int tx = max(0, (x - kInpaintR) / kTile); tx <= min(tiles_x - 1, (x + kInpaintR) / kTile); ++tx)
        any = any || __ldg(tile_occ + ty * tiles_x + tx) != 0;
    if (any) {
      // rings of Chebyshev radius r: after ring r every texel with d^2 < (r+1)^2 and every one with Manhattan distance <= r has
      // been seen.  The nearest search texel lies within Euclidean distance 32 when any lies within Manhattan distance 32.
      bool near = false;
      int best = 0x7fffffff;
      long long bidx = -1;
      for (int r = 1; r <= kInpaintR; ++r) {
        for (int dy = -r; dy <= r; ++dy) {
          const int yy = y + dy;
          if (yy < 0 || yy >= height) continue;
          const int step = (dy == -r || dy == r) ? 1 : 2 * r;
          for (int dx = -r; dx <= r; dx += step) {
            const int xx = x + dx;
            if (xx < 0 || xx >= width) continue;
            const size_t j = size_t(yy) * width + xx;
            if (!__ldg(search + j)) continue;
            const int d2 = dx * dx + dy * dy;
            near = near || (abs(dx) + abs(dy) <= kInpaintR);
            if (d2 < best || (d2 == best && (long long)j < bidx)) {
              best = d2;
              bidx = (long long)j;
            }
          }
        }
        if (near && best < (r + 1) * (r + 1)) break;
      }
      if (near) from = int(bidx);
    }
  }
  const unsigned char* s = img + 5 * (from >= 0 ? size_t(from) : me);
#pragma unroll
  for (int c = 0; c < 5; ++c) out[5 * me + c] = __ldg(s + c);
  src[me] = from;
}

__global__ void downsample_kernel(const unsigned char* __restrict__ img, int width, int height, unsigned char* __restrict__ out) {
  const int w2 = width / 2, h2 = height / 2;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)w2 * h2 * 5) return;
  const int c = int(i % 5);
  const long long p = i / 5;
  const int y = int(p / w2), x = int(p - (long long)y * w2);
  const unsigned char* a = img + (size_t(2 * y) * width + 2 * x) * 5 + c;
  const size_t row = size_t(width) * 5;
  out[i] = (unsigned char)((unsigned(a[0]) + a[5] + a[row] + a[row + 5] + 2u) >> 2);
}

bool tx_grid(int width, int height, long long& N, int& nblk) {
  if (width < 1 || height < 1) return false;
  N = (long long)width * height;
  if (N > 0x7fffffffLL) return false;   // texel indices are int32
  nblk = int((N + kTxTile - 1) / kTxTile);
  return true;
}

}  // namespace

extern "C" {

int nero_tex_raster(const float* vt, const int* ft, int T, int width, int height, unsigned int* owner, int* cover, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  long long N;
  int nblk;
  if (T < 0 || !owner || !cover || (T > 0 && (!vt || !ft)) || !tx_grid(width, height, N, nblk)) return NERO_ERR_ARG;
  if ((long long)width * 256 >= (1LL << 30) || (long long)height * 256 >= (1LL << 30)) return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(owner, 0xff, size_t(N) * sizeof(unsigned), st));
  NERO_CUDA_TRY(cudaMemsetAsync(cover, 0, size_t(N) * sizeof(int), st));
  if (T == 0) return NERO_OK;
  raster_kernel<<<(T + 127) / 128, 128, 0, st>>>(vt, ft, T, width, height, owner, cover);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_tex_compact_count(const unsigned int* owner, int width, int height, int* blk_cnt, long long* blk_off, long long* total,
                           void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  long long N;
  int nblk;
  if (!owner || !blk_cnt || !blk_off || !total || !tx_grid(width, height, N, nblk)) return NERO_ERR_ARG;
  texel_count_kernel<<<nblk, kTxThreads, 0, st>>>(owner, N, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nblk, st);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_tex_compact_emit(const unsigned int* owner, int width, int height, const float* vt, const int* ft, const float* verts,
                          const int* faces, const long long* blk_off, long long n, int* texel, float* xyz, void* stream) {
  long long N;
  int nblk;
  if (!owner || !blk_off || n < 0 || !tx_grid(width, height, N, nblk) || n > N) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  if (!vt || !ft || !verts || !faces || !texel || !xyz) return NERO_ERR_ARG;
  texel_emit_kernel<<<nblk, kTxThreads, 0, (cudaStream_t)stream>>>(owner, N, width, height, vt, ft, verts, faces, blk_off, texel, xyz);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_tex_encode(const float* mat, const int* texel, long long n, int width, int height, unsigned char* img, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  long long N;
  int nblk;
  if (!img || n < 0 || !tx_grid(width, height, N, nblk) || n > N || (n > 0 && (!mat || !texel))) return NERO_ERR_ARG;
  NERO_CUDA_TRY(cudaMemsetAsync(img, 0, size_t(N) * 5, st));
  if (n == 0) return NERO_OK;
  encode_kernel<<<unsigned((n + 255) / 256), 256, 0, st>>>(mat, texel, n, img);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_tex_inpaint(const unsigned char* img, const unsigned int* owner, int width, int height, unsigned char* search, int* tile_occ,
                     unsigned char* out, int* src, void* stream) {
  const cudaStream_t st = (cudaStream_t)stream;
  long long N;
  int nblk;
  if (!img || !owner || !search || !tile_occ || !out || !src || !tx_grid(width, height, N, nblk)) return NERO_ERR_ARG;
  const int tiles_x = (width + kTile - 1) / kTile, tiles_y = (height + kTile - 1) / kTile;
  NERO_CUDA_TRY(cudaMemsetAsync(tile_occ, 0, size_t(tiles_x) * tiles_y * sizeof(int), st));
  const dim3 grid(tiles_x, tiles_y);
  search_kernel<<<grid, 256, 0, st>>>(owner, width, height, search, tile_occ, tiles_x);
  inpaint_kernel<<<grid, 256, 0, st>>>(img, owner, width, height, search, tile_occ, tiles_x, tiles_y, out, src);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_tex_downsample(const unsigned char* img, int width, int height, unsigned char* out, void* stream) {
  long long N;
  int nblk;
  if (!img || !out || !tx_grid(width, height, N, nblk) || (width & 1) || (height & 1)) return NERO_ERR_ARG;
  const long long m = (long long)(width / 2) * (height / 2) * 5;
  downsample_kernel<<<unsigned((m + 255) / 256), 256, 0, (cudaStream_t)stream>>>(img, width, height, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
