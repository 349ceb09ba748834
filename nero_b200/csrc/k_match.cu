// All-pair descriptor matching on the integer tensor cores: the GPU replacement of COLMAP's exhaustive_matcher (its
// matching half; k_verify.cu is the geometric half).  The protocol is stated in nero_b200/features.py, the ABI in
// include/nero_features.h.
//
//   match    one CTA of two warpgroups per directed tile: 128 rows of image a against every 128-column chunk of image b.
//            Each 128-byte descriptor row is one SWIZZLE_128B row of a K-major operand; the chunks of b stream through a
//            double buffer by cp.async while the previous chunk's four m64n128k32 u8 wgmmas and epilogue run.  The s32 dot
//            products are exact, so |a|^2 + |b|^2 - 2 a.b is the exact squared distance; each row's best and second best
//            stay in registers (ties to the lower column) and are merged over the four lanes that share the row.
//   mutual   one block per forward tile: ratio, distance and cross-check tests, then count -> block_offsets -> emit, so
//            each pair's matches come out in row order.
// Both directions of a pair are tiles of the same launch; the cross-check reads the backward direction's row bests, so
// nothing depends on which CTA finishes first.
#include <climits>

#include "common.cuh"
#include "compact.cuh"
#include "ptx.cuh"
#include "../../include/nero_features.h"

namespace nero {
namespace {

constexpr int kTile = NERO_FEATURES_TILE;
constexpr int kDim = NERO_FEATURES_DIM;
constexpr int kThreads = 256;               // two warpgroups, 64 rows each
constexpr int kTileBytes = kTile * kDim;    // 16 KB

static_assert(kDim == 128 && kTile == 128, "one descriptor row is one 128-byte swizzle row; one chunk is one N = 128 MMA");

template <int N>
__device__ __forceinline__ void fence_iregs(int* r) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// 128 rows of 128 bytes from src into the K-major SWIZZLE_128B tile at dst: 16-byte chunk c of row r lands at chunk
// c ^ (r & 7) of the row
__device__ __forceinline__ void load_tile(uint32_t dst, const unsigned char* __restrict__ src) {
#pragma unroll
  for (int k = 0; k < kTileBytes / 16 / kThreads; ++k) {
    const int q = threadIdx.x + k * kThreads;
    const int r = q >> 3, c = q & 7;
    cp_async16(dst + r * kDim + ((c ^ (r & 7)) << 4), src + (size_t)r * kDim + c * 16, 16);
  }
}

__device__ __forceinline__ void take(int d, int col, int& b1, int& i1, int& b2) {
  if (d < b1) {
    b2 = b1;
    b1 = d;
    i1 = col;
  } else if (d < b2) {
    b2 = d;
  }
}

// merges the (best, index, second) of the lane `mask` away
__device__ __forceinline__ void merge(int& b1, int& i1, int& b2, int mask) {
  const int ob1 = __shfl_xor_sync(0xffffffffu, b1, mask), oi1 = __shfl_xor_sync(0xffffffffu, i1, mask);
  const int ob2 = __shfl_xor_sync(0xffffffffu, b2, mask);
  if (ob1 < b1 || (ob1 == b1 && (unsigned)oi1 < (unsigned)i1)) {
    b2 = min(b1, ob2);
    b1 = ob1;
    i1 = oi1;
  } else {
    b2 = min(b2, ob1);
  }
}

__global__ void __launch_bounds__(kThreads, 1) match_kernel(const unsigned char* __restrict__ desc, const int* __restrict__ norms,
                                                            const int* __restrict__ tiles, int* __restrict__ best) {
  __shared__ __align__(1024) unsigned char sA[kTileBytes];
  __shared__ __align__(1024) unsigned char sB[2][kTileBytes];
  const int* tl = tiles + 5 * blockIdx.x;
  const int a_off = tl[0], a_rows = tl[1], b_off = tl[2], b_rows = tl[3], out = tl[4];
  const int tid = threadIdx.x, lane = tid & 31, g = tid >> 7, wq = (tid >> 5) & 3;
  const int r0 = g * 64 + wq * 16 + (lane >> 2), r1 = r0 + 8;
  const int na0 = __ldg(norms + a_off + r0), na1 = __ldg(norms + a_off + r1);
  const uint32_t a_addr = smem_u32(sA), b_addr0 = smem_u32(sB[0]), b_addr1 = smem_u32(sB[1]);
  const uint64_t da = make_desc_k_sw128(a_addr + g * 64 * kDim);
  const int nch = (b_rows + kTile - 1) / kTile;
  int b1a = INT_MAX, i1a = -1, b2a = INT_MAX, b1b = INT_MAX, i1b = -1, b2b = INT_MAX;
  load_tile(a_addr, desc + (size_t)a_off * kDim);
  if (nch > 0) load_tile(b_addr0, desc + (size_t)b_off * kDim);
  cp_async_commit();
  int acc[kTile / 2];
  for (int ch = 0; ch < nch; ++ch) {
    if (ch + 1 < nch) {
      load_tile((ch & 1) ? b_addr0 : b_addr1, desc + (size_t)(b_off + (ch + 1) * kTile) * kDim);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint64_t db = make_desc_k_sw128((ch & 1) ? b_addr1 : b_addr0);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kDim / 32; ++k) WgmmaU8<kTile>::mma(acc, da + 2 * k, db + 2 * k, k > 0);
    wgmma_commit();
    wgmma_wait<0>();
    fence_iregs<kTile / 2>(acc);
    const int c0 = ch * kTile + ((lane & 3) << 1);
#pragma unroll
    for (int i = 0; i < kTile / 2; ++i) {
      const int col = c0 + ((i >> 2) << 3) + (i & 1);
      if (col < b_rows) {
        const int nb = __ldg(norms + b_off + col);
        if ((i >> 1) & 1)
          take(na1 + nb - 2 * acc[i], col, b1b, i1b, b2b);
        else
          take(na0 + nb - 2 * acc[i], col, b1a, i1a, b2a);
      }
    }
    __syncthreads();
  }
  merge(b1a, i1a, b2a, 1);
  merge(b1a, i1a, b2a, 2);
  merge(b1b, i1b, b2b, 1);
  merge(b1b, i1b, b2b, 2);
  if ((lane & 3) == 0) {
    if (r0 < a_rows) {
      int* o = best + 3 * ((size_t)out + r0);
      o[0] = i1a; o[1] = b1a; o[2] = b2a;
    }
    if (r1 < a_rows) {
      int* o = best + 3 * ((size_t)out + r1);
      o[0] = i1b; o[1] = b1b; o[2] = b2b;
    }
  }
}

__device__ __forceinline__ bool keep_row(const int* __restrict__ best, const int* __restrict__ f, int r, int num, int den, int max_d1) {
  if (r >= f[2]) return false;
  const int* rec = best + 3 * ((size_t)f[0] + r);
  const int c = rec[0], d1 = rec[1], d2 = rec[2];
  return c >= 0 && (long long)den * d1 < (long long)num * d2 && d1 <= max_d1 && best[3 * ((size_t)f[1] + c)] == f[3] + r;
}

__global__ void __launch_bounds__(kTile) mutual_count_kernel(const int* __restrict__ best, const int* __restrict__ fwd, int num, int den,
                                                             int max_d1, int* __restrict__ cnt) {
  __shared__ int s_w[kTile / 32];
  const int* f = fwd + 4 * blockIdx.x;
  int tot;
  block_scan<kTile>(keep_row(best, f, threadIdx.x, num, den, max_d1), s_w, &tot);
  if (threadIdx.x == 0) cnt[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kTile) mutual_emit_kernel(const int* __restrict__ best, const int* __restrict__ fwd, int num, int den,
                                                            int max_d1, const long long* __restrict__ off, unsigned* __restrict__ matches,
                                                            long long cap) {
  __shared__ int s_w[kTile / 32];
  const int* f = fwd + 4 * blockIdx.x;
  const int r = threadIdx.x;
  const bool k = keep_row(best, f, r, num, den, max_d1);
  int tot;
  const long long m = off[blockIdx.x] + block_scan<kTile>(k, s_w, &tot);
  if (k && m < cap) {
    matches[2 * m] = (unsigned)(f[3] + r);
    matches[2 * m + 1] = (unsigned)best[3 * ((size_t)f[0] + r)];
  }
}

}  // namespace

extern "C" {

int nero_features_match(const unsigned char* desc, const int* norms, const int* tiles, int T, int* best, void* stream) {
  if (T < 0 || (T > 0 && (!desc || !norms || !tiles || !best)) || ((uintptr_t)desc & 15)) return NERO_ERR_ARG;
  if (T == 0) return NERO_OK;
  match_kernel<<<T, kThreads, 0, (cudaStream_t)stream>>>(desc, norms, tiles, best);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_features_mutual(const int* best, const int* fwd, int T, int num, int den, int max_d1, int* blk_count, long long* blk_off,
                         long long* total, unsigned int* matches, long long cap, void* stream) {
  if (T < 0 || !total || (T > 0 && (!best || !fwd || !blk_count || !blk_off)) || cap < 0 || (cap > 0 && !matches) || num < 1 || den < 1 ||
      num > den || max_d1 < 0)
    return NERO_ERR_ARG;
  cudaStream_t st = (cudaStream_t)stream;
  if (T > 0) mutual_count_kernel<<<T, kTile, 0, st>>>(best, fwd, num, den, max_d1, blk_count);
  block_offsets<1>(blk_count, blk_off, total, T, st);
  if (T > 0) mutual_emit_kernel<<<T, kTile, 0, st>>>(best, fwd, num, den, max_d1, blk_off, matches, cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
