// Ordered stream compaction for the offline kernels (count -> scan -> emit): each file's count kernel writes one int count
// per block (or kW interleaved counts), block_offsets turns them into int64 exclusive offsets in block order and the totals,
// and each file's emit kernel places its block's items at blk_off[block] + block_scan(...).  No atomics decide placement,
// so the output order is fixed by the input alone.
#pragma once
#include <cuda_runtime.h>

namespace nero {

// exclusive prefix of x over the block in thread order; *total = block sum.  s_w: kThreads/32 ints.  Ends with a barrier,
// so s_w may be reused by the next call (a loop over sub-tiles).
template <int kThreads>
__device__ __forceinline__ int block_scan(int x, int* s_w, int* total) {
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
  for (int w = 0; w < kThreads / 32; ++w) {
    const int v = s_w[w];
    before += w < wid ? v : 0;
    tot += v;
  }
  __syncthreads();
  *total = tot;
  return before + incl - x;
}

__device__ __forceinline__ long long warp_incl(long long x, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const long long v = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += v;
  }
  return x;
}

// The library's files are compiled separately without relocatable device code, so each one gets its own copy of the kernel.
namespace {

constexpr int kOffsetThreads = 1024;

// one block: exclusive scans of kW interleaved count streams in block order (chunks of 1024 with an int64 carry), and their
// totals
template <int kW>
__global__ void __launch_bounds__(kOffsetThreads) block_offsets_kernel(const int* __restrict__ cnt, long long* __restrict__ off,
                                                                       long long* __restrict__ totals, long long nblk) {
  __shared__ long long s_w[kW][32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  long long carry[kW];
#pragma unroll
  for (int w = 0; w < kW; ++w) carry[w] = 0;
  for (long long c0 = 0; c0 < nblk; c0 += kOffsetThreads) {
    const long long b = c0 + threadIdx.x;
    long long v[kW], iv[kW];
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      v[w] = b < nblk ? cnt[kW * b + w] : 0;
      iv[w] = warp_incl(v[w], lane);
      if (lane == 31) s_w[w][wid] = iv[w];
    }
    __syncthreads();
    if (wid == 0) {
#pragma unroll
      for (int w = 0; w < kW; ++w) s_w[w][lane] = warp_incl(s_w[w][lane], lane);
    }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kW; ++w) {
      const long long pre = wid ? s_w[w][wid - 1] : 0;
      if (b < nblk) off[kW * b + w] = carry[w] + pre + iv[w] - v[w];
      carry[w] += s_w[w][31];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 0; w < kW; ++w) totals[w] = carry[w];
  }
}

// off[kW * b + w] = sum of cnt[kW * b' + w] over b' < b, totals[w] = the sum over all nblk blocks.  One launch, unchecked:
// the caller checks its launches together.
template <int kW>
void block_offsets(const int* cnt, long long* off, long long* totals, long long nblk, cudaStream_t stream) {
  block_offsets_kernel<kW><<<1, kOffsetThreads, 0, stream>>>(cnt, off, totals, nblk);
}

}  // namespace

}  // namespace nero
