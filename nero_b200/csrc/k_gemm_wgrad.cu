// wgmma weight-gradient kernel: dW[n, k] = sum_m dY[m, n] * X[m, k]  (+ sum_m dY2[m, n] * X2[m, k]).
//
// The contraction runs over SAMPLES (rows of both fp32 row-major inputs), so in memory the MMA's M / N dimension (features)
// is the contiguous one: both operands are MN-major wgmma operands.  All 256 threads copy sample rows as they lie -- 8
// features of one sample per task (two float4 loads when aligned), split to bf16 hi / lo, one 16-byte shared store per plane
// into the MN-major SWIZZLE_128B atom.  Stage layout per plane: [feature block of 64][sample group of 8][8 rows x 128 B]
// (SBO = 1024, LBO = 4096 with 32-sample stages); the loads of stage g + 1 are in flight while the MMAs of stage g run.
// Split-K over CTAs: CTA (p, t) owns a contiguous range of 32-sample stages of output row tile t, accumulates a 128 x NW fp32
// tile in registers (two warpgroups of 64 rows) and adds it into slice p of the [P][rows][ld] accumulator (plain loads and
// stores: the slice belongs to that CTA alone, so the result does not depend on the order in which CTAs finish).
// nero_wgrad_finish (k_weights.cu) then sums the P slices in a fixed order and applies the weight-norm chain rule.  The
// caller zeroes the accumulator.
// The optional second pair implements the double-backward term of the SDF network,
//   dW_k = abar_k^T h_k + v_k^T ubar_k      (SURVEY.md Appendix A.3, K4),
// in ONE accumulator.  Column sums of dY (bias gradient) are produced by the dY loads for free.
#include "gemm_common.cuh"

namespace nero {

struct WgradParams {
  const float* dY; int ldy; const float* X; int ldx;
  const float* dY2; int ldy2; const float* X2; int ldx2;
  int n0; int n_valid;   // output rows [n0 + 128*blockIdx.y, +128) = dY columns; columns >= n_valid read as zero
  int k0; int k_valid;   // output cols [k0, k0+NW) = X columns; columns >= k_valid read as zero
  float* partial; int ld_partial; int rows_partial;  // [P][rows_partial][ld_partial], accumulated into (zeroed by the caller)
  float* bias_partial;                               // [P][rows_partial] (may be null), accumulated into
  const int* m_ptr; int m_cap;
};

constexpr int WG_BM = 128, WG_BK = 32;
constexpr int kWgThreads = 256;
constexpr uint32_t kMnSbo = 1024, kMnLbo = (WG_BK / 8) * 1024;
template <int NW> struct WgCfg {
  static constexpr uint32_t a_plane = WG_BM * WG_BK * 2, b_plane = NW * WG_BK * 2;
  static constexpr uint32_t stage_bytes = 2 * a_plane + 2 * b_plane;
  static constexpr uint32_t smem_bytes = 2 * stage_bytes + 1024 /*align*/ + 8 * 128 * 4 /*bias sums per warp*/;
};

__device__ __forceinline__ uint32_t mn_chunk_offset(uint32_t chunk, uint32_t s) {   // chunk = feature/8, s = sample in stage
  const uint32_t r = s & 7u;
  return (chunk >> 3) * kMnLbo + (s >> 3) * kMnSbo + r * 128u + (((chunk & 7u) ^ r) << 4);
}

__device__ __forceinline__ void add2(float* addr, float a, float b) {
  float2 v = *reinterpret_cast<float2*>(addr);
  v.x += a;
  v.y += b;
  *reinterpret_cast<float2*>(addr) = v;
}

// 8 consecutive features [col, col + 8) of sample row srow; rows >= M and features >= lim read as zero
__device__ __forceinline__ void load8(const float* __restrict__ src, int ld, bool vec, int srow, int M, int col, int lim, float* x) {
  const float* q = src + size_t(srow) * ld + col;
  if (srow < M && vec && col + 7 < lim) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(q)), b = __ldg(reinterpret_cast<const float4*>(q + 4));
    x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w; x[4] = b.x; x[5] = b.y; x[6] = b.z; x[7] = b.w;
  } else {
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = (srow < M && col + j < lim) ? __ldg(q + j) : 0.0f;
  }
}
__device__ __forceinline__ void store8(uint8_t* hi, uint8_t* lo, uint32_t off, const float* x) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split2(x[2 * j], x[2 * j + 1], hw[j], lw[j]);
  *reinterpret_cast<uint4*>(hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  *reinterpret_cast<uint4*>(lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

template <int NW>
__global__ void __launch_bounds__(kWgThreads, 1) gemm_wgrad_kernel(const WgradParams p) {
  using Cfg = WgCfg<NW>;
  constexpr int CB = NW / 8;                  // 16-byte feature chunks per X row
  constexpr int NB = (WG_BK * CB) / kWgThreads;   // X tasks per thread and stage: 4 / 2 / 1
  constexpr int SB = kWgThreads / CB;         // sample stride between a thread's X tasks
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  float* s_bias = reinterpret_cast<float*>(smem + 2 * Cfg::stage_bytes);   // [8 warps][128]

  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, w = t >> 5, l = t & 31;
  int M = p.m_ptr ? *p.m_ptr : p.m_cap;
  if (M > p.m_cap) M = p.m_cap;
  const int P = gridDim.x;
  const int n0 = p.n0 + int(blockIdx.y) * WG_BM;
  const int total_chunks = (M + WG_BK - 1) / WG_BK;
  const int cpp = (total_chunks + P - 1) / P;
  const int c_begin = min(total_chunks, int(blockIdx.x) * cpp), c_end = min(total_chunks, c_begin + cpp);
  const int npairs = p.dY2 ? 2 : 1;
  const int nc1 = c_end - c_begin;
  const int nchunks = nc1 * npairs;
  if (nchunks == 0) return;

  auto vec = [](const float* q, int ld) { return q && ((reinterpret_cast<uintptr_t>(q) & 15) == 0) && ((ld & 3) == 0); };
  const bool vy = vec(p.dY, p.ldy), vx = vec(p.X, p.ldx), vy2 = vec(p.dY2, p.ldy2), vx2 = vec(p.X2, p.ldx2);
  // this thread's tasks (constant over stages): dY feature chunk a_ch of samples a_s, a_s + 16; X chunk b_ch of b_s + SB j
  const uint32_t a_ch = tid & 15, a_s = tid >> 4;
  const uint32_t b_ch = tid % CB, b_s = tid / CB;
  const int a_col = n0 + int(a_ch) * 8, b_col = p.k0 + int(b_ch) * 8;
  float bsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float acc[NW / 2];
#pragma unroll
  for (int i = 0; i < NW / 2; ++i) acc[i] = 0.0f;

  for (int g = 0; g < nchunks; ++g) {
    const int s = g & 1;
    const int pair = g / nc1;
    const int s0 = (c_begin + g % nc1) * WG_BK;
    uint8_t* st = smem + s * Cfg::stage_bytes;
    float xa[2][8], xb[NB][8];
#pragma unroll
    for (int i = 0; i < 2; ++i)
      load8(pair ? p.dY2 : p.dY, pair ? p.ldy2 : p.ldy, pair ? vy2 : vy, s0 + int(a_s) + 16 * i, M, a_col, p.n_valid, xa[i]);
#pragma unroll
    for (int j = 0; j < NB; ++j)
      load8(pair ? p.X2 : p.X, pair ? p.ldx2 : p.ldx, pair ? vx2 : vx, s0 + int(b_s) + SB * j, M, b_col, p.k_valid, xb[j]);
    // every warpgroup has finished the MMAs of stage g - 2 (wgmma_wait<1> below): buffer s is free
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      store8(st, st + Cfg::a_plane, mn_chunk_offset(a_ch, a_s + 16 * i), xa[i]);
      if (pair == 0) {
#pragma unroll
        for (int j = 0; j < 8; ++j) bsum[j] += xa[i][j];
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j)
      store8(st + 2 * Cfg::a_plane, st + 2 * Cfg::a_plane + Cfg::b_plane, mn_chunk_offset(b_ch, b_s + SB * j), xb[j]);
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t a_hi = smem_u32(st) + wg * kMnLbo, a_lo = a_hi + Cfg::a_plane;   // this warpgroup's 64 features
    const uint32_t b_hi = smem_u32(st) + 2 * Cfg::a_plane, b_lo = b_hi + Cfg::b_plane;
    fence_regs<NW / 2>(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < WG_BK / 16; ++k) {     // 16 samples = two 8-row groups per MMA
      const uint32_t ko = k * 2 * kMnSbo;
      mma_split3<NW, 1, 1>(acc, make_desc_mn_sw128(a_hi + ko, kMnLbo, kMnSbo), make_desc_mn_sw128(a_lo + ko, kMnLbo, kMnSbo),
                           make_desc_mn_sw128(b_hi + ko, kMnLbo, kMnSbo), make_desc_mn_sw128(b_lo + ko, kMnLbo, kMnSbo), 1);
    }
    wgmma_commit();
    wgmma_wait<1>();
    fence_regs<NW / 2>(acc);
  }
  wgmma_wait<0>();
  fence_regs<NW / 2>(acc);
  // column sums of dY: the 16 threads of one feature chunk (lanes l, l + 16 of all 8 warps) are summed in a fixed order
#pragma unroll
  for (int j = 0; j < 8; ++j) bsum[j] += __shfl_xor_sync(0xffffffffu, bsum[j], 16);
  if ((tid & 31) < 16) {
#pragma unroll
    for (int j = 0; j < 8; ++j) s_bias[(tid >> 5) * 128 + a_ch * 8 + j] = bsum[j];
  }
  // -------- epilogue: the 128 x NW tile is added into this CTA's slice of the layer's accumulator
  float* slice = p.partial + size_t(blockIdx.x) * p.rows_partial * p.ld_partial;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int orow = n0 + wg * 64 + w * 16 + (l >> 2) + 8 * h;
    if (orow >= p.rows_partial) continue;
    float* prow = slice + size_t(orow) * p.ld_partial + p.k0 + 2 * (l & 3);
#pragma unroll
    for (int jb = 0; jb < NW / 8; ++jb) add2(prow + 8 * jb, acc[4 * jb + 2 * h], acc[4 * jb + 2 * h + 1]);
  }
  __syncthreads();
  if (tid < 128 && p.bias_partial && p.k0 == 0 && n0 + tid < p.rows_partial) {
    float b = 0.0f;
#pragma unroll
    for (int wi = 0; wi < 8; ++wi) b += s_bias[wi * 128 + tid];
    p.bias_partial[size_t(blockIdx.x) * p.rows_partial + n0 + tid] += b;
  }
}

template <int NW>
static int launch_wgrad(const WgradParams& p, int P, int n_tiles, cudaStream_t stream) {
  using Cfg = WgCfg<NW>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_wgrad_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::smem_bytes) != cudaSuccess)
      return NERO_ERR_CUDA;
    attr_set = true;
  }
  gemm_wgrad_kernel<NW><<<dim3(P, n_tiles), kWgThreads, Cfg::smem_bytes, stream>>>(p);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

// Accumulates partial[P][rows_partial][ld_partial] for output rows [0, n_rows_pad) and columns [0, k_pad)
// (k_pad multiple of 64), decomposed into 128-row tiles (grid.y) x {256,128,64}-column tiles (separate launches).
extern "C" int nero_wgrad(const float* dY, int ldy, int n_valid, const float* X, int ldx, int k_valid,
                          const float* dY2, int ldy2, const float* X2, int ldx2,
                          float* partial, int ld_partial, int rows_partial, float* bias_partial,
                          int n_rows_pad, int k_pad, int P, const int* m_ptr, int m_cap, void* stream_) {
  WgradParams p{dY, ldy, X, ldx, dY2, ldy2, X2, ldx2, 0, n_valid, 0, k_valid, partial, ld_partial, rows_partial, bias_partial,
                m_ptr, m_cap};
  const cudaStream_t stream = (cudaStream_t)stream_;
  if (!dY || !X || !partial || (dY2 && !X2)) return NERO_ERR_ARG;
  if ((p.ld_partial & 3) || k_pad % 64 || n_rows_pad % 16 || P <= 0) return NERO_ERR_ARG;
  const int n_tiles = (n_rows_pad + 127) / 128;
  p.n0 = 0;
  int k0 = 0;
  while (k0 < k_pad) {
    const int rem = k_pad - k0;
    p.k0 = k0;
    int rc;
    if (rem >= 256) { rc = launch_wgrad<256>(p, P, n_tiles, stream); k0 += 256; }
    else if (rem >= 128) { rc = launch_wgrad<128>(p, P, n_tiles, stream); k0 += 128; }
    else { rc = launch_wgrad<64>(p, P, n_tiles, stream); k0 += 64; }
    if (rc != NERO_OK) return rc;
  }
  return NERO_OK;
}

}  // namespace nero
