// wgmma weight-gradient kernel: dW[n, k] = sum_m dY[m, n] * X[m, k]  (+ sum_m dY2[m, n] * X2[m, k]).
//
// The contraction runs over SAMPLES (rows of both fp32 row-major inputs), so in memory the MMA's M / N dimension (features)
// is the contiguous one: both operands are MN-major wgmma operands.
// Operand stream, per 16-sample stage: every thread copies its own 8-feature pieces of the stage's sample rows as they lie
// (two 16-byte cp.async each) into a ring of kRawStages fp32 stages, kRawStages - 1 stages ahead of the MMAs; once its own
// copies of stage g have landed, the same thread splits them to bf16 hi / lo and stores them into the MN-major SWIZZLE_128B
// atom of MMA stage g % kMmaStages ([feature block of 64][sample group of 8][8 rows x 128 B], SBO = 1024, LBO = 2048).
// No thread reads another thread's raw copies, so the raw ring needs no barrier; one barrier per stage publishes the bf16
// stage to the MMAs, and with three MMA stages that same barrier also tells every thread that the MMAs of stage g - 3,
// which read the MMA stage it overwrites next, have completed (every warpgroup waits for its group g - 3 in iteration g - 2).
// Split-K over CTAs: CTA (p, t) owns a contiguous range of 32-sample chunks of output row tile t, accumulates a 128 x NW fp32
// tile in registers (two warpgroups of 64 rows) and stores it into slice p of the [P][rows][ld] accumulator.  CTA (p, t) is
// the only writer of its [n0, n0 + 128) x [k0, k0 + NW) window of slice p and writes it once, so the slices need no zeroing,
// and a CTA without samples stores zeros.  nero_wgrad_finish (k_weights.cu) then sums the P slices in a fixed order and
// applies the weight-norm chain rule.
// The optional second pair implements the double-backward term of the SDF network,
//   dW_k = abar_k^T h_k + v_k^T ubar_k      (SURVEY.md Appendix A.3, K4),
// in the same registers.  Column sums of dY (bias gradient) are produced from the dY copies for free.
#include "gemm_common.cuh"

namespace nero {

struct WgradParams {
  const float* dY; int ldy; const float* X; int ldx;
  const float* dY2; int ldy2; const float* X2; int ldx2;
  int n0; int n_valid;   // output rows [n0 + 128*blockIdx.y, +128) = dY columns; columns >= n_valid read as zero
  int k0; int k_valid;   // output cols [k0, k0+NW) = X columns; columns >= k_valid read as zero
  float* partial; int ld_partial; int rows_partial;  // [P][rows_partial][ld_partial]: the launch's window of every slice is stored
  float* bias_partial;                               // [P][rows_partial] (may be null), stored by the k0 == 0 launch
  const int* m_ptr; int m_cap;
};

constexpr int WG_BM = 128;
constexpr int WG_CHUNK = 32;   // split-K granule: CTA p owns chunks [p * cpp, (p + 1) * cpp) of 32 samples
constexpr int WG_BK = 16;      // samples per pipeline stage = one MMA k-step
constexpr int kRawStages = 4, kMmaStages = 3;
constexpr int kWgThreads = 256;
constexpr uint32_t kMnSbo = 1024, kMnLbo = (WG_BK / 8) * 1024;
template <int NW> struct WgCfg {
  static constexpr uint32_t a_plane = WG_BM * WG_BK * 2, b_plane = NW * WG_BK * 2;
  static constexpr uint32_t mma_stage = 2 * a_plane + 2 * b_plane;
  static constexpr uint32_t raw_a = WG_BK * WG_BM * 4, raw_stage = raw_a + WG_BK * NW * 4;   // fp32 [16][128] ‖ [16][NW]
  static constexpr uint32_t bias_off = kMmaStages * mma_stage + kRawStages * raw_stage;
  static constexpr uint32_t smem_bytes = bias_off + 8 * 128 * 4 /*bias sums per warp*/ + 1024 /*align*/;
};
static_assert(WgCfg<256>::smem_bytes <= 227 * 1024, "gemm_wgrad_kernel<256> exceeds the shared-memory limit");

__device__ __forceinline__ uint32_t mn_chunk_offset(uint32_t chunk, uint32_t s) {   // chunk = feature/8, s = sample in stage
  const uint32_t r = s & 7u;
  return (chunk >> 3) * kMnLbo + (s >> 3) * kMnSbo + r * 128u + (((chunk & 7u) ^ r) << 4);
}

// copies 8 consecutive features [col, col + 8) of sample row srow to shared dst (32 bytes); rows >= M and features >= lim
// become zero.  Aligned operands go by two 16-byte cp.async that read only the features below lim; an operand that is not
// 16-byte aligned is loaded and stored by the thread itself (visible to it in program order, like its landed copies)
__device__ __forceinline__ void copy8(uint32_t dst, const float* __restrict__ src, int ld, bool vec, int srow, int M, int col, int lim) {
  const float* q = src + size_t(srow) * ld + col;
  if (vec) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = srow < M ? min(max(lim - col - 4 * h, 0), 4) : 0;   // features of this half to read
      cp_async16(dst + 16 * h, n ? q + 4 * h : src, 4u * n);
    }
  } else {
    float x[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] = (srow < M && col + j < lim) ? __ldg(q + j) : 0.0f;
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(x[0]), "f"(x[1]), "f"(x[2]), "f"(x[3]) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + 16), "f"(x[4]), "f"(x[5]), "f"(x[6]), "f"(x[7]) : "memory");
  }
}
__device__ __forceinline__ void lds8(uint32_t src, float* x) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3]) : "r"(src) : "memory");
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[4]), "=f"(x[5]), "=f"(x[6]), "=f"(x[7]) : "r"(src + 16) : "memory");
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
  constexpr int CB = NW / 8;                       // 8-feature (32-byte) chunks per X row
  constexpr int SB = kWgThreads / CB;              // sample stride between a thread's X tasks: 8 / 16 / 32
  constexpr int NB = (WG_BK + SB - 1) / SB;        // X tasks per thread and stage: 2 / 1 / 1 (threads >= 128 idle at NW = 64)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* raw = smem + kMmaStages * Cfg::mma_stage;
  float* s_bias = reinterpret_cast<float*>(smem + Cfg::bias_off);   // [8 warps][128]

  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, w = t >> 5, l = t & 31;
  int M = p.m_ptr ? *p.m_ptr : p.m_cap;
  if (M > p.m_cap) M = p.m_cap;
  const int P = gridDim.x;
  const int n0 = p.n0 + int(blockIdx.y) * WG_BM;
  const int total_chunks = (M + WG_CHUNK - 1) / WG_CHUNK;
  const int cpp = (total_chunks + P - 1) / P;
  const int c_begin = min(total_chunks, int(blockIdx.x) * cpp), c_end = min(total_chunks, c_begin + cpp);
  const int nc1 = c_end - c_begin;                          // 32-sample chunks per pair (0: the CTA stores zeros)
  const int nst1 = nc1 * (WG_CHUNK / WG_BK);                 // 16-sample stages per pair
  const int nstages = nst1 * (p.dY2 ? 2 : 1);

  auto vec = [](const float* q, int ld) { return q && ((reinterpret_cast<uintptr_t>(q) & 15) == 0) && ((ld & 3) == 0); };
  const bool vy = vec(p.dY, p.ldy), vx = vec(p.X, p.ldx), vy2 = vec(p.dY2, p.ldy2), vx2 = vec(p.X2, p.ldx2);
  // this thread's pieces of every stage: dY feature chunk a_ch of sample a_s; X chunk b_ch of samples b_s + SB j.  Sample
  // a_s of the two 16-sample stages of a chunk is sample a_s, a_s + 16 of the chunk: the bias sums add in chunk order
  const uint32_t a_ch = tid & 15, a_s = tid >> 4;
  const uint32_t b_ch = tid % CB, b_s = tid / CB;
  const int a_col = n0 + int(a_ch) * 8, b_col = p.k0 + int(b_ch) * 8;
  const uint32_t raw0 = smem_u32(raw);
  const uint32_t a_raw = a_s * (WG_BM * 4) + a_ch * 32, b_raw = Cfg::raw_a + b_s * (NW * 4) + b_ch * 32;

  auto issue = [&](int q) {        // copies of stage q into raw stage q % kRawStages
    const int pair = q >= nst1;
    const int qq = q - pair * nst1;
    const int s0 = c_begin * WG_CHUNK + qq * WG_BK;
    const uint32_t st = raw0 + uint32_t(q % kRawStages) * Cfg::raw_stage;
    copy8(st + a_raw, pair ? p.dY2 : p.dY, pair ? p.ldy2 : p.ldy, pair ? vy2 : vy, s0 + int(a_s), M, a_col, p.n_valid);
#pragma unroll
    for (int j = 0; j < NB; ++j)
      if (b_s + SB * j < uint32_t(WG_BK))
        copy8(st + b_raw + j * SB * (NW * 4), pair ? p.X2 : p.X, pair ? p.ldx2 : p.ldx, pair ? vx2 : vx, s0 + int(b_s) + SB * j, M,
              b_col, p.k_valid);
  };

  float bsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float acc[NW / 2];
#pragma unroll
  for (int i = 0; i < NW / 2; ++i) acc[i] = 0.0f;

#pragma unroll 1
  for (int q = 0; q < kRawStages - 1; ++q) {
    if (q < nstages) issue(q);
    cp_async_commit();
  }
  for (int g = 0; g < nstages; ++g) {
    if (g + kRawStages - 1 < nstages) issue(g + kRawStages - 1);   // into the raw stage this thread converted last iteration
    cp_async_commit();
    cp_async_wait<kRawStages - 1>();                                  // this thread's copies of stage g have landed
    const uint32_t rs = raw0 + uint32_t(g % kRawStages) * Cfg::raw_stage;
    uint8_t* st = smem + (g % kMmaStages) * Cfg::mma_stage;
    {
      float x[8];
      lds8(rs + a_raw, x);
      store8(st, st + Cfg::a_plane, mn_chunk_offset(a_ch, a_s), x);
      if (g < nst1) {
#pragma unroll
        for (int j = 0; j < 8; ++j) bsum[j] += x[j];
      }
    }
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      if (b_s + SB * j < uint32_t(WG_BK)) {
        float x[8];
        lds8(rs + b_raw + j * SB * (NW * 4), x);
        store8(st + 2 * Cfg::a_plane, st + 2 * Cfg::a_plane + Cfg::b_plane, mn_chunk_offset(b_ch, b_s + SB * j), x);
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    const uint32_t a_hi = smem_u32(st) + wg * kMnLbo, a_lo = a_hi + Cfg::a_plane;   // this warpgroup's 64 features
    const uint32_t b_hi = smem_u32(st) + 2 * Cfg::a_plane, b_lo = b_hi + Cfg::b_plane;
    fence_regs<NW / 2>(acc);
    wgmma_fence();
    mma_split3<NW, 1, 1>(acc, make_desc_mn_sw128(a_hi, kMnLbo, kMnSbo), make_desc_mn_sw128(a_lo, kMnLbo, kMnSbo),
                         make_desc_mn_sw128(b_hi, kMnLbo, kMnSbo), make_desc_mn_sw128(b_lo, kMnLbo, kMnSbo), 1);
    wgmma_commit();
    wgmma_wait<1>();
    fence_regs<NW / 2>(acc);
  }
  wgmma_wait<0>();
  fence_regs<NW / 2>(acc);
  cp_async_wait<0>();
  // column sums of dY: the 16 threads of one feature chunk (lanes l, l + 16 of all 8 warps) are summed in a fixed order
#pragma unroll
  for (int j = 0; j < 8; ++j) bsum[j] += __shfl_xor_sync(0xffffffffu, bsum[j], 16);
  if ((tid & 31) < 16) {
#pragma unroll
    for (int j = 0; j < 8; ++j) s_bias[(tid >> 5) * 128 + a_ch * 8 + j] = bsum[j];
  }
  // -------- epilogue: the 128 x NW tile is stored into this CTA's slice of the layer's accumulator
  float* slice = p.partial + size_t(blockIdx.x) * p.rows_partial * p.ld_partial;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int orow = n0 + wg * 64 + w * 16 + (l >> 2) + 8 * h;
    if (orow >= p.rows_partial) continue;
    float* prow = slice + size_t(orow) * p.ld_partial + p.k0 + 2 * (l & 3);
#pragma unroll
    for (int jb = 0; jb < NW / 8; ++jb)
      *reinterpret_cast<float2*>(prow + 8 * jb) = make_float2(acc[4 * jb + 2 * h], acc[4 * jb + 2 * h + 1]);
  }
  __syncthreads();
  if (tid < 128 && p.bias_partial && p.k0 == 0 && n0 + tid < p.rows_partial) {
    float b = 0.0f;
#pragma unroll
    for (int wi = 0; wi < 8; ++wi) b += s_bias[wi * 128 + tid];
    p.bias_partial[size_t(blockIdx.x) * p.rows_partial + n0 + tid] = b;
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

// Stores partial[P][rows_partial][ld_partial] for output rows [0, n_rows_pad) and columns [0, k_pad)
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
