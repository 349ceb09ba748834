// wgmma weight-gradient kernel: dW[n, k] = sum_m dY[m, n] * X[m, k]  (+ sum_m dY2[m, n] * X2[m, k]).
//
// The contraction runs over SAMPLES (rows of both fp32 row-major inputs), so in memory the MMA's M / N dimension (features)
// is the contiguous one: both operands are MN-major wgmma operands.
// Operand stream, per 16-sample stage: the stage's sample rows arrive as they lie in a ring of kRawStages fp32 stages,
// kRawStages - 1 stages ahead of the MMAs.  When every operand is 16-byte aligned (the tensors a training step passes),
// thread 0 brings a stage with two tensor copies (TMA: a 16 x 128 box of dY and a 16 x NW box of X) that complete the raw
// stage's mbarrier; otherwise (an operand that is not 16-byte aligned, or an empty tensor) every thread loads its own
// 8-feature pieces and stores them itself.  Per-thread cp.async copies, which the tensor copies replaced, cost the
// issuing warps about half of each stage's cycles on an H100 (DESIGN.md section 6, "Weight-gradient pass: tensor copies
// for the operand ring").  Once stage g has landed, every thread splits its own pieces to bf16
// hi / lo and stores them into the MN-major SWIZZLE_128B atom of MMA stage g % kMmaStages ([feature block of 64][sample
// group of 8][8 rows x 128 B], SBO = 1024, LBO = 2048).  One barrier per stage publishes the bf16 stage to the MMAs; it
// also tells thread 0 that every thread has read the raw stage it refills next, and, with three MMA stages, tells every
// thread that the MMAs of stage g - 3, which read the MMA stage it overwrites next, have completed (every warpgroup waits
// for its group g - 3 in iteration g - 2).
// Split-K over CTAs: CTA (p, t) owns a contiguous range of 32-sample chunks of output row tile t, accumulates a 128 x NW fp32
// tile in registers (two warpgroups of 64 rows) and stores it into slice p of the [P][rows][ld] accumulator.  CTA (p, t) is
// the only writer of its [n0, n0 + 128) x [k0, k0 + NW) window of slice p and writes it once, so the slices need no zeroing,
// and a CTA without samples stores zeros.  nero_wgrad_finish (k_weights.cu) then sums the P slices in a fixed order and
// applies the weight-norm chain rule.
// The optional second pair implements the double-backward term of the SDF network,
//   dW_k = abar_k^T h_k + v_k^T ubar_k      (SURVEY.md Appendix A.3, K4),
// in the same registers.  Column sums of dY (bias gradient) are produced from the dY copies for free.
#include <cudaTypedefs.h>

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
  int tma;               // operands come by the tensor maps below (all 16-byte aligned), else by per-thread copies
};
// 2-D fp32 tensor maps of dY, X (dY2, X2) over [m_cap rows][n_valid / k_valid columns], boxes of 16 rows x 128 / NW columns
struct WgradMaps { CUtensorMap y, x, y2, x2; };

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
  static constexpr uint32_t bar_off = bias_off + 8 * 128 * 4;                                  // after the bias sums per warp
  static constexpr uint32_t smem_bytes = bar_off + kRawStages * 8 /*raw_full*/ + 1024 /*align*/;
};
static_assert(WgCfg<256>::smem_bytes <= 227 * 1024, "gemm_wgrad_kernel<256> exceeds the shared-memory limit");

__device__ __forceinline__ uint32_t mn_chunk_offset(uint32_t chunk, uint32_t s) {   // chunk = feature/8, s = sample in stage
  const uint32_t r = s & 7u;
  return (chunk >> 3) * kMnLbo + (s >> 3) * kMnSbo + r * 128u + (((chunk & 7u) ^ r) << 4);
}

// copies 8 consecutive features [col, col + 8) of sample row srow to shared dst (32 bytes); rows >= M and features >= lim
// become zero.  The thread loads and stores them itself, so they are visible to it in program order (operands without
// tensor maps: not 16-byte aligned, or empty)
__device__ __forceinline__ void copy8(uint32_t dst, const float* __restrict__ src, int ld, int srow, int M, int col, int lim) {
  const float* q = src + size_t(srow) * ld + col;
  float x[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = (srow < M && col + j < lim) ? __ldg(q + j) : 0.0f;
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(x[0]), "f"(x[1]), "f"(x[2]), "f"(x[3]) : "memory");
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + 16), "f"(x[4]), "f"(x[5]), "f"(x[6]), "f"(x[7]) : "memory");
}
__device__ __forceinline__ void lds8(uint32_t src, float* x) {
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[0]), "=f"(x[1]), "=f"(x[2]), "=f"(x[3]) : "r"(src) : "memory");
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(x[4]), "=f"(x[5]), "=f"(x[6]), "=f"(x[7]) : "r"(src + 16) : "memory");
}
// a sample row at or past M reads as zero (the tensor copies bring rows up to m_cap)
__device__ __forceinline__ void zero_past(float* x, bool row_ok) {
#pragma unroll
  for (int j = 0; j < 8; ++j) x[j] = row_ok ? x[j] : 0.0f;
}
__device__ __forceinline__ void store8(uint8_t* hi, uint8_t* lo, uint32_t off, const float* x) {
  uint32_t hw[4], lw[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) split2(x[2 * j], x[2 * j + 1], hw[j], lw[j]);
  *reinterpret_cast<uint4*>(hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
  *reinterpret_cast<uint4*>(lo + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

template <int NW>
__global__ void __launch_bounds__(kWgThreads, 1) gemm_wgrad_kernel(const WgradParams p, const __grid_constant__ WgradMaps maps) {
  using Cfg = WgCfg<NW>;
  constexpr int CB = NW / 8;                       // 8-feature (32-byte) chunks per X row
  constexpr int SB = kWgThreads / CB;              // sample stride between a thread's X tasks: 8 / 16 / 32
  constexpr int NB = (WG_BK + SB - 1) / SB;        // X tasks per thread and stage: 2 / 1 / 1 (threads >= 128 idle at NW = 64)
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* raw = smem + kMmaStages * Cfg::mma_stage;
  float* s_bias = reinterpret_cast<float*>(smem + Cfg::bias_off);   // [8 warps][128]
  uint64_t* raw_full = reinterpret_cast<uint64_t*>(smem + Cfg::bar_off);   // [kRawStages]: the stage's tensor copies landed

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
    if (p.tma) {
      // one thread brings the stage: a 16 x 128 box of dY and a 16 x NW box of X (columns past the limit and rows past
      // m_cap arrive as zeros, rows in [M, m_cap) are zeroed as they are converted), completing raw_full of the raw stage
      if (tid == 0) {
        uint8_t* rs = raw + (q % kRawStages) * Cfg::raw_stage;
        uint64_t* bar = &raw_full[q % kRawStages];
        mbar_arrive_expect_tx(bar, Cfg::raw_stage);
        tma_load_2d(rs, pair ? &maps.y2 : &maps.y, n0, s0, bar);
        tma_load_2d(rs + Cfg::raw_a, pair ? &maps.x2 : &maps.x, p.k0, s0, bar);
      }
      return;
    }
    const uint32_t st = raw0 + uint32_t(q % kRawStages) * Cfg::raw_stage;
    copy8(st + a_raw, pair ? p.dY2 : p.dY, pair ? p.ldy2 : p.ldy, s0 + int(a_s), M, a_col, p.n_valid);
#pragma unroll
    for (int j = 0; j < NB; ++j)
      if (b_s + SB * j < uint32_t(WG_BK))
        copy8(st + b_raw + j * SB * (NW * 4), pair ? p.X2 : p.X, pair ? p.ldx2 : p.ldx, s0 + int(b_s) + SB * j, M, b_col, p.k_valid);
  };

  float bsum[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  float acc[NW / 2];
#pragma unroll
  for (int i = 0; i < NW / 2; ++i) acc[i] = 0.0f;

  if (tid == 0) {
    for (int s = 0; s < kRawStages; ++s) mbar_init(&raw_full[s], 1);
    fence_mbar_init();
  }
  __syncthreads();
  bool timed_out = false;

#pragma unroll 1
  for (int q = 0; q < kRawStages - 1; ++q)
    if (q < nstages) issue(q);
  for (int g = 0; g < nstages; ++g) {
    if (g + kRawStages - 1 < nstages) issue(g + kRawStages - 1);   // into the raw stage converted last iteration
    if (p.tma) mbar_wait_flag(&raw_full[g % kRawStages], uint32_t(g / kRawStages) & 1u, timed_out);   // the stage's boxes
    const int s0 = c_begin * WG_CHUNK + (g - (g >= nst1) * nst1) * WG_BK;   // the stage's first sample
    const uint32_t rs = raw0 + uint32_t(g % kRawStages) * Cfg::raw_stage;
    uint8_t* st = smem + (g % kMmaStages) * Cfg::mma_stage;
    {
      float x[8];
      lds8(rs + a_raw, x);
      zero_past(x, s0 + int(a_s) < M);
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
        zero_past(x, s0 + int(b_s) + SB * j < M);
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
  if (timed_out) __trap();
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

// cuTensorMapEncodeTiled from the driver the runtime uses (no link against libcuda)
static PFN_cuTensorMapEncodeTiled_v12000 tensor_map_encoder() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* f = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(f);
  }
  return fn;
}
// [rows][cols] fp32 with row stride ld (floats), read in boxes of WG_BK rows x box_cols columns
static bool make_map(CUtensorMap* m, const float* base, int ld, int cols, int rows, int box_cols) {
  const PFN_cuTensorMapEncodeTiled_v12000 enc = tensor_map_encoder();
  if (!enc || cols <= 0 || rows <= 0) return false;
  const cuuint64_t dim[2] = {cuuint64_t(cols), cuuint64_t(rows)}, stride[1] = {cuuint64_t(ld) * 4u};
  const cuuint32_t box[2] = {cuuint32_t(box_cols), cuuint32_t(WG_BK)}, estr[2] = {1, 1};
  return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dim, stride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int NW>
static int launch_wgrad(const WgradParams& p, WgradMaps& maps, int P, int n_tiles, cudaStream_t stream) {
  using Cfg = WgCfg<NW>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_wgrad_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::smem_bytes) != cudaSuccess)
      return NERO_ERR_CUDA;
    attr_set = true;
  }
  WgradParams q = p;
  if (q.tma)   // X boxes are NW columns wide
    q.tma = make_map(&maps.x, p.X, p.ldx, p.k_valid, p.m_cap, NW) && (!p.X2 || make_map(&maps.x2, p.X2, p.ldx2, p.k_valid, p.m_cap, NW));
  gemm_wgrad_kernel<NW><<<dim3(P, n_tiles), kWgThreads, Cfg::smem_bytes, stream>>>(q, maps);
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
                m_ptr, m_cap, 0};
  const cudaStream_t stream = (cudaStream_t)stream_;
  if (!dY || !X || !partial || (dY2 && !X2)) return NERO_ERR_ARG;
  if ((p.ld_partial & 3) || k_pad % 64 || n_rows_pad % 16 || P <= 0) return NERO_ERR_ARG;
  const int n_tiles = (n_rows_pad + 127) / 128;
  // aligned operands (16-byte base and row stride) go by tensor copies; an empty tensor or an unaligned operand by the
  // per-thread copies
  auto aligned = [](const float* q, int ld) { return !q || (((reinterpret_cast<uintptr_t>(q) & 15) == 0) && (ld & 3) == 0); };
  const bool all_aligned = aligned(dY, ldy) && aligned(X, ldx) && aligned(dY2, ldy2) && aligned(X2, ldx2);
  if (all_aligned && !tensor_map_encoder()) return NERO_ERR_CUDA;
  WgradMaps maps{};
  p.tma = all_aligned && make_map(&maps.y, dY, ldy, n_valid, m_cap, WG_BM) &&
          (!dY2 || make_map(&maps.y2, dY2, ldy2, n_valid, m_cap, WG_BM));
  p.n0 = 0;
  int k0 = 0;
  while (k0 < k_pad) {
    const int rem = k_pad - k0;
    p.k0 = k0;
    int rc;
    if (rem >= 256) { rc = launch_wgrad<256>(p, maps, P, n_tiles, stream); k0 += 256; }
    else if (rem >= 128) { rc = launch_wgrad<128>(p, maps, P, n_tiles, stream); k0 += 128; }
    else { rc = launch_wgrad<64>(p, maps, P, n_tiles, stream); k0 += 64; }
    if (rc != NERO_OK) return rc;
  }
  return NERO_OK;
}

}  // namespace nero
