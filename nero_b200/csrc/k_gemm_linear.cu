// wgmma linear-layer kernel: OUT[M, N] = epilogue( A[M, K] * W[N, K]^T ).
//
//  * A is fp32 row-major in HBM.  All 256 threads load a 128 x 64 chunk of it with coalesced float4, split every value into
//    bf16 hi + lo (packed cvt.rn.bf16x2) and store both planes in the K-major SWIZZLE_128B layout wgmma reads.  The loads
//    of chunk c + 1 are in flight while the MMAs of chunk c run (two smem stages).
//  * W is pre-split and pre-swizzled once per step by nero_prep_weight (k_weights.cu) into the exact shared-memory image
//    (32-wide K chunks, SWIZZLE_64B), so a 64-wide K chunk of it is ONE cp.async.bulk (UBLKCP) from L2, completing on an
//    mbarrier.
//  * Two warpgroups, 64 rows each, issue wgmma.m64nNk16 (bf16 x bf16 -> fp32 registers), three per k-step (split-bf16,
//    gemm_common.cuh); N = the padded layer width (16 .. 256), so one instruction covers the whole output row range.
//  * The epilogue runs on the accumulator registers (pairs of adjacent columns, 8-byte accesses: every 32-byte sector a
//    warp touches is used whole), specialised at compile time (template EPI).
//  * Persistent CTAs (one per SM), tiles of 128 rows, row count read from device memory (no host sync for the
//    data-dependent number of live samples).
//
// Reference op sites replaced: every nn.Linear (+weight_norm, +Softplus/ReLU/Sigmoid/exp) of
// network/field.py:130-147 (SDFNetwork), :258-283 (NeRFNetwork), :310-346 (make_predictor), and the
// autograd-generated input-gradient GEMMs of their backward / double-backward (SURVEY.md K2-K4, K10, K13).
#include "gemm_common.cuh"

namespace nero {

struct LinearParams {
  const float* A; int lda; int k_valid;
  const uint8_t* wimg; int n_pad; int k_chunks;
  const float* bias; int n_bias;
  float* out; int ldo; int ncol_out; float oscale;
  int mode; int act; float act_param;
  const float* H; int ldh; float hscale; int dact;
  const float* V; int ldv;
  float* out2; int ldo2;
  const float* addend; int ldadd;
  int ncol_main; float* tail; int ldt;
  const int* m_ptr; int m_cap;
};

constexpr int BM = 128;
constexpr int kLinearThreads = 256;
constexpr uint32_t kABytes = BM * 128;           // one bf16 plane of an A chunk (128 rows x 64 K, 16 KB)

template <int NPAD> struct LinCfg {
  static constexpr uint32_t b_plane = NPAD * 128;   // the hi and lo planes of one 32-wide K chunk of W
  static constexpr uint32_t stage_bytes = 2 * kABytes + 2 * b_plane;
  static constexpr uint32_t smem_bytes = 2 * stage_bytes + 1024 /*align*/ + 64 /*barriers*/;
};

template <int NPAD, int EPI>
__global__ void __launch_bounds__(kLinearThreads, 1) gemm_linear_kernel(const LinearParams p) {
  using Cfg = LinCfg<NPAD>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + 2 * Cfg::stage_bytes);   // [2] W chunk landed

  const int tid = threadIdx.x, wg = tid >> 7, t = tid & 127, w = t >> 5, l = t & 31;
  int M = p.m_ptr ? *p.m_ptr : p.m_cap;
  if (M > p.m_cap) M = p.m_cap;
  const int num_tiles = (M + BM - 1) / BM;
  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_mbar_init();
  }
  __syncthreads();

  const EpiArgs e{p.bias, p.n_bias, p.out, p.ldo, p.H, p.ldh, p.hscale, p.addend, p.ldadd, p.V, p.ldv, p.out2, p.ldo2,
                  p.tail, p.ldt, p.ncol_out, p.ncol_main, p.oscale, p.act, p.act_param};
  const int lr = tid >> 4, c4 = (tid & 15) * 4;   // A loads: rows lr + 16 i, columns c4 .. c4 + 3 of the chunk
  int g = 0;                                      // chunk counter (stage g & 1, mbarrier phase (g >> 1) & 1)
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    float acc[NPAD / 2];
#pragma unroll
    for (int i = 0; i < NPAD / 2; ++i) acc[i] = 0.0f;
    for (int c = 0; c < p.k_chunks; ++c, ++g) {
      const int s = g & 1;
      uint8_t* st = smem + s * Cfg::stage_bytes;
      float4 x[8];
      const int kcol = c * 64 + c4;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = tile * BM + lr + 16 * i;
        x[i] = (kcol < p.k_valid && r < M) ? ld_stream4(p.A + size_t(r) * p.lda + kcol)
                                            : make_float4(0.f, 0.f, 0.f, 0.f);
      }
      // every warpgroup has finished the MMAs of chunk g - 2 (wgmma_wait<1> below): stage s is free
      __syncthreads();
      if (tid == 0) {
        mbar_arrive_expect_tx(&full[s], 2 * Cfg::b_plane);
        weight_copy(st + 2 * kABytes, p.wimg + size_t(c) * 2 * Cfg::b_plane, 2 * Cfg::b_plane, &full[s]);
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const uint32_t off = sw128_offset(lr + 16 * i, c4);
        uint2 hv, lv;
        split2(x[i].x, x[i].y, hv.x, lv.x);
        split2(x[i].z, x[i].w, hv.y, lv.y);
        *reinterpret_cast<uint2*>(st + off) = hv;
        *reinterpret_cast<uint2*>(st + kABytes + off) = lv;
      }
      fence_proxy_async_smem();
      __syncthreads();
      mbar_wait(&full[s], (g >> 1) & 1);
      const uint32_t a_hi = smem_u32(st) + wg * 64 * 128, a_lo = a_hi + kABytes;
      // the weight chunk is two 32-wide K chunks, each a hi and a lo plane of NPAD rows x 64 B (SWIZZLE_64B)
      const uint32_t b0 = smem_u32(st) + 2 * kABytes;
      fence_regs<NPAD / 2>(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t b_hi = b0 + (k >> 1) * Cfg::b_plane + 32 * (k & 1), b_lo = b_hi + Cfg::b_plane / 2;
        mma_split3<NPAD, 0, 0>(acc, make_desc_k_sw128(a_hi + 32 * k), make_desc_k_sw128(a_lo + 32 * k), make_desc_k_sw64(b_hi),
                               make_desc_k_sw64(b_lo), (c | k) != 0);
      }
      wgmma_commit();
      wgmma_wait<1>();
      fence_regs<NPAD / 2>(acc);
    }
    wgmma_wait<0>();
    fence_regs<NPAD / 2>(acc);
    const long row0 = long(tile) * BM + wg * 64 + w * 16 + (l >> 2);
    epi_fragment<EPI, NPAD / 8>(e, row0, row0 < M, row0 + 8 < M, l, NPAD / 8,
                                [&](int jb, int h, long row, int col, bool row_ok, const EpiIn& in) {
      if (row_ok && col < p.ncol_out) epi_pair<EPI>(e, row, col, true, acc[4 * jb + 2 * h], acc[4 * jb + 2 * h + 1], in);
    });
  }
}

template <int NPAD, int EPI>
static int launch_linear(const LinearParams& p, cudaStream_t stream) {
  using Cfg = LinCfg<NPAD>;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_linear_kernel<NPAD, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::smem_bytes) != cudaSuccess)
      return NERO_ERR_CUDA;
    attr_set = true;
  }
  int tiles_cap = (p.m_cap + BM - 1) / BM;
  if (tiles_cap <= 0) return NERO_OK;
  int grid = tiles_cap < kNumSMs ? tiles_cap : kNumSMs;
  gemm_linear_kernel<NPAD, EPI><<<grid, kLinearThreads, Cfg::smem_bytes, stream>>>(p);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

template <int NPAD>
static int dispatch_epi(const LinearParams& p, cudaStream_t stream) {
  if (p.mode == EPI_BIAS_ACT) {
    if (p.act == ACT_SOFTPLUS100) return launch_linear<NPAD, EK_BIAS_SOFTPLUS>(p, stream);
    if (p.act == ACT_RELU) return launch_linear<NPAD, EK_BIAS_RELU>(p, stream);
    return launch_linear<NPAD, EK_BIAS_GENERIC>(p, stream);
  }
  if (p.mode == EPI_TANGENT) return launch_linear<NPAD, EK_TANGENT>(p, stream);
  if (!p.H || p.dact == ACT_NONE) return launch_linear<NPAD, EK_DACT_NONE>(p, stream);
  if (p.dact == ACT_RELU) return launch_linear<NPAD, EK_DACT_RELU>(p, stream);
  return launch_linear<NPAD, EK_DACT_SOFTPLUS>(p, stream);
}

extern "C" int nero_linear(const float* A, int lda, int k_valid, const void* wimg, int n_pad, int k_chunks, const float* bias, int n_bias,
                           float* out, int ldo, int ncol_out, float oscale, int mode, int act, float act_param,
                           const float* H, int ldh, float hscale, int dact, const float* V, int ldv, float* out2, int ldo2,
                           const float* addend, int ldadd, int ncol_main, float* tail, int ldt,
                           const int* m_ptr, int m_cap, void* stream_) {
  const LinearParams p{A, lda, k_valid, (const uint8_t*)wimg, n_pad, k_chunks, bias, n_bias, out, ldo, ncol_out, oscale, mode, act, act_param,
                       H, ldh, hscale, dact, V, ldv, out2, ldo2, addend, ldadd, ncol_main, tail, ldt, m_ptr, m_cap};
  const cudaStream_t stream = (cudaStream_t)stream_;
  if (!A || !wimg || !out || ncol_out > n_pad) return NERO_ERR_ARG;
  if (p.k_chunks <= 0 || (p.k_valid & 3) || (p.lda & 3) || (reinterpret_cast<uintptr_t>(p.A) & 15)) return NERO_ERR_ARG;
  if (p.mode == EPI_TANGENT && (!p.H || !p.V || !p.out2 || p.dact != ACT_SOFTPLUS100)) return NERO_ERR_ARG;
  if (p.mode == EPI_MUL_DACT && p.dact != ACT_NONE && !p.H) return NERO_ERR_ARG;
  if (!pair_aligned(p.H, p.ldh) || !pair_aligned(p.V, p.ldv) || !pair_aligned(p.addend, p.ldadd)) return NERO_ERR_ARG;
  switch (p.n_pad) {
    case 16: return dispatch_epi<16>(p, stream);
    case 64: return dispatch_epi<64>(p, stream);
    case 128: return dispatch_epi<128>(p, stream);
    case 224: return dispatch_epi<224>(p, stream);
    case 256: return dispatch_epi<256>(p, stream);
    default: return NERO_ERR_ARG;
  }
}

}  // namespace nero
