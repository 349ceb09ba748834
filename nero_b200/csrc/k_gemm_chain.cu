// Fused MLP-CHAIN kernel on wgmma: a 128-row tile of samples flows through a whole sequence of linear layers without its
// activations ever leaving the SM between layers.
//
//   Shared memory: the A operand of the current layer as split-bf16 (hi and lo planes, K-major SWIZZLE_128B, up to 256 K
//   columns = 128 KB) and a ring of kWStages weight stages.  Two consumer warpgroups own 64 rows each: per layer they issue,
//   per 16-wide k-step, A_lo*W_hi + A_hi*W_lo + A_hi*W_hi into fp32 accumulators in registers (wgmma.m64n128k16 over the
//   layer's N range in one or two halves of 128 columns: a narrower layer computes columns it never reads back, one MMA
//   shape keeps the kernel within the register file), then apply bias/activation or the derivative products of the
//   gradient sweeps to those registers, store what the layer saves to HBM, and write the NEXT layer's A operand over the
//   current one (each warp only touches its own rows, whose MMAs it has waited for).
//   The weights stream from L2 as pre-swizzled images: one stage = the hi and lo planes of one 32-wide K chunk for one half
//   of the N range (up to 16 KB, K-major SWIZZLE_64B, cp.async.bulk), kWStages ahead of the MMAs across layers and tiles.
//   The warp that releases a stage last refills its slot (w_release), so no warp ever waits for another to free a slot.
//   (No separate producer warp: at 256 threads a consumer thread may hold 255 registers, which the two 64-wide fp32
//   accumulator halves need; 288 or 384 threads cap it at 168 and spill.)
//
// This realises SURVEY.md K2/K3/K4/K10/K13 "activations stay on-chip across layers".
//
// Skip connection of the SDF network (field.py:139-140): a layer with `csrc` set takes columns >= ncol_out of the
// next A operand from that buffer, where ray_fill / pe_tangent pre-stored PE/sqrt2 resp. its tangent.
#include "gemm_common.cuh"

namespace nero {

constexpr int kMaxChainLayers = 10;
static_assert(sizeof(nero_chain_params::L) / sizeof(nero_chain_layer) == kMaxChainLayers, "the C ABI's nero_chain_params.L length");

// ---------------------------------------------------------------------------------------------- configuration
constexpr int CH_BM = 128;
constexpr int kChThreads = 2 * 128;                 // two warpgroups of 64 rows
constexpr int kWStages = 6;
constexpr int HN = 128;                             // accumulator columns per N half
constexpr uint32_t kHalfBytes = HN * 64;            // one plane of 128 weight rows x 32 K
constexpr uint32_t kWStageBytes = 2 * kHalfBytes;   // hi + lo planes
constexpr uint32_t kAPlane = CH_BM * 128;           // one bf16 plane of one 64-wide K chunk of the A operand (16 KB)
constexpr uint32_t kABytes = 4 * 2 * kAPlane;       // K <= 256: four chunks x (hi, lo)
constexpr uint32_t kChSmemBytes = kABytes + kWStages * kWStageBytes + 1024 /*align*/ + 128 /*barriers, counters*/;
static_assert(kChSmemBytes <= 232448, "shared memory budget");

// columns (col, col + 1) of A row r (tile-local) as split-bf16.  Shared-space stores: a generic store could alias the
// epilogue's global loads as far as the compiler knows, which would keep it from issuing those loads ahead.
// The stores are predicated on `on` (no branch), so the epilogue's unrolled pairs stay one basic block.
__device__ __forceinline__ void put_a2(uint8_t* s_a, int r, int col, float y0, float y1, bool on = true) {
  uint32_t hi, lo;
  split2(y0, y1, hi, lo);
  const uint32_t q = smem_u32(s_a) + (col >> 6) * (2 * kAPlane) + sw128_offset(r, col & 63);
  sts_u32_if(q, hi, on);
  sts_u32_if(q + kAPlane, lo, on);
}
__device__ __forceinline__ float csrc_at(const nero_chain_layer& L, long row, int col, bool row_ok) {
  return (L.csrc && row_ok) ? __ldcs(L.csrc + row * L.ld_csrc + col) : 0.0f;
}

// position of a weight stage in the (tile, layer, N half, 32-wide K chunk) sequence the MMAs walk; g is its index
struct WCursor {
  int tile, li, hf, kc, g;
};
struct ConsumerCtx {
  uint8_t* s_a; uint8_t* s_w; uint64_t* full; uint32_t* rel;
  int wg, w, l;
  int g;                      // weight stages consumed so far
  WCursor q;                  // the stage kWStages ahead of the next one this warp releases
  int num_tiles;
};

// the stage after q
__device__ __forceinline__ void w_advance(const nero_chain_params& p, WCursor& q) {
  const nero_chain_layer& L = p.L[q.li];
  ++q.g;
  if (++q.kc == 2 * L.k_chunks) {
    q.kc = 0;
    if (++q.hf == (L.n_pad > HN ? 2 : 1)) {
      q.hf = 0;
      if (++q.li == p.n_layers) { q.li = 0; q.tile += gridDim.x; }
    }
  }
}
// one thread: load stage q into ring slot q.g % kWStages, whose previous contents every warp has released
__device__ __forceinline__ void w_load(const nero_chain_params& p, const WCursor& q, uint8_t* s_w, uint64_t* full, int num_tiles) {
  if (q.tile >= num_tiles) return;
  const nero_chain_layer& L = p.L[q.li];
  const uint32_t plane = uint32_t(L.n_pad) * 64u;
  const int s = q.g % kWStages;
  // rows [hf*128, +rows) of the chunk's hi plane and of its lo plane; stage rows beyond them only feed unused columns
  const uint32_t bytes = min(kHalfBytes, plane - q.hf * kHalfBytes);
  const uint8_t* src = static_cast<const uint8_t*>(L.wimg) + size_t(q.kc) * 2u * plane + size_t(q.hf) * kHalfBytes;
  mbar_arrive_expect_tx(&full[s], 2u * bytes);
  weight_copy(s_w + s * kWStageBytes, src, bytes, &full[s]);
  weight_copy(s_w + s * kWStageBytes + kHalfBytes, src + plane, bytes, &full[s]);
}
// This warp is done with the stage in slot s: its warpgroup's MMAs reading it have completed.  Every warp releases every
// stage once and in order, so the stage it releases is g = u * kWStages + s (use u of slot s) and its cursor c.q is
// stage g + kWStages, the slot's next contents.  Lane 0 counts the release on the slot's counter rel[s], which never
// resets: use u is fully released when it reaches 8 (u + 1), so the add that returns 8 u + 7 is the last of the 8 warps.
// That lane loads stage g + kWStages and re-arms full[s] for it, the phase of parity (u + 1) & 1 the MMAs of that stage
// wait for; every warp has passed its wait on phase u, so the arrival cannot complete a phase still waited on.  The
// counter's acquire-release add orders the other warps' completed MMA reads of the slot before the copy that overwrites it.
__device__ __forceinline__ void w_release(const nero_chain_params& p, ConsumerCtx& c, int s) {
  if (c.l == 0 && (atom_add_acq_rel_smem(smem_u32(&c.rel[s]), 1u) & 7u) == 7u) w_load(p, c.q, c.s_w, c.full, c.num_tiles);
  w_advance(p, c.q);
  __syncwarp();
}

#ifdef NERO_CHAIN_PHASES
// Diagnostic build only (tools/chain_phases.py).  Thread 0 of each warpgroup adds the SM cycles of each phase of a layer
// to p.phase_clk[((blockIdx.x * 2 + wg) * kMaxChainLayers + li) * kChPhases + phase]; the phases are the first A
// operand's load (layer 0), the wait for the layer's first weight stage, the MMAs, the epilogue (from the last MMA's
// completion) and the closing barrier.  After 132 * 2 * kMaxChainLayers * kChPhases counters, thread 0 of each CTA adds
// its cycles and its %globaltimer nanoseconds from start to end, which converts cycles to time.
constexpr int kChPhases = 5;
enum ChPhase : int { PH_A0 = 0, PH_WAIT = 1, PH_MMA = 2, PH_EPI = 3, PH_BAR = 4 };
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void phase_mark(const nero_chain_params& p, int li, int ph, long long& t0) {
  if (p.phase_clk && (threadIdx.x & 127) == 0) {
    const long long t = clock64();
    p.phase_clk[((blockIdx.x * 2 + (threadIdx.x >> 7)) * kMaxChainLayers + li) * kChPhases + ph] += t - t0;
    t0 = t;
  }
}
#define CH_PHASE_START(t0) long long t0 = clock64()
#define CH_PHASE(li, ph, t0) phase_mark(p, li, ph, t0)
#else
#define CH_PHASE_START(t0)
#define CH_PHASE(li, ph, t0)
#endif

// the MMAs of one layer followed by its epilogue, for this thread's warpgroup
template <int KIND>
__device__ __forceinline__ void chain_layer(const nero_chain_params& p, const nero_chain_layer& L, ConsumerCtx& c, int tile,
                                            int rows_valid, int li) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  CH_PHASE_START(t_ph);
  const int nh = L.n_pad > HN ? 2 : 1;
  float acc[2][HN / 2];
  int prev = -1;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    if (hf >= nh) break;
    for (int kc = 0; kc < 2 * L.k_chunks; ++kc, ++c.g) {    // 32-wide K chunks: the A operand's 64-wide chunk kc / 2
      const int s = c.g % kWStages;
      mbar_wait(&c.full[s], (c.g / kWStages) & 1);
      if (hf == 0 && kc == 0) CH_PHASE(li, PH_WAIT, t_ph);
      const uint32_t a_hi = smem_u32(c.s_a) + (kc >> 1) * (2 * kAPlane) + 64 * (kc & 1) + c.wg * 64 * 128, a_lo = a_hi + kAPlane;
      const uint32_t b_hi = smem_u32(c.s_w) + s * kWStageBytes, b_lo = b_hi + kHalfBytes;
      fence_regs<HN / 2>(acc[hf]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 2; ++k)
        mma_split3<HN, 0, 0>(acc[hf], make_desc_k_sw128(a_hi + 32 * k), make_desc_k_sw128(a_lo + 32 * k), make_desc_k_sw64(b_hi + 32 * k),
                             make_desc_k_sw64(b_lo + 32 * k), (kc | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();
      fence_regs<HN / 2>(acc[hf]);
      if (prev >= 0) w_release(p, c, prev);     // the stage read by the previous group is free
      prev = s;
    }
  }
  wgmma_wait<0>();
  fence_regs<HN / 2>(acc[0]);
  if (nh > 1) fence_regs<HN / 2>(acc[1]);
  CH_PHASE(li, PH_MMA, t_ph);
  w_release(p, c, prev);
  // every MMA of the layer that reads this warpgroup's A rows has completed before any of them is overwritten
  named_bar(1 + c.wg, 128);

  const EpiArgs e{L.bias, L.n_bias, L.save, L.ld_save, L.H, L.ldh, L.hscale, KIND == EK_TANGENT ? nullptr : L.addend, L.ldadd,
                  L.V, L.ldv, L.out2, L.ldo2, L.tail, L.ldt, L.ncol_out, L.ncol_main, L.oscale, L.act, L.act_param};
  const int rl0 = c.wg * 64 + c.w * 16 + (c.l >> 2);
  const bool ok0 = rl0 < rows_valid, ok1 = rl0 + 8 < rows_valid;
  // Plain layer: all 256 accumulator columns are main columns (no tail, no skip-concat columns, next A exactly 256 wide),
  // every bias column exists, and the outputs take 8-byte pair stores (H, V and the addend do: checked at launch).  Then
  // no column test of the general epilogue below can fail, and the plain one runs without them.  The SDF, NeRF and
  // predictor hidden layers of every pass are plain; the skip layer, the heads and the 39-wide first layers are not.
  const bool plain = L.n_pad == 2 * HN && L.ncol_out == 2 * HN && (kBias || L.ncol_main >= 2 * HN) &&
                     (!kBias || !L.bias || L.n_bias >= 2 * HN) && pair_aligned(L.save, L.ld_save) &&
                     (KIND != EK_TANGENT || pair_aligned(L.out2, L.ldo2));
  if (plain) {
    // row pointers at this thread's column 2 (l % 4) of its rows; the columns of its pairs are immediates off them
    const int c0 = 2 * (c.l & 3);
    PlainRows pr;
    float* out[2];
    float* out2[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long row = long(tile) * CH_BM + rl0 + 8 * h;
      pr.h[h] = L.H + row * L.ldh + c0;
      pr.v[h] = L.V + row * L.ldv + c0;
      pr.a[h] = e.addend + row * L.ldadd + c0;
      pr.ok[h] = h ? ok1 : ok0;
      pr.add[h] = pr.ok[h] && e.addend;
      out[h] = L.save + row * L.ld_save + c0;
      out2[h] = L.out2 + row * L.ldo2 + c0;
    }
    const bool st_out = L.save != nullptr, st_a = L.write_a;
    const float* bias = L.bias + c0;
    // next-A byte address of column 8 jb + c0 of row rl0 + 8 h: sw128_offset's 16-byte unit (jb & 7) ^ (rl0 & 7) is
    // a_row ^ ((jb & 7) << 4) (bits 4-6 of a_row hold rl0 & 7, and nothing else of it is in those bits); the 64-wide
    // chunk jb / 8 and the row offset h are immediates
    const uint32_t a_row = (smem_u32(c.s_a) + rl0 * 128 + 2 * c0) | ((rl0 & 7) << 4);
    epi_fragment_plain<KIND, 2 * HN / 8>(pr, [&](int jb, int h, const EpiIn& in) {
      const int hf = jb / (HN / 8), i = 4 * (jb % (HN / 8)) + 2 * h;
      float b0 = 0.0f, b1 = 0.0f;
      if constexpr (kBias) {    // two 4-byte loads: a bias is a view of a parameter buffer and need not be 8-byte aligned
        if (L.bias) { b0 = __ldg(bias + 8 * jb); b1 = __ldg(bias + 8 * jb + 1); }
      }
      float2 t;
      float2 r = epi_values<KIND>(e, acc[hf][i], acc[hf][i + 1], b0, b1, in, t);
      if constexpr (KIND == EK_TANGENT) {
        if (pr.ok[h]) __stcs(reinterpret_cast<float2*>(out2[h] + 8 * jb), t);
      }
      epi_add<KIND>(e, in, r);
      if (st_out && pr.ok[h]) __stcs(reinterpret_cast<float2*>(out[h] + 8 * jb), r);
      uint32_t hi, lo;
      split2(r.x, r.y, hi, lo);
      const uint32_t q = (a_row ^ ((jb & 7) << 4)) + (jb >> 3) * (2 * kAPlane) + h * (8 * 128);
      sts_u32_if(q, hi, st_a);
      sts_u32_if(q + kAPlane, lo, st_a);
    });
  } else {
    const int nmain = kBias ? L.ncol_out : min(L.ncol_out, L.ncol_main);
    const int n_a = L.write_a ? max(L.a_blocks * 16, L.n_pad) : 0;       // next-A columns to define
    const float* csrc = L.csrc;
    const int ld_csrc = L.ld_csrc;
    const bool skip_cols = csrc && nmain < n_a;                            // some of them come from csrc
    epi_fragment<KIND, 2 * HN / 8>(e, long(tile) * CH_BM + rl0, ok0, ok1, c.l, nh * (HN / 8),
                                   [&](int jb, int h, long row, int col, bool row_ok, const EpiIn& in) {
      const int hf = jb / (HN / 8), i = 4 * (jb % (HN / 8)) + 2 * h;
      // zeros at and beyond ncol_out (>= the main columns), where it stores nothing: no branch around it
      float2 r = epi_pair<KIND>(e, row, col, row_ok, acc[hf][i], acc[hf][i + 1], in);
      // next-A columns >= nmain come from csrc (r is zero there); loads and stores are predicated, not branched around
      const float* q = csrc + row * ld_csrc + col;
      if (skip_cols && row_ok && col >= nmain) r.x = __ldcs(q);
      if (skip_cols && row_ok && col + 1 >= nmain) r.y = __ldcs(q + 1);
      put_a2(c.s_a, rl0 + 8 * h, col, r.x, r.y, col < n_a);
    });
    // next-A columns beyond the accumulator (skip-concat source or zero): each warp fills its own 16 rows
    const int extra = (n_a - L.n_pad) >> 1;
    for (int i = c.l; i < 16 * extra; i += 32) {
      const int rl = c.wg * 64 + c.w * 16 + i / extra, col = L.n_pad + 2 * (i % extra);
      const long row = long(tile) * CH_BM + rl;
      const bool row_ok = rl < rows_valid;
      put_a2(c.s_a, rl, col, csrc_at(L, row, col, row_ok), csrc_at(L, row, col + 1, row_ok));
    }
  }
  fence_proxy_async_smem();
  CH_PHASE(li, PH_EPI, t_ph);
  named_bar(1 + c.wg, 128);
  CH_PHASE(li, PH_BAR, t_ph);
}

// FAM: 0 = bias/activation epilogues (forward chains), 1 = derivative-product epilogues (gradient sweeps), 2 = tangent
// sweep.  One instantiation per family keeps the code of each kernel small.
template <int FAM>
__global__ void __launch_bounds__(kChThreads, 1) gemm_chain_kernel(const __grid_constant__ nero_chain_params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* s_a = smem;
  uint8_t* s_w = smem + kABytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(s_w + kWStages * kWStageBytes);   // [kWStages]  W stage landed
  uint32_t* rel = reinterpret_cast<uint32_t*>(full + kWStages);                  // [kWStages]  warp releases (w_release)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int M = p.m_ptr ? *p.m_ptr : p.m_cap;
  if (M > p.m_cap) M = p.m_cap;
  const int num_tiles = (M + CH_BM - 1) / CH_BM;
#ifdef NERO_CHAIN_PHASES
  const long long clk_start = clock64();
  const uint64_t ns_start = globaltimer_ns();
#endif
  if (threadIdx.x == 0) {
    for (int s = 0; s < kWStages; ++s) { mbar_init(&full[s], 1); rel[s] = 0; }
    fence_mbar_init();
  }
  __syncthreads();

  ConsumerCtx c{s_a, s_w, full, rel, warp >> 2, warp & 3, lane, 0, WCursor{int(blockIdx.x), 0, 0, 0, 0}, num_tiles};
  for (int i = 0; i < kWStages; ++i) {
    if (threadIdx.x == 0) w_load(p, c.q, s_w, full, num_tiles);
    w_advance(p, c.q);
  }
  const int n4 = p.L[0].k_chunks * 16;     // float4 columns the first layer's MMAs read (zeros beyond k_valid0)
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int rows_valid = min(CH_BM, M - tile * CH_BM);
    CH_PHASE_START(t_a0);
    // ---- first A operand: fp32 rows from HBM -> split-bf16; each warp converts its own 16 rows, 16 * n4 float4 = 8 per
    // lane and K chunk, in batches of 4 whose loads are all issued before the first conversion
    {
      for (int b = 0; b < 2 * p.L[0].k_chunks; ++b) {
        float4 x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = lane + 32 * (4 * b + u), rl = c.wg * 64 + c.w * 16 + i / n4, col = 4 * (i % n4);
          const float* q = p.A0 + (long(tile) * CH_BM + rl) * p.lda0 + col;    // 16-byte aligned: checked at launch
          x[u] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (rl < rows_valid && col < p.k_valid0) x[u] = ld_stream4(q);
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const int i = lane + 32 * (4 * b + u), rl = c.wg * 64 + c.w * 16 + i / n4, col = 4 * (i % n4);
          put_a2(s_a, rl, col, x[u].x, x[u].y);
          put_a2(s_a, rl, col + 2, x[u].z, x[u].w);
        }
      }
      fence_proxy_async_smem();
      named_bar(1 + c.wg, 128);
      CH_PHASE(0, PH_A0, t_a0);
    }
    for (int li = 0; li < p.n_layers; ++li) {
      const nero_chain_layer& L = p.L[li];
      if constexpr (FAM == 0) {
        if (L.kind == EK_BIAS_SOFTPLUS) chain_layer<EK_BIAS_SOFTPLUS>(p, L, c, tile, rows_valid, li);
        else if (L.kind == EK_BIAS_RELU) chain_layer<EK_BIAS_RELU>(p, L, c, tile, rows_valid, li);
        else chain_layer<EK_BIAS_GENERIC>(p, L, c, tile, rows_valid, li);
      } else if constexpr (FAM == 1) {
        if (L.kind == EK_DACT_SOFTPLUS) chain_layer<EK_DACT_SOFTPLUS>(p, L, c, tile, rows_valid, li);
        else if (L.kind == EK_DACT_RELU) chain_layer<EK_DACT_RELU>(p, L, c, tile, rows_valid, li);
        else chain_layer<EK_DACT_NONE>(p, L, c, tile, rows_valid, li);
      } else {
        chain_layer<EK_TANGENT>(p, L, c, tile, rows_valid, li);
      }
    }
  }
#ifdef NERO_CHAIN_PHASES
  if (p.phase_clk && threadIdx.x == 0) {
    unsigned long long* cta = p.phase_clk + kNumSMs * 2 * kMaxChainLayers * kChPhases + 2 * blockIdx.x;
    cta[0] += clock64() - clk_start;
    cta[1] += globaltimer_ns() - ns_start;
  }
#endif
}

// ---------------------------------------------------------------------------------------------- host side
extern "C" int nero_chain(const void* chain_params_host, void* stream) {
  if (!chain_params_host) return NERO_ERR_ARG;
  const nero_chain_params& p = *static_cast<const nero_chain_params*>(chain_params_host);
  if (p.n_layers <= 0 || p.n_layers > kMaxChainLayers || (p.lda0 & 3) || (p.k_valid0 & 3) || p.k_valid0 > 256 || !p.A0 ||
      (reinterpret_cast<uintptr_t>(p.A0) & 15))
    return NERO_ERR_ARG;
  for (int l = 0; l < p.n_layers; ++l) {
    const nero_chain_layer& L = p.L[l];
    if (L.n_pad % 16 || L.n_pad < 16 || L.n_pad > 256) return NERO_ERR_ARG;
    if (!pair_aligned(L.H, L.ldh) || !pair_aligned(L.V, L.ldv) || !pair_aligned(L.addend, L.ldadd)) return NERO_ERR_ARG;
    if (L.k_chunks < 1 || L.k_chunks > 4 || L.ncol_out > L.n_pad || !L.wimg) return NERO_ERR_ARG;
    if (L.write_a && (L.a_blocks > 16 || (l + 1 < p.n_layers && L.a_blocks < 4 * p.L[l + 1].k_chunks))) return NERO_ERR_ARG;
    if (L.kind == EK_TANGENT && (!L.H || !L.V || !L.out2)) return NERO_ERR_ARG;
    if ((L.kind == EK_DACT_SOFTPLUS || L.kind == EK_DACT_RELU) && !L.H) return NERO_ERR_ARG;
  }
  int fam = -1;
  for (int l = 0; l < p.n_layers; ++l) {
    const int k = p.L[l].kind;
    const int f = k <= EK_BIAS_GENERIC ? 0 : (k == EK_TANGENT ? 2 : 1);
    if (fam >= 0 && f != fam) return NERO_ERR_ARG;   // a chain is homogeneous: forward, gradient sweep or tangent sweep
    fam = f;
  }
  const int tiles_cap = (p.m_cap + CH_BM - 1) / CH_BM;
  if (tiles_cap <= 0) return NERO_OK;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(gemm_chain_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_chain_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChSmemBytes) != cudaSuccess ||
        cudaFuncSetAttribute(gemm_chain_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChSmemBytes) != cudaSuccess)
      return NERO_ERR_CUDA;
    attr_set = true;
  }
  const int grid = tiles_cap < kNumSMs ? tiles_cap : kNumSMs;
  if (fam == 0) gemm_chain_kernel<0><<<grid, kChThreads, kChSmemBytes, (cudaStream_t)stream>>>(p);
  else if (fam == 1) gemm_chain_kernel<1><<<grid, kChThreads, kChSmemBytes, (cudaStream_t)stream>>>(p);
  else gemm_chain_kernel<2><<<grid, kChThreads, kChSmemBytes, (cudaStream_t)stream>>>(p);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
