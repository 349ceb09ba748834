// Device helpers shared by the wgmma GEMM kernels (k_gemm_linear.cu, k_gemm_chain.cu, k_gemm_wgrad.cu).
//
// Every GEMM runs as split-bf16: an fp32 operand x is stored as bf16 hi + bf16 lo (x ~= hi + lo, ~2^-17 relative) and a
// product is A_lo*B_hi + A_hi*B_lo + A_hi*B_hi (the lo*lo term, ~2^-18 relative, is dropped), accumulated in fp32.
//
// Accumulator fragment of wgmma m64nNk16 (fp32): thread t of the warpgroup (warp w = t / 32, lane l) holds d[i] at
//   row 16 w + l / 4 + 8 ((i / 2) % 2),  column 8 (i / 4) + 2 (l % 4) + (i % 2)
// i.e. pairs of adjacent columns; the epilogues below work on such pairs.
#pragma once
#include "common.cuh"
#include "ptx.cuh"

namespace nero {

// compile-time epilogue kinds
enum EpiKind : int { EK_BIAS_SOFTPLUS = 0, EK_BIAS_RELU = 1, EK_BIAS_GENERIC = 2, EK_DACT_SOFTPLUS = 3, EK_DACT_RELU = 4,
                     EK_DACT_NONE = 5, EK_TANGENT = 6 };

__device__ __forceinline__ float ex2_ftz(float x) {   // MUFU.EX2 without the denormal-range fix-up of exp2f()
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float lg2_ftz(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// fast softplus(beta=100): max error ~1e-9 absolute (ex2/lg2 approximations, 1+t rounding).  softplus(x) >= x everywhere
// and the clamped branch saturates at softplus(0.2) = 0.2 + 2e-11, so torch's threshold select is a plain max
__device__ __forceinline__ float softplus100_fast(float x) {
  const float t = lg2_ftz(1.0f + ex2_ftz(fminf(x, 0.2f) * (100.0f * 1.4426950408889634f)));
  return fmaxf(x, t * (0.6931471805599453f * 0.01f));
}
// sigma(100 a) from h = softplus(a) (possibly stored scaled by 1/hscale): 1 - 2^(-100*log2e*hscale*h); for
// 100*hscale*h > 20 the exponential is < 2.1e-9, below fp32 resolution of 1 - t, so no branch is needed
__device__ __forceinline__ float dsoftplus100_fast(float h, float hscale) {
  return 1.0f - ex2_ftz(-(100.0f * 1.4426950408889634f) * hscale * h);
}

__device__ __forceinline__ void split2(float x0, float x1, uint32_t& hi, uint32_t& lo) {
  __nv_bfloat162 h = __floats2bfloat162_rn(x0, x1);
  const uint32_t hb = *reinterpret_cast<uint32_t*>(&h);
  const float h0 = __uint_as_float(hb << 16), h1 = __uint_as_float(hb & 0xffff0000u);
  __nv_bfloat162 l = __floats2bfloat162_rn(x0 - h0, x1 - h1);
  hi = hb;
  lo = *reinterpret_cast<uint32_t*>(&l);
}

// one 16-deep k-step of the split-bf16 product for one warpgroup (small terms first)
template <int N, int TA, int TB>
__device__ __forceinline__ void mma_split3(float* d, uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, uint32_t acc) {
  Wgmma<N>::template mma<TA, TB>(d, a_lo, b_hi, acc);
  Wgmma<N>::template mma<TA, TB>(d, a_hi, b_lo, 1);
  Wgmma<N>::template mma<TA, TB>(d, a_hi, b_hi, 1);
}

// L2 policy of the GEMM kernels: every CTA re-reads each layer's weight image from L2, while a launch streams hundreds of
// MB of row operands and results that it touches once.  The weight copies are evict-last, and the row operands (first A
// operand, the chain's skip-concat source, epilogue operands) and the results are read and written with streaming
// accesses (ld / st.global.cs: evict-first), so that stream does not push the weights out of L2.  Bias vectors, which
// every CTA re-reads, keep the default policy.  On an H100 the evict-last copies alone measured no faster, but on top of
// the streaming accesses they take another ~1.8 ms off the chain launches of a step (DESIGN.md section 6).
__device__ __forceinline__ void weight_copy(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  bulk_copy_g2s(smem_dst, gmem_src, bytes, bar, l2_policy_evict_last());
}
__device__ __forceinline__ float4 ld_stream4(const float* g) { return __ldcs(reinterpret_cast<const float4*>(g)); }

// two adjacent fp32 values (col, col + 1) (col even) of one row; columns >= lim and rows that are not ok read as zero.
// g is 8-byte aligned and ld even (checked at launch), so at an even lim every pair is one 8-byte load; at an odd lim
// the last pair has one column and every pair takes two 4-byte loads.  The loads are predicated rather than branched
// around, so a caller can issue many of them before it uses the first.  Each epilogue operand is read once per launch, so
// the loads are streaming (ld.global.cs: evict-first in L1 and L2) and leave L2 to the weight images every CTA re-reads;
// with the default policy the gradient sweeps ran about 1.5x longer on an H100 (DESIGN.md section 6).
template <bool kEvenLim>
__device__ __forceinline__ float2 ld2(const float* __restrict__ g, int ld, long row, int col, int lim, bool ok) {
  const float* q = g + row * ld + col;
  float2 x = make_float2(0.f, 0.f);
  if constexpr (kEvenLim) {
    if (ok && col < lim) x = __ldcs(reinterpret_cast<const float2*>(q));
  } else {
    if (ok && col < lim) x.x = __ldcs(q);
    if (ok && col + 1 < lim) x.y = __ldcs(q + 1);
  }
  return x;
}
// an epilogue operand pointer may be null or must allow 8-byte pair loads
__host__ __device__ inline bool pair_aligned(const float* g, int ld) {
  return !g || ((reinterpret_cast<uintptr_t>(g) & 7) == 0 && (ld & 1) == 0);
}
// Written as three independently guarded stores rather than early returns, so that the compiler predicates them and the
// epilogues' unrolled pairs stay one basic block it can schedule across.
__device__ __forceinline__ void st2(float* __restrict__ g, int ld, long row, int col, int lim, bool ok, float a, float b) {
  const bool in0 = ok && g && col < lim, in1 = in0 && col + 1 < lim;
  float* q = g + row * ld + col;
  const bool pair = in1 && (reinterpret_cast<uintptr_t>(q) & 7) == 0;
  if (pair) __stcs(reinterpret_cast<float2*>(q), make_float2(a, b));
  if (in0 && !pair) __stcs(q, a);
  if (in1 && !pair) __stcs(q + 1, b);
}

// operands of the epilogue of one layer (nero_linear / one layer of nero_chain; see include/nero_b200.h)
struct EpiArgs {
  const float* bias; int n_bias;
  float* out; int ldo;
  const float* H; int ldh; float hscale;
  const float* addend; int ldadd;
  const float* V; int ldv;
  float* out2; int ldo2;
  float* tail; int ldt;
  int ncol_out, ncol_main;
  float oscale; int act; float act_param;
};

// the HBM operands H, V and addend of one column pair of a derivative-product epilogue
struct EpiIn {
  float2 h, v, a;
};
template <int KIND, bool kEvenLim>
__device__ __forceinline__ EpiIn epi_load(const EpiArgs& e, long row, int col, bool row_ok) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  EpiIn in{make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
  if constexpr (!kBias) {
    const int nmain = min(e.ncol_out, e.ncol_main);
    if constexpr (KIND != EK_DACT_NONE) in.h = ld2<kEvenLim>(e.H, e.ldh, row, col, nmain, row_ok);
    if constexpr (KIND == EK_TANGENT) in.v = ld2<kEvenLim>(e.V, e.ldv, row, col, nmain, row_ok);
    in.a = ld2<kEvenLim>(e.addend, e.ldadd, row, col, nmain, row_ok && e.addend);
  }
  return in;
}

// The arithmetic of accumulator columns (v0, v1) of one row with the bias (b0, b1) of those columns (bias kinds) or the
// operands `in` (the others): returns the values `out` stores, but for the addend (epi_add), and in the tangent sweep
// sets t to those out2 stores.  Both epilogue paths below run these same operations in this order, so they compute
// bit-identical values.
template <int KIND>
__device__ __forceinline__ float2 epi_values(const EpiArgs& e, float v0, float v1, float b0, float b1, const EpiIn& in, float2& t) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  float r0, r1;
  if constexpr (kBias) {
    float y0 = v0 + b0;
    float y1 = v1 + b1;
    if constexpr (KIND == EK_BIAS_SOFTPLUS) { y0 = softplus100_fast(y0); y1 = softplus100_fast(y1); }
    else if constexpr (KIND == EK_BIAS_RELU) { y0 = fmaxf(y0, 0.0f); y1 = fmaxf(y1, 0.0f); }
    else { y0 = apply_act(y0, e.act, e.act_param); y1 = apply_act(y1, e.act, e.act_param); }
    r0 = e.oscale * y0;
    r1 = e.oscale * y1;
  } else {
    float s0 = 1.0f, s1 = 1.0f;
    if constexpr (KIND != EK_DACT_NONE) {
      const float2 h = in.h;
      if constexpr (KIND == EK_DACT_RELU) { s0 = h.x > 0.0f ? 1.0f : 0.0f; s1 = h.y > 0.0f ? 1.0f : 0.0f; }
      else { s0 = dsoftplus100_fast(h.x, e.hscale); s1 = dsoftplus100_fast(h.y, e.hscale); }
    }
    r0 = e.oscale * s0 * v0;
    r1 = e.oscale * s1 * v1;
    if constexpr (KIND == EK_TANGENT) {
      const float2 v = in.v;
      t = make_float2(100.0f * (1.0f - s0) * v.x * v0, 100.0f * (1.0f - s1) * v.y * v1);
    }
  }
  return make_float2(r0, r1);
}
// the derivative-product epilogues' addend, added last
template <int KIND>
__device__ __forceinline__ void epi_add(const EpiArgs& e, const EpiIn& in, float2& r) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  if constexpr (!kBias) {
    if (e.addend) {
      const float2 a = in.a;
      r.x += a.x;
      r.y += a.y;
    }
  }
}

// Epilogue of accumulator columns (col, col + 1) of one row, with its operands `in` from epi_load: writes
// out / out2 / tail as the kind defines and returns the result values (those a following layer of a chain reads in the
// main columns).  Rows that are not ok are computed with zero operands and not stored.
template <int KIND>
__device__ __forceinline__ float2 epi_pair(const EpiArgs& e, long row, int col, bool row_ok, float v0, float v1, const EpiIn& in) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  const int nmain = kBias ? e.ncol_out : min(e.ncol_out, e.ncol_main);
  float b0 = 0.0f, b1 = 0.0f;
  if constexpr (kBias) {
    b0 = (e.bias && col < e.n_bias) ? __ldg(e.bias + col) : 0.0f;
    b1 = (e.bias && col + 1 < e.n_bias) ? __ldg(e.bias + col + 1) : 0.0f;
  }
  float2 t;
  float2 r = epi_values<KIND>(e, v0, v1, b0, b1, in, t);
  if constexpr (KIND == EK_TANGENT) st2(e.out2, e.ldo2, row, col, nmain, row_ok, t.x, t.y);
  epi_add<KIND>(e, in, r);
  if constexpr (!kBias) {
    // skip-branch columns [ncol_main, ncol_out) carry oscale * acc and go to the tail buffer
    if (e.tail && row_ok) {
      if (col >= e.ncol_main && col < e.ncol_out) __stcs(e.tail + row * e.ldt + (col - e.ncol_main), e.oscale * v0);
      if (col + 1 >= e.ncol_main && col + 1 < e.ncol_out) __stcs(e.tail + row * e.ldt + (col + 1 - e.ncol_main), e.oscale * v1);
    }
  }
  st2(e.out, e.ldo, row, col, nmain, row_ok, r.x, r.y);
  return make_float2(col < nmain ? r.x : 0.0f, col + 1 < nmain ? r.y : 0.0f);
}

// Column blocks (8 accumulator columns each) whose operand loads a thread issues back to back.  An epilogue that loads
// each operand right before using it keeps one load per warp in flight and runs at a fraction of HBM bandwidth; here
// the loads of group g + 1 are in flight while group g computes: 8 (16 with an addend) independent 8-byte loads per
// thread, 8 in the tangent sweep, whose two operands per pair at 4 blocks would not fit the registers beside the
// accumulators.
template <int KIND> constexpr int kEpiGroup = KIND == EK_TANGENT ? 2 : 4;

// Runs body(jb, h, row, col, row_ok, in) for every pair of this thread's accumulator fragment in column blocks jb < nb
// (nb <= NB, a multiple of the group size) and rows row0 (h = 0) and row0 + 8 (h = 1), with `in` its epi_load operands.
template <int KIND, int NB, class Body>
__device__ __forceinline__ void epi_fragment(const EpiArgs& e, long row0, bool ok0, bool ok1, int lane, int nb, Body&& body) {
  constexpr int G = NB < kEpiGroup<KIND> ? NB : kEpiGroup<KIND>;
  static_assert(NB % G == 0, "whole groups of column blocks");
  EpiIn in[2][2 * G];
  const bool even_lim = (min(e.ncol_out, e.ncol_main) & 1) == 0;
  auto load = [&](int g, EpiIn* dst) {
    if (even_lim) {
#pragma unroll
      for (int j = 0; j < G; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) dst[2 * j + h] = epi_load<KIND, true>(e, row0 + 8 * h, 8 * (g * G + j) + 2 * (lane & 3), h ? ok1 : ok0);
    } else {
#pragma unroll
      for (int j = 0; j < G; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) dst[2 * j + h] = epi_load<KIND, false>(e, row0 + 8 * h, 8 * (g * G + j) + 2 * (lane & 3), h ? ok1 : ok0);
    }
  };
  load(0, in[0]);
#pragma unroll
  for (int g = 0; g < NB / G; ++g) {
    if (g * G >= nb) break;
    if ((g + 1) * G < nb) load(g + 1, in[(g + 1) & 1]);
#pragma unroll
    for (int j = 0; j < G; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        body(g * G + j, h, row0 + 8 * h, 8 * (g * G + j) + 2 * (lane & 3), h ? ok1 : ok0, in[g & 1][2 * j + h]);
  }
}

// ---- plain layers.  A chain layer is plain when none of the per-pair tests of epi_load / epi_pair / st2 can fail for it
// (k_gemm_chain.cu: chain_layer); then each operand row is one pointer per thread, every column a compile-time offset from
// it, and only the row tests remain.  `ok`: the row exists; `add`: it exists and the layer has an addend.
struct PlainRows {
  const float* h[2]; const float* v[2]; const float* a[2];
  bool ok[2], add[2];
};
// the operands of columns (c, c + 1) of this thread's row row0 + 8 h, c relative to the row pointers of `pr`
template <int KIND>
__device__ __forceinline__ EpiIn plain_load(const PlainRows& pr, int h, int c) {
  constexpr bool kBias = (KIND == EK_BIAS_SOFTPLUS || KIND == EK_BIAS_RELU || KIND == EK_BIAS_GENERIC);
  EpiIn in{make_float2(0.f, 0.f), make_float2(0.f, 0.f), make_float2(0.f, 0.f)};
  if constexpr (!kBias) {
    if constexpr (KIND != EK_DACT_NONE) if (pr.ok[h]) in.h = __ldcs(reinterpret_cast<const float2*>(pr.h[h] + c));
    if constexpr (KIND == EK_TANGENT) if (pr.ok[h]) in.v = __ldcs(reinterpret_cast<const float2*>(pr.v[h] + c));
    if constexpr (KIND != EK_TANGENT) if (pr.add[h]) in.a = __ldcs(reinterpret_cast<const float2*>(pr.a[h] + c));
  }
  return in;
}
// epi_fragment for a plain layer: body(jb, h, in) for all NB column blocks, with the same group-ahead loads
template <int KIND, int NB, class Body>
__device__ __forceinline__ void epi_fragment_plain(const PlainRows& pr, Body&& body) {
  constexpr int G = NB < kEpiGroup<KIND> ? NB : kEpiGroup<KIND>;
  static_assert(NB % G == 0, "whole groups of column blocks");
  EpiIn in[2][2 * G];
  auto load = [&](int g, EpiIn* dst) {
#pragma unroll
    for (int j = 0; j < G; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) dst[2 * j + h] = plain_load<KIND>(pr, h, 8 * (g * G + j));
  };
  load(0, in[0]);
#pragma unroll
  for (int g = 0; g < NB / G; ++g) {
    if (g + 1 < NB / G) load(g + 1, in[(g + 1) & 1]);
#pragma unroll
    for (int j = 0; j < G; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h) body(g * G + j, h, in[g & 1][2 * j + h]);
  }
}

}  // namespace nero
