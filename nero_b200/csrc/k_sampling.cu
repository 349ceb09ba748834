// NeuS hierarchical sampling kernels (network/renderer.py:403-443, 355-401; network/field.py:399-429):
//   sample_init  : coarse inner z (n_samples), background inverse-depth z (n_bg), PE rows of the coarse points
//   upsample     : ONE WARP PER RAY -- finite-difference cos, min with the previous section, NeuS alpha at the
//                  clipped inv_s, transmittance product, pdf/cdf, inverse-CDF at the 16 deterministic u's
//                  (searchsorted right=True), PE rows of the 16 new points.  The two scans run sequentially in
//                  one lane on shared memory, in torch's cumprod/cumsum order, because the inverse CDF is
//                  ill-conditioned where a bin's mass is ~1e-5 (see DESIGN.md "sampling parity").
//   merge        : rank-merge of the 16 sorted new samples into the sorted list (replaces torch.sort + gather,
//                  renderer.py:391-399), optionally carrying the SDF values.
//   occ_*        : the occlusion-loss march (field.py:432-484) reusing the same per-ray machinery.
#include "common.cuh"
#include "math_enc.cuh"

namespace nero {

constexpr float kInvSqrt2s = 0.70710678118654752440f;
constexpr int kMaxN = 128;   // max samples per ray handled by the warp kernels

__device__ __forceinline__ float sigmoid_t(float x) { return 1.0f / (1.0f + expf(-x)); }

__device__ __forceinline__ void write_pe_rows(const float* o, const float* d, float z, float* x0_row, float* hc_row) {
  float p[3];
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[c], __fmul_rn(d[c], z));
  float pe[39];
  pe_encode<3>(p, 6, pe);
  for (int c = 0; c < 39; ++c) { x0_row[c] = pe[c]; hc_row[217 + c] = pe[c] * kInvSqrt2s; }
}

struct SampleInitParams {
  const float* rays_o; const float* rays_d; const float* near; const float* far; int R;
  int n; int nb;
  const float* lin_inner;      // torch.linspace(0,1,n)
  const float* bg_base;        // linspace(1e-3, 1-1/(nb+1), nb)
  const float* bg_lower; const float* bg_upper;   // stratification bounds (renderer.py:419-421)
  const float* rand_inner;     // [R] or null
  const float* rand_bg;        // [R,nb] or null
  float* z; int ldz;           // [R, ldz] inner samples (first n)
  float* z_bg; int ldzb;       // [R, ...] background samples (nb)
  float* X0; int ldx; float* HC; int ldh;   // PE rows of point (r*n + j)
};

__global__ void sample_init_kernel(const SampleInitParams q) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int r = idx / q.n, j = idx % q.n;
  if (r >= q.R) return;
  const float near = q.near[r], far = q.far[r];
  float z = __fadd_rn(near, __fmul_rn(__fsub_rn(far, near), q.lin_inner[j]));
  if (q.rand_inner) z = __fadd_rn(z, __fdiv_rn(__fmul_rn(__fsub_rn(q.rand_inner[r], 0.5f), 2.0f), float(q.n)));
  q.z[size_t(r) * q.ldz + j] = z;
  const float o[3] = {q.rays_o[r * 3], q.rays_o[r * 3 + 1], q.rays_o[r * 3 + 2]};
  const float d[3] = {q.rays_d[r * 3], q.rays_d[r * 3 + 1], q.rays_d[r * 3 + 2]};
  write_pe_rows(o, d, z, q.X0 + size_t(idx) * q.ldx, q.HC + size_t(idx) * q.ldh);
  if (j < q.nb) {
    // z_bg[r, j] = far / flip(zo)[j] + 1/nb
    const int k = q.nb - 1 - j;
    float zo = q.bg_base[k];
    if (q.rand_bg) zo = __fadd_rn(q.bg_lower[k], __fmul_rn(__fsub_rn(q.bg_upper[k], q.bg_lower[k]), q.rand_bg[size_t(r) * q.nb + k]));
    q.z_bg[size_t(r) * q.ldzb + j] = __fadd_rn(__fdiv_rn(far, zo), 1.0f / float(q.nb));
  }
}

struct UpsampleParams {
  const float* rays_o; const float* rays_d; int R;
  const float* z; int ldz; const float* sdf; int lds; int n;
  int n_new;                       // 16
  const float* variance; float inv_s_cap; int clip;   // inv_s = clip ? min(exp(10 var), cap) : cap
  int surface_variant;             // 0: renderer.upsample, 1: field.get_weights (occlusion march)
  float* new_z; int ldn;           // [R, n_new]
  float* X0; int ldx; float* HC; int ldh;     // PE rows of new point (r*n_new + k); may be null
  float* wsum;                     // [R] sum of weights (occlusion ground truth) or null
  const float* origins;            // occ variant: per-ray origin/dir come from rays_o/rays_d directly
};

// weights of the n-1 sections of one ray -> s_w; returns nothing.  Lane-parallel part + sequential scans.
__device__ __forceinline__ void section_weights(const UpsampleParams& q, int lane, const float* o, const float* d,
                                                const float* s_z, const float* s_sdf, float* s_cos, float* s_w, float inv_s) {
  const int n = q.n;
  for (int j = lane; j < n - 1; j += 32)
    s_cos[j] = __fdiv_rn(__fsub_rn(s_sdf[j + 1], s_sdf[j]), __fadd_rn(__fsub_rn(s_z[j + 1], s_z[j]), 1e-5f));
  __syncwarp();
  for (int j = lane; j < n - 1; j += 32) {
    const float zp = s_z[j], zn = s_z[j + 1];
    float cosv, mask = 1.0f;
    if (q.surface_variant) {
      const float c = s_cos[j];
      mask = c < 0.f ? 1.0f : 0.0f;             // field.py:441-442
      cosv = fminf(c, 0.0f);
    } else {
      const float prev = j > 0 ? s_cos[j - 1] : 0.0f;
      cosv = fminf(prev, s_cos[j]);             // renderer.py:370-372
      cosv = fminf(fmaxf(cosv, -1e3f), 0.0f);
      float pa[3], pb[3];
      for (int c = 0; c < 3; ++c) { pa[c] = __fadd_rn(o[c], __fmul_rn(d[c], zp)); pb[c] = __fadd_rn(o[c], __fmul_rn(d[c], zn)); }
      const float ra = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(pa[0], pa[0]), __fmul_rn(pa[1], pa[1])), __fmul_rn(pa[2], pa[2])));
      const float rb = sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(pb[0], pb[0]), __fmul_rn(pb[1], pb[1])), __fmul_rn(pb[2], pb[2])));
      const bool inside = (ra < 1.0f) || (rb < 1.0f);
      cosv = inside ? cosv : 0.0f * cosv;
    }
    const float mid = __fmul_rn(__fadd_rn(s_sdf[j], s_sdf[j + 1]), 0.5f);
    const float dist = __fsub_rn(zn, zp);
    const float half = __fmul_rn(__fmul_rn(cosv, dist), 0.5f);
    const float pc = sigmoid_t(__fmul_rn(__fsub_rn(mid, half), inv_s));
    const float nc = sigmoid_t(__fmul_rn(__fadd_rn(mid, half), inv_s));
    float alpha = __fdiv_rn(__fadd_rn(__fsub_rn(pc, nc), 1e-5f), __fadd_rn(pc, 1e-5f));
    alpha = alpha * mask;
    s_w[j] = alpha;   // alpha for now
  }
  __syncwarp();
  if (lane == 0) {   // weights = alpha * cumprod([1, 1 - alpha + 1e-7])[:-1]  (sequential, torch order)
    float T = 1.0f;
    for (int j = 0; j < n - 1; ++j) {
      const float a = s_w[j];
      s_w[j] = __fmul_rn(a, T);
      T = __fmul_rn(T, __fadd_rn(__fsub_rn(1.0f, a), 1e-7f));
    }
  }
  __syncwarp();
}

__global__ void upsample_kernel(const UpsampleParams q) {
  __shared__ float sh[4][4 * kMaxN + 8];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + wib;
  if (r >= q.R) return;
  float* s_z = sh[wib];
  float* s_sdf = s_z + kMaxN;
  float* s_cos = s_sdf + kMaxN;
  float* s_w = s_cos + kMaxN;   // weights, then cdf (n entries incl. leading 0) -- cdf stored in s_cos after use
  const int n = q.n;
  const float o[3] = {q.rays_o[r * 3], q.rays_o[r * 3 + 1], q.rays_o[r * 3 + 2]};
  const float d[3] = {q.rays_d[r * 3], q.rays_d[r * 3 + 1], q.rays_d[r * 3 + 2]};
  for (int j = lane; j < n; j += 32) { s_z[j] = q.z[size_t(r) * q.ldz + j]; s_sdf[j] = q.sdf[size_t(r) * q.lds + j]; }
  __syncwarp();
  const float inv_full = expf(q.variance[0] * 10.0f);
  const float inv_s = q.clip ? fminf(inv_full, q.inv_s_cap) : q.inv_s_cap;
  section_weights(q, lane, o, d, s_z, s_sdf, s_cos, s_w, inv_s);
  if (q.wsum) {   // occlusion ground truth: sum of the section weights (renderer.py:545)
    float t = 0.f;
    for (int j = lane; j < n - 1; j += 32) t += s_w[j];
    for (int of = 16; of > 0; of >>= 1) t += __shfl_xor_sync(0xffffffffu, t, of);
    if (lane == 0) q.wsum[r] = t;
  }
  if (!q.new_z) return;
  // sample_pdf (field.py:399-429, det=True)
  float part = 0.f;
  for (int j = lane; j < n - 1; j += 32) { s_w[j] = __fadd_rn(s_w[j], 1e-5f); part += s_w[j]; }
  for (int of = 16; of > 0; of >>= 1) part += __shfl_xor_sync(0xffffffffu, part, of);
  __syncwarp();
  float* s_cdf = s_cos;   // reuse
  if (lane == 0) {
    float c = 0.0f;
    s_cdf[0] = 0.0f;
    for (int j = 0; j < n - 1; ++j) { c = __fadd_rn(c, __fdiv_rn(s_w[j], part)); s_cdf[j + 1] = c; }
  }
  __syncwarp();
  if (lane < q.n_new) {
    const int m = q.n_new;
    // torch.linspace(0.5/m, 1-0.5/m, m)
    const float start = 0.5f / m, end = 1.0f - 0.5f / m;
    const float step = (end - start) / float(m - 1);
    const float u = lane < m / 2 ? start + step * lane : end - step * (m - 1 - lane);
    // searchsorted(right=True): first index with cdf[idx] > u
    int lo = 0, hi = n;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_cdf[mid] > u) hi = mid; else lo = mid + 1; }
    const int below = max(lo - 1, 0), above = min(n - 1, lo);
    const float cb = s_cdf[below], ca = s_cdf[above];
    float denom = __fsub_rn(ca, cb);
    if (denom < 1e-5f) denom = 1.0f;
    const float t = __fdiv_rn(__fsub_rn(u, cb), denom);
    const float zb = s_z[below], za = s_z[above];
    const float zs = __fadd_rn(zb, __fmul_rn(t, __fsub_rn(za, zb)));
    q.new_z[size_t(r) * q.ldn + lane] = zs;
    if (q.X0) {
      const size_t row = size_t(r) * q.n_new + lane;
      write_pe_rows(o, d, zs, q.X0 + row * q.ldx, q.HC + row * q.ldh);
    }
  }
}

// merge sorted z[R,n] (+sdf) with sorted new_z[R,m] (+new_sdf) -> out_z[R,n+m] (+out_sdf)
__global__ void merge_kernel(const float* __restrict__ z, int ldz, const float* __restrict__ sdf, int lds, int n,
                             const float* __restrict__ nz, int ldn, const float* __restrict__ nsdf, int ldns, int m,
                             float* oz, int ldoz, float* osdf, int ldos, int R) {
  __shared__ float sh[4][kMaxN + 32];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * 4 + wib;
  if (r >= R) return;
  float* s_z = sh[wib];
  float* s_n = s_z + kMaxN;
  for (int j = lane; j < n; j += 32) s_z[j] = z[size_t(r) * ldz + j];
  for (int j = lane; j < m; j += 32) s_n[j] = nz[size_t(r) * ldn + j];
  __syncwarp();
  for (int j = lane; j < n; j += 32) {
    const float v = s_z[j];
    int cnt = 0;
    for (int k = 0; k < m; ++k) cnt += s_n[k] < v ? 1 : 0;
    oz[size_t(r) * ldoz + j + cnt] = v;
    if (osdf) osdf[size_t(r) * ldos + j + cnt] = sdf[size_t(r) * lds + j];
  }
  for (int k = lane; k < m; k += 32) {
    const float v = s_n[k];
    int lo = 0, hi = n;   // number of old entries <= v
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_z[mid] <= v) lo = mid + 1; else hi = mid; }
    oz[size_t(r) * ldoz + k + lo] = v;
    if (osdf) osdf[size_t(r) * ldos + k + lo] = nsdf[size_t(r) * ldns + k];
  }
}

// occlusion march set-up (field.py:464-475): for selected point p and direction dir:
//   max_dist = -d.p + sqrt((d.p)^2 - |p|^2 + 1 + 1e-6);  z_j = max_dist * linspace(0,1,sn0)[j];  PE rows of p + z_j d
__global__ void occ_init_kernel(const float* __restrict__ pts, const float* __restrict__ refl, const int* __restrict__ sel,
                                const int* p_ptr, int p_cap, int sn0, const float* __restrict__ lin, float* o_out,
                                float* d_out, float* z, int ldz, float* X0, int ldx, float* HC, int ldh) {
  int P = p_ptr ? *p_ptr : p_cap;
  if (P > p_cap) P = p_cap;
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const int pi = idx / sn0, j = idx % sn0;
  if (pi >= P) return;
  const int i = sel[pi];
  const float4 p4 = *reinterpret_cast<const float4*>(pts + size_t(i) * 4);
  const float4 r4 = *reinterpret_cast<const float4*>(refl + size_t(i) * 4);
  const float o[3] = {p4.x, p4.y, p4.z}, d[3] = {r4.x, r4.y, r4.z};
  const float dtx = o[0] * d[0] + o[1] * d[1] + o[2] * d[2];
  const float xtx = o[0] * o[0] + o[1] * o[1] + o[2] * o[2];
  const float md = -dtx + sqrtf(dtx * dtx - xtx + 1.0f + 1e-6f);
  const float zz = __fmul_rn(md, lin[j]);
  z[size_t(pi) * ldz + j] = zz;
  if (j == 0) for (int c = 0; c < 3; ++c) { o_out[pi * 3 + c] = o[c]; d_out[pi * 3 + c] = d[c]; }
  // points = z * dirs + origins (field.py:433)
  float p[3];
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(__fmul_rn(zz, d[c]), o[c]);
  float pe[39];
  pe_encode<3>(p, 6, pe);
  float* x0 = X0 + size_t(idx) * ldx;
  float* hc = HC + size_t(idx) * ldh;
  for (int c = 0; c < 39; ++c) { x0[c] = pe[c]; hc[217 + c] = pe[c] * kInvSqrt2s; }
}

// candidate mask of the occlusion loss (renderer.py:530-533) and compaction in sample order, in two passes: pass 0 stores
// each block's candidate count, pass 1 recomputes the mask and writes the candidates at the block's offset (the sum of the
// counts of the blocks before it).  The list is the same every run, so is the random subset drawn from it.
constexpr int kOccMaxBlocks = 16384;
__device__ int occ_block_counts[kOccMaxBlocks];

template <int PASS>
__global__ void occ_select_kernel(const float* __restrict__ pts, const float* __restrict__ Y8, int ldy, int sdf_col,
                                  const float* __restrict__ G, const int* __restrict__ ray_in, const float* __restrict__ rays_d,
                                  float sdf_thresh, const int* m_ptr, int m_cap, int* sel, int* count) {
  __shared__ int s_warp[32];
  __shared__ int s_base;
  int M = m_ptr ? *m_ptr : m_cap;
  if (M > m_cap) M = m_cap;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int flag = 0;
  if (i < M) {
    const float4 p = *reinterpret_cast<const float4*>(pts + size_t(i) * 4);
    const float4 g = *reinterpret_cast<const float4*>(G + size_t(i) * 4);
    const int r = ray_in[i];
    float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
    const float dn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
    const float nd = (g.x * d[0] + g.y * d[1] + g.z * d[2]) / dn;
    const float nrm = sqrtf(p.x * p.x + p.y * p.y + p.z * p.z);
    flag = (nrm < 0.999f) && (fabsf(Y8[size_t(i) * ldy + sdf_col]) < sdf_thresh) && (nd < 0.f);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  const int wcnt = __popc(bal), wrank = __popc(bal & ((1u << lane) - 1u));
  if (lane == 0) s_warp[warp] = wcnt;
  __syncthreads();
  if (warp == 0) {
    int v = lane < (blockDim.x >> 5) ? s_warp[lane] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    s_warp[lane] = incl - v;
    if (PASS == 0 && lane == 31) occ_block_counts[blockIdx.x] = incl;
    if (PASS == 1) {
      int base = 0;
      for (int b = lane; b < int(blockIdx.x); b += 32) base += occ_block_counts[b];
      for (int o = 16; o > 0; o >>= 1) base += __shfl_xor_sync(0xffffffffu, base, o);
      if (lane == 31) {
        s_base = base;
        if (blockIdx.x == gridDim.x - 1) *count = base + incl;
      }
    }
  }
  if (PASS == 0) return;
  __syncthreads();
  if (flag) sel[s_base + s_warp[warp] + wrank] = i;
}

// L1 occlusion loss pieces: loss_sum += |occ_prob[sel] - gt| ; docc[sel] = sign(..) (scaled by 1/P on the host side).
// One block, summed in a fixed order (the subset holds at most a few thousand points).
constexpr int kOccLossThreads = 1024;
__global__ void occ_loss_kernel(const float* __restrict__ occ_prob, const float* __restrict__ gt, const int* __restrict__ sel,
                                const int* p_ptr, int p_cap, float* loss_sum, float* docc_sign) {
  __shared__ float s_l[kOccLossThreads];
  int P = p_ptr ? *p_ptr : p_cap;
  if (P > p_cap) P = p_cap;
  float l = 0.f;
  for (int pi = threadIdx.x; pi < P; pi += blockDim.x) {
    const int i = sel[pi];
    const float df = occ_prob[i] - gt[pi];
    l += fabsf(df);
    docc_sign[i] = df > 0.f ? 1.0f : (df < 0.f ? -1.0f : 0.0f);
  }
  s_l[threadIdx.x] = l;
  __syncthreads();
  for (int h = blockDim.x >> 1; h > 0; h >>= 1) {
    if (int(threadIdx.x) < h) s_l[threadIdx.x] += s_l[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *loss_sum += s_l[0];
}

static inline int blocks_for(long n, int per) { return int((n + per - 1) / per); }

extern "C" {

int nero_sample_init(const float* rays_o, const float* rays_d, const float* near, const float* far, int R, int n, int nb,
                     const float* lin_inner, const float* bg_base, const float* bg_lower, const float* bg_upper,
                     const float* rand_inner, const float* rand_bg, float* z, int ldz, float* z_bg, int ldzb,
                     float* X0, int ldx, float* HC, int ldh, void* stream) {
  if (R <= 0) return NERO_OK;
  if (nb > n) return NERO_ERR_ARG;
  const SampleInitParams q{rays_o, rays_d, near, far, R, n, nb, lin_inner, bg_base, bg_lower, bg_upper, rand_inner, rand_bg, z, ldz, z_bg,
                           ldzb, X0, ldx, HC, ldh};
  sample_init_kernel<<<blocks_for(long(R) * n, 128), 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_upsample(const float* rays_o, const float* rays_d, int R, const float* z, int ldz, const float* sdf, int lds, int n, int n_new,
                  const float* variance, float inv_s_cap, int clip, int surface_variant, float* new_z, int ldn,
                  float* X0, int ldx, float* HC, int ldh, float* wsum, void* stream) {
  if (R <= 0) return NERO_OK;
  if (n > kMaxN || n_new > 32 || n < 2) return NERO_ERR_ARG;
  const UpsampleParams q{rays_o, rays_d, R, z, ldz, sdf, lds, n, n_new, variance, inv_s_cap, clip, surface_variant, new_z, ldn, X0, ldx, HC,
                         ldh, wsum, nullptr};
  upsample_kernel<<<blocks_for(R, 4), 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_merge_samples(const float* z, int ldz, const float* sdf, int lds, int n, const float* nz, int ldn, const float* nsdf, int ldns,
                       int m, float* oz, int ldoz, float* osdf, int ldos, int R, void* stream) {
  if (R <= 0) return NERO_OK;
  if (n > kMaxN || m > 32) return NERO_ERR_ARG;
  merge_kernel<<<blocks_for(R, 4), 128, 0, (cudaStream_t)stream>>>(z, ldz, sdf, lds, n, nz, ldn, nsdf, ldns, m, oz, ldoz, osdf, ldos, R);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_occ_init(const float* pts, const float* refl, const int* sel, const int* p_ptr, int p_cap, int sn0, const float* lin,
                  float* o_out, float* d_out, float* z, int ldz, float* X0, int ldx, float* HC, int ldh, void* stream) {
  if (p_cap <= 0) return NERO_OK;
  occ_init_kernel<<<blocks_for(long(p_cap) * sn0, 128), 128, 0, (cudaStream_t)stream>>>(pts, refl, sel, p_ptr, p_cap, sn0, lin, o_out, d_out, z,
                                                                                        ldz, X0, ldx, HC, ldh);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_occ_select(const float* pts, const float* Y8, int ldy, int sdf_col, const float* G, const int* ray_in, const float* rays_d,
                    float sdf_thresh, const int* m_ptr, int m_cap, int* sel, int* count, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const int nb = blocks_for(m_cap, 1024);
  if (nb > kOccMaxBlocks) return NERO_ERR_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  occ_select_kernel<0><<<nb, 1024, 0, st>>>(pts, Y8, ldy, sdf_col, G, ray_in, rays_d, sdf_thresh, m_ptr, m_cap, sel, count);
  occ_select_kernel<1><<<nb, 1024, 0, st>>>(pts, Y8, ldy, sdf_col, G, ray_in, rays_d, sdf_thresh, m_ptr, m_cap, sel, count);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_occ_loss(const float* occ_prob, const float* gt, const int* sel, const int* p_ptr, int p_cap, float* loss_sum, float* docc_sign,
                  void* stream) {
  if (p_cap <= 0) return NERO_OK;
  occ_loss_kernel<<<1, kOccLossThreads, 0, (cudaStream_t)stream>>>(occ_prob, gt, sel, p_ptr, p_cap, loss_sum, docc_sign);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
