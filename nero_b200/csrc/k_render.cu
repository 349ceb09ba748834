// Warp-per-ray / per-sample kernels of render_core (network/renderer.py:550-606):
//   ray_classify / ray_scan / ray_fill : section lengths, mid-points, inside-unit-sphere masks and ORDERED
//       compaction of inner / outer samples (replaces points[inner_mask], alpha[inner_mask]=..., the host syncs
//       of torch.sum(mask)>0 at renderer.py:567,570) + positional encodings of both sample sets
//   sdf_alpha fwd/bwd  : NeuS SDF->alpha with cos annealing and the eikonal term (renderer.py:484-512, :574)
//   pe_grad / pe_tangent : the PE Jacobian ends of the analytic SDF-gradient sweeps (field.py:155-167)
//   nerf_post fwd/bwd  : density/colour activation of the outer NeRF (renderer.py:346-347, 514-520)
//   composite fwd/bwd  : alpha compositing w = a * cumprod(1 - a + 1e-7), rgb = sum w c (renderer.py:578-579)
#include "common.cuh"
#include "math_shade.cuh"
#include "tile_io.cuh"

namespace nero {

constexpr float kInvSqrt2 = 0.70710678118654752440f;
static inline int blocks_for(long n, int per) { return int((n + per - 1) / per); }

__device__ __forceinline__ int load_count(const int* p, int cap) {
  int m = p ? *p : cap;
  return m > cap ? cap : m;
}

// mid-point of sample j of ray r and its section length, exactly as renderer.py:554-558 (no FMA contraction)
__device__ __forceinline__ void sample_point(const float* __restrict__ z, int S, int j, const float* o, const float* d,
                                             float* p, float* dist) {
  const float zj = z[j];
  const float ds = (j + 1 < S) ? __fsub_rn(z[j + 1], zj) : __fsub_rn(zj, z[j - 1]);
  const float mid = __fadd_rn(zj, __fmul_rn(ds, 0.5f));
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[c], __fmul_rn(d[c], mid));
  *dist = ds;
}
__device__ __forceinline__ float norm3_rn(const float* p) {
  return sqrtf(__fadd_rn(__fadd_rn(__fmul_rn(p[0], p[0]), __fmul_rn(p[1], p[1])), __fmul_rn(p[2], p[2])));
}

__global__ void ray_classify_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ z_vals, int R, int S, int* cnt_in, int* cnt_out) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const float o[3] = {rays_o[r * 3], rays_o[r * 3 + 1], rays_o[r * 3 + 2]};
  const float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  int nin = 0;
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    bool inner = false;
    if (j < S) {
      float p[3], dist;
      sample_point(z_vals + size_t(r) * S, S, j, o, d, p, &dist);
      inner = norm3_rn(p) <= 1.0f;
    }
    nin += __popc(__ballot_sync(0xffffffffu, inner));
  }
  if (lane == 0) { cnt_in[r] = nin; cnt_out[r] = S - nin; }
}

// single-block exclusive scan of the per-ray counts; totals -> n_in / n_out (device ints)
__global__ void ray_scan_kernel(const int* cnt_in, const int* cnt_out, int R, int* off_in, int* off_out, int* n_in, int* n_out) {
  __shared__ int s_in[1024], s_out[1024];
  __shared__ int carry_in, carry_out;
  if (threadIdx.x == 0) { carry_in = 0; carry_out = 0; }
  __syncthreads();
  for (int base = 0; base < R; base += 1024) {
    const int i = base + threadIdx.x;
    int a = i < R ? cnt_in[i] : 0, b = i < R ? cnt_out[i] : 0;
    s_in[threadIdx.x] = a; s_out[threadIdx.x] = b;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      int ta = 0, tb = 0;
      if (threadIdx.x >= o) { ta = s_in[threadIdx.x - o]; tb = s_out[threadIdx.x - o]; }
      __syncthreads();
      s_in[threadIdx.x] += ta; s_out[threadIdx.x] += tb;
      __syncthreads();
    }
    if (i < R) { off_in[i] = carry_in + s_in[threadIdx.x] - a; off_out[i] = carry_out + s_out[threadIdx.x] - b; }
    __syncthreads();
    if (threadIdx.x == 1023) { carry_in += s_in[1023]; carry_out += s_out[1023]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { *n_in = carry_in; *n_out = carry_out; }
}

struct FillParams {
  const float* rays_o; const float* rays_d; const float* z_vals; int R; int S;
  const int* off_in; const int* off_out;
  int* slot;                       // [R,S]: inner index i >= 0, outer index encoded as -1-io
  float* pts; int* ray_in;         // [cap_in,4] (x,y,z,dist), [cap_in]
  float* X0; int ld_x0;            // PE6(p) (39) -> cols [0,39)
  float* Y8; int ld_y8;            // p -> cols [256,259)
  float* H4; int ld_h4;            // PE6(p)/sqrt2 -> cols [217,256)
  float* XN; int ld_xn;            // outer: PE10([p/|p|, 1/|p|]) (84)
  float* H5; int ld_h5;            // outer: same 84 columns (skip concat of the NeRF MLP, field.py:268-269)
  float* FV; int ld_fv;            // outer: PE4(-dir) (27) -> cols [256,283)
  float* dist_out; int* ray_out;   // [cap_out]
};

// one warp per ray; the encoded rows are staged per warp (tile_io.cuh): within a 32-sample step the inner samples of the warp
// are consecutive rows of the compacted inner matrices (and likewise the outer ones), so each group is stored as whole rows
constexpr int kFillLd = 85;          // PE10 of 4 coordinates = 84 columns, + 1
constexpr int kFillWarps = 4;
__global__ void __launch_bounds__(kFillWarps * 32) ray_fill_kernel(const FillParams q) {
  __shared__ float s_tile[kFillWarps][32][kFillLd];
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= q.R) return;
  float (*tile)[kFillLd] = s_tile[threadIdx.x >> 5];
  const int S = q.S;
  const float o[3] = {q.rays_o[r * 3], q.rays_o[r * 3 + 1], q.rays_o[r * 3 + 2]};
  const float d[3] = {q.rays_d[r * 3], q.rays_d[r * 3 + 1], q.rays_d[r * 3 + 2]};
  const float dn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
  int base_in = q.off_in[r], base_out = q.off_out[r];
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    bool valid = j < S, inner = false;
    float p[3] = {0, 0, 0}, dist = 0.f;
    if (valid) {
      sample_point(q.z_vals + size_t(r) * S, S, j, o, d, p, &dist);
      inner = norm3_rn(p) <= 1.0f;
    }
    const unsigned bi = __ballot_sync(0xffffffffu, valid && inner);
    const unsigned bo = __ballot_sync(0xffffffffu, valid && !inner);
    const unsigned lt = (1u << lane) - 1u;
    const int n_i = __popc(bi), n_o = __popc(bo);
    const int rank = inner ? __popc(bi & lt) : __popc(bo & lt);
    // ---- inner samples: rows [base_in, base_in + n_i)
    if (valid && inner) {
      const int i = base_in + rank;
      q.slot[size_t(r) * S + j] = i;
      *reinterpret_cast<float4*>(q.pts + size_t(i) * 4) = make_float4(p[0], p[1], p[2], dist);
      q.ray_in[i] = r;
      pe_encode<3>(p, 6, tile[rank]);
      float* y8 = q.Y8 + size_t(i) * q.ld_y8 + 256;
      y8[0] = p[0]; y8[1] = p[1]; y8[2] = p[2];
    }
    if (n_i) {
      warp_rows_store<kFillLd>(tile, q.X0 + size_t(base_in) * q.ld_x0, q.ld_x0, 39, n_i, lane);
      warp_rows_store<kFillLd>(tile, q.H4 + size_t(base_in) * q.ld_h4 + 217, q.ld_h4, 39, n_i, lane, kInvSqrt2);
    }
    // ---- outer samples: rows [base_out, base_out + n_o)
    if (valid && !inner) {
      const int io = base_out + rank;
      q.slot[size_t(r) * S + j] = -1 - io;
      q.dist_out[io] = dist;
      q.ray_out[io] = r;
      // renderer.py:515-516: norm = |p| ; points = cat[p/norm, 1/norm]
      const float nrm = norm3_rn(p);
      const float p4[4] = {p[0] / nrm, p[1] / nrm, p[2] / nrm, 1.0f / nrm};
      pe_encode<4>(p4, 10, tile[rank]);
    }
    if (n_o) {
      warp_rows_store<kFillLd>(tile, q.XN + size_t(base_out) * q.ld_xn, q.ld_xn, 84, n_o, lane);
      warp_rows_store<kFillLd>(tile, q.H5 + size_t(base_out) * q.ld_h5, q.ld_h5, 84, n_o, lane);
      if (valid && !inner) {
        const float view[3] = {-d[0] / dn, -d[1] / dn, -d[2] / dn};   // -F.normalize(rays_d) (renderer.py:564,568)
        pe_encode<3>(view, 4, tile[rank]);
      }
      warp_rows_store<kFillLd>(tile, q.FV + size_t(base_out) * q.ld_fv + 256, q.ld_fv, 27, n_o, lane);
    }
    base_in += n_i;
    base_out += n_o;
  }
}

// ------------------------------------------------------------------ init-sdf regulariser points (renderer.py:591-594)
// mask = |mid-point| < radius over ALL samples; ordered compaction of the points + PE rows for a value-only SDF pass
__global__ void reg_classify_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d,
                                    const float* __restrict__ z_vals, int R, int S, float radius, int* cnt) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const float o[3] = {rays_o[r * 3], rays_o[r * 3 + 1], rays_o[r * 3 + 2]};
  const float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  int n = 0;
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    bool in = false;
    if (j < S) {
      float p[3], dist;
      sample_point(z_vals + size_t(r) * S, S, j, o, d, p, &dist);
      in = norm3_rn(p) < radius;
    }
    n += __popc(__ballot_sync(0xffffffffu, in));
  }
  if (lane == 0) cnt[r] = n;
}
__global__ void reg_fill_kernel(const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ z_vals,
                                int R, int S, float radius, const int* __restrict__ off, float* pts, float* X0, int ldx, float* H4,
                                int ldh) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const float o[3] = {rays_o[r * 3], rays_o[r * 3 + 1], rays_o[r * 3 + 2]};
  const float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  int base = off[r];
  for (int j0 = 0; j0 < S; j0 += 32) {
    const int j = j0 + lane;
    bool in = false;
    float p[3] = {0, 0, 0}, dist = 0.f;
    if (j < S) {
      sample_point(z_vals + size_t(r) * S, S, j, o, d, p, &dist);
      in = norm3_rn(p) < radius;
    }
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if (in) {
      const int i = base + __popc(b & ((1u << lane) - 1u));
      *reinterpret_cast<float4*>(pts + size_t(i) * 4) = make_float4(p[0], p[1], p[2], dist);
      float pe[39];
      pe_encode<3>(p, 6, pe);
      for (int c = 0; c < 39; ++c) { X0[size_t(i) * ldx + c] = pe[c]; H4[size_t(i) * ldh + 217 + c] = pe[c] * kInvSqrt2; }
    }
    base += __popc(b);
  }
}

// arbitrary query points (validation render, renderer.py:465-482): PTS / identity ray ids / PE rows / xyz for the material input
__global__ void points_fill_kernel(const float* __restrict__ pts3, int N, float* pts, int* ray_in, float* X0, int ldx, float* Y8,
                                   int ldy, float* H4, int ldh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float p[3] = {pts3[i * 3], pts3[i * 3 + 1], pts3[i * 3 + 2]};
  if (pts) *reinterpret_cast<float4*>(pts + size_t(i) * 4) = make_float4(p[0], p[1], p[2], 0.f);
  if (ray_in) ray_in[i] = i;
  float pe[39];
  pe_encode<3>(p, 6, pe);
  for (int c = 0; c < 39; ++c) { X0[size_t(i) * ldx + c] = pe[c]; H4[size_t(i) * ldh + 217 + c] = pe[c] * kInvSqrt2; }
  if (Y8) { Y8[size_t(i) * ldy + 256] = p[0]; Y8[size_t(i) * ldy + 257] = p[1]; Y8[size_t(i) * ldy + 258] = p[2]; }
}

// ------------------------------------------------------------------ SDF-gradient sweep ends
// V[i,j] = softplus'(a)(from H) * row[j]      (first step of the reverse sweep: v_7 = sigma_7 * W_8[0,:])
__global__ void dact_times_row_kernel(const float* __restrict__ H, int ldh, const float* __restrict__ row, float* V, int ldv,
                                      int ncol, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  if (((ncol | ldh | ldv) & 3) == 0 && ((reinterpret_cast<uintptr_t>(H) | reinterpret_cast<uintptr_t>(row) | reinterpret_cast<uintptr_t>(V)) & 15) == 0) {   // float4 path (every caller: 256-wide rows)
    const int q4 = ncol >> 2;
    const unsigned total = unsigned(M) * unsigned(q4);
    for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
      const unsigned i = idx / unsigned(q4), j = (idx % unsigned(q4)) * 4u;
      const float4 h = *reinterpret_cast<const float4*>(H + size_t(i) * ldh + j);
      const float4 w = *reinterpret_cast<const float4*>(row + j);
      *reinterpret_cast<float4*>(V + size_t(i) * ldv + j) =
          make_float4(dsoftplus100_from_h(h.x) * w.x, dsoftplus100_from_h(h.y) * w.y, dsoftplus100_from_h(h.z) * w.z, dsoftplus100_from_h(h.w) * w.w);
    }
    return;
  }
  const size_t total = size_t(M) * ncol;
  for (size_t idx = blockIdx.x * size_t(blockDim.x) + threadIdx.x; idx < total; idx += size_t(gridDim.x) * blockDim.x) {
    const int i = int(idx / ncol), j = int(idx % ncol);
    V[size_t(i) * ldv + j] = dsoftplus100_from_h(H[size_t(i) * ldh + j]) * row[j];
  }
}

// Y[i,:] += a[i*lda] * X[i,:]        (abar_7 += dsdf * v_7: the sdf-row term of the value backward)
__global__ void row_axpy_kernel(const float* __restrict__ a, int lda, const float* __restrict__ X, int ldx, float* Y, int ldy,
                                int ncol, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const size_t total = size_t(M) * (ncol / 4);
  for (size_t idx = blockIdx.x * size_t(blockDim.x) + threadIdx.x; idx < total; idx += size_t(gridDim.x) * blockDim.x) {
    const int i = int(idx / (ncol / 4)), j = int(idx % (ncol / 4)) * 4;
    const float s = a[size_t(i) * lda];
    const float4 x = *reinterpret_cast<const float4*>(X + size_t(i) * ldx + j);
    float4 y = *reinterpret_cast<float4*>(Y + size_t(i) * ldy + j);
    y.x += s * x.x; y.y += s * x.y; y.z += s * x.z; y.w += s * x.w;
    *reinterpret_cast<float4*>(Y + size_t(i) * ldy + j) = y;
  }
}

// g = J_PE^T (U0 + USKIP)     (row READS stay per thread: a thread walks its own row, every sector it touches is fetched
// once and then served from L1 -- staging them through shared memory was measured 2x slower; only row WRITES are staged)
__global__ void pe_grad_kernel(const float* __restrict__ X0, int ldx, const float* __restrict__ U0, int ldu,
                               const float* __restrict__ US, int lds, float* G, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float u[39], g[3];
  for (int c = 0; c < 39; ++c) u[c] = U0[size_t(i) * ldu + c] + US[size_t(i) * lds + c];
  pe_backward<3>(X0 + size_t(i) * ldx, 6, u, g);
  *reinterpret_cast<float4*>(G + size_t(i) * 4) = make_float4(g[0], g[1], g[2], 0.f);
}

// ubar_0 = J_PE dg  -> UB0[:, 0:39];  UB4[:, 217:256] = ubar_0 / sqrt2
constexpr int kPeLd = 41;            // PE6 of 3 coordinates = 39 columns
__global__ void __launch_bounds__(128) pe_tangent_kernel(const float* __restrict__ X0, int ldx, const float* __restrict__ DG, float* UB0,
                                                         int ld0, float* UB4, int ld4, const int* m_ptr, int m_cap) {
  __shared__ float s_x[4][32][kPeLd];
  const int M = load_count(m_ptr, m_cap);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int base = blockIdx.x * blockDim.x + warp * 32;
  if (base >= M) return;
  const int rows = min(32, M - base);
  if (lane < rows) {
    const float4 dg4 = *reinterpret_cast<const float4*>(DG + size_t(base + lane) * 4);
    const float dg[3] = {dg4.x, dg4.y, dg4.z};
    pe_tangent<3>(X0 + size_t(base + lane) * ldx, 6, dg, s_x[warp][lane]);
  }
  warp_rows_store<kPeLd>(s_x[warp], UB0 + size_t(base) * ld0, ld0, 39, rows, lane);
  warp_rows_store<kPeLd>(s_x[warp], UB4 + size_t(base) * ld4 + 217, ld4, 39, rows, lane, kInvSqrt2);
}

// ------------------------------------------------------------------ SDF -> alpha
__device__ __forceinline__ float inv_s_of(const float* variance) {
  return fminf(fmaxf(expf(variance[0] * 10.0f), 1e-6f), 1e6f);   // field.py:192, renderer.py:491
}

__global__ void sdf_alpha_fwd_kernel(const float* __restrict__ Y8, int ldy, int sdf_col, const float* __restrict__ G,
                                     const float* __restrict__ pts, const int* __restrict__ ray_in,
                                     const float* __restrict__ rays_d, const float* variance, const float* car_p, float* alpha,
                                     float* gerr, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int r = ray_in[i];
  float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  const float dn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
  for (int c = 0; c < 3; ++c) d[c] /= dn;
  const float4 g4 = *reinterpret_cast<const float4*>(G + size_t(i) * 4);
  const float g[3] = {g4.x, g4.y, g4.z};
  const SdfAlphaOut o = sdf_alpha_fwd(Y8[size_t(i) * ldy + sdf_col], g, d, pts[size_t(i) * 4 + 3], inv_s_of(variance), *car_p);
  alpha[i] = o.alpha;
  gerr[i] = o.grad_err;
}

// d inv_s is a sum over all samples: each block writes its warp-ordered partial to dinvs_partials[block] and
// sdf_alpha_bwd_finish_kernel adds them up in a fixed order, so the result is the same every run (no floating-point atomics)
constexpr int kDinvsMaxBlocks = 65536;
__device__ float dinvs_partials[kDinvsMaxBlocks];

__global__ void sdf_alpha_bwd_kernel(const float* __restrict__ Y8, int ldy, int sdf_col, const float* __restrict__ G,
                                     const float* __restrict__ pts, const int* __restrict__ ray_in,
                                     const float* __restrict__ rays_d, const float* variance, const float* car_p,
                                     const float* __restrict__ dalpha, const float* __restrict__ dgerr, float* dY8, int lddy,
                                     float* DG, float* d_inv_s, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  float dis = 0.0f;
  if (i < M) {
    const int r = ray_in[i];
    float d[3] = {rays_d[r * 3], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
    const float dn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
    for (int c = 0; c < 3; ++c) d[c] /= dn;
    const float4 g4 = *reinterpret_cast<const float4*>(G + size_t(i) * 4);
    const float g[3] = {g4.x, g4.y, g4.z};
    float4 dg4 = *reinterpret_cast<float4*>(DG + size_t(i) * 4);
    float dg[3] = {dg4.x, dg4.y, dg4.z};
    float dsdf;
    dis = sdf_alpha_bwd(Y8[size_t(i) * ldy + sdf_col], g, d, pts[size_t(i) * 4 + 3], inv_s_of(variance), *car_p, dalpha[i],
                        dgerr ? dgerr[i] : 0.0f, &dsdf, dg);
    dY8[size_t(i) * lddy + sdf_col] = dsdf;
    *reinterpret_cast<float4*>(DG + size_t(i) * 4) = make_float4(dg[0], dg[1], dg[2], 0.f);
  }
  __shared__ float s_w[32];
  for (int o = 16; o > 0; o >>= 1) dis += __shfl_xor_sync(0xffffffffu, dis, o);
  if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = dis;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.0f;
    for (int wi = 0; wi < int(blockDim.x >> 5); ++wi) t += s_w[wi];
    dinvs_partials[blockIdx.x] = t;
  }
}
__global__ void sdf_alpha_bwd_finish_kernel(int nparts, float* d_inv_s) {
  __shared__ float s_t[256];
  float t = 0.0f;
  for (int i = threadIdx.x; i < nparts; i += blockDim.x) t += dinvs_partials[i];
  s_t[threadIdx.x] = t;
  __syncthreads();
  for (int h = blockDim.x >> 1; h > 0; h >>= 1) {
    if (int(threadIdx.x) < h) s_t[threadIdx.x] += s_t[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *d_inv_s += s_t[0];
}

// ------------------------------------------------------------------ outer NeRF post
__global__ void nerf_post_fwd_kernel(const float* __restrict__ dens, int ldd, const float* __restrict__ rgb, int ldr,
                                     const float* __restrict__ dist, float* alpha, float* color, const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float a, c[3];
  nerf_post_fwd(dens[size_t(i) * ldd], dist[i], rgb + size_t(i) * ldr, &a, c);
  alpha[i] = a;
  *reinterpret_cast<float4*>(color + size_t(i) * 4) = make_float4(c[0], c[1], c[2], 0.f);
}
__global__ void nerf_post_bwd_kernel(const float* __restrict__ dens, int ldd, const float* __restrict__ rgb, int ldr,
                                     const float* __restrict__ dist, const float* __restrict__ dalpha,
                                     const float* __restrict__ dcolor, float* ddens, int lddd, float* drgb, int lddr,
                                     const int* m_ptr, int m_cap) {
  const int M = load_count(m_ptr, m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  float dd, dr[3];
  nerf_post_bwd(dens[size_t(i) * ldd], dist[i], rgb + size_t(i) * ldr, dalpha[i], dcolor + size_t(i) * 4, &dd, dr);
  ddens[size_t(i) * lddd] = dd;
  for (int c = 0; c < 3; ++c) drgb[size_t(i) * lddr + c] = dr[c];
}

// ------------------------------------------------------------------ compositing (warp per ray)
// lane l owns samples [l*SPL, (l+1)*SPL); exclusive product scan over lanes via shuffles.
template <bool BWD>
__global__ void composite_kernel(const int* __restrict__ slot, int R, int S, const float* __restrict__ a_in,
                                 const float* __restrict__ c_in, const float* __restrict__ a_out,
                                 const float* __restrict__ c_out, float* rgb, float* weights_out,
                                 const float* __restrict__ drgb, float* da_in, float* dc_in, float* da_out, float* dc_out) {
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  constexpr int MAXSPL = 8;
  const int spl = (S + 31) / 32;
  float a[MAXSPL], cr[MAXSPL], cg[MAXSPL], cb[MAXSPL];
  int sl[MAXSPL];
  float tprod = 1.0f;
#pragma unroll
  for (int k = 0; k < MAXSPL; ++k) {
    const int j = lane * spl + k;
    a[k] = 0.f; cr[k] = cg[k] = cb[k] = 0.f; sl[k] = 0;
    if (k < spl && j < S) {
      const int s = slot[size_t(r) * S + j];
      sl[k] = s;
      if (s >= 0) { a[k] = a_in[s]; const float4 c = *reinterpret_cast<const float4*>(c_in + size_t(s) * 4); cr[k] = c.x; cg[k] = c.y; cb[k] = c.z; }
      else { const int so = -1 - s; a[k] = a_out[so]; const float4 c = *reinterpret_cast<const float4*>(c_out + size_t(so) * 4); cr[k] = c.x; cg[k] = c.y; cb[k] = c.z; }
      tprod *= (1.0f - a[k] + 1e-7f);
    }
  }
  // exclusive scan of lane products
  float incl = tprod;
  for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl *= t; }
  float T = __shfl_up_sync(0xffffffffu, incl, 1);
  if (lane == 0) T = 1.0f;
  float w[MAXSPL], Tk[MAXSPL];
  float sr = 0.f, sg = 0.f, sb = 0.f;
#pragma unroll
  for (int k = 0; k < MAXSPL; ++k) {
    Tk[k] = T; w[k] = a[k] * T;
    sr += w[k] * cr[k]; sg += w[k] * cg[k]; sb += w[k] * cb[k];
    const int j = lane * spl + k;
    if (k < spl && j < S) {
      T *= (1.0f - a[k] + 1e-7f);
      if (!BWD && weights_out) weights_out[size_t(r) * S + j] = w[k];
    }
  }
  if (!BWD) {
    for (int o = 16; o > 0; o >>= 1) { sr += __shfl_xor_sync(0xffffffffu, sr, o); sg += __shfl_xor_sync(0xffffffffu, sg, o); sb += __shfl_xor_sync(0xffffffffu, sb, o); }
    if (lane == 0) { rgb[r * 3] = sr; rgb[r * 3 + 1] = sg; rgb[r * 3 + 2] = sb; }
    return;
  }
  // backward: dalpha_j = T_j s_j - (sum_{k>j} w_k s_k) / (1 - a_j + 1e-7),  s_j = drgb . c_j ;  dc_j = w_j drgb
  const float d0 = drgb[r * 3], d1 = drgb[r * 3 + 1], d2 = drgb[r * 3 + 2];
  float s[MAXSPL], lane_ws = 0.f;
#pragma unroll
  for (int k = 0; k < MAXSPL; ++k) { s[k] = d0 * cr[k] + d1 * cg[k] + d2 * cb[k]; lane_ws += w[k] * s[k]; }
  // suffix sum over lanes (exclusive): sum of lane_ws for lanes > lane
  float suf = lane_ws;
  for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_down_sync(0xffffffffu, suf, o); if (lane + o < 32) suf += t; }
  float after = suf - lane_ws;   // lanes strictly after
#pragma unroll
  for (int k = MAXSPL - 1; k >= 0; --k) {
    const int j = lane * spl + k;
    if (k < spl && j < S) {
      const float da = Tk[k] * s[k] - after / (1.0f - a[k] + 1e-7f);
      after += w[k] * s[k];
      const int sidx = sl[k];
      if (sidx >= 0) { da_in[sidx] = da; *reinterpret_cast<float4*>(dc_in + size_t(sidx) * 4) = make_float4(w[k] * d0, w[k] * d1, w[k] * d2, 0.f); }
      else { const int so = -1 - sidx; da_out[so] = da; *reinterpret_cast<float4*>(dc_out + size_t(so) * 4) = make_float4(w[k] * d0, w[k] * d1, w[k] * d2, 0.f); }
    }
  }
}

// ------------------------------------------------------------------ C ABI entry points (include/nero_b200.h)

extern "C" {

int nero_ray_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, int* cnt_in, int* cnt_out,
                     int* off_in, int* off_out, int* n_in, int* n_out, void* stream) {
  if (R <= 0) return NERO_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  ray_classify_kernel<<<blocks_for(long(R) * 32, 256), 256, 0, st>>>(rays_o, rays_d, z_vals, R, S, cnt_in, cnt_out);
  ray_scan_kernel<<<1, 1024, 0, st>>>(cnt_in, cnt_out, R, off_in, off_out, n_in, n_out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_reg_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, int* cnt, int* cnt_dummy,
                     int* off, int* off_dummy, int* n, int* n_dummy, void* stream) {
  if (R <= 0) return NERO_OK;
  const cudaStream_t st = (cudaStream_t)stream;
  reg_classify_kernel<<<blocks_for(long(R) * 32, 256), 256, 0, st>>>(rays_o, rays_d, z_vals, R, S, radius, cnt);
  ray_scan_kernel<<<1, 1024, 0, st>>>(cnt, cnt_dummy, R, off, off_dummy, n, n_dummy);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_reg_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, const int* off, float* pts,
                  float* X0, int ldx, float* H4, int ldh, void* stream) {
  if (R <= 0) return NERO_OK;
  reg_fill_kernel<<<blocks_for(long(R) * 32, 128), 128, 0, (cudaStream_t)stream>>>(rays_o, rays_d, z_vals, R, S, radius, off, pts, X0, ldx,
                                                                                   H4, ldh);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_points_fill(const float* pts3, int N, float* pts, int* ray_in, float* X0, int ldx, float* Y8, int ldy, float* H4, int ldh, void* stream) {
  if (N <= 0) return NERO_OK;
  points_fill_kernel<<<blocks_for(N, 128), 128, 0, (cudaStream_t)stream>>>(pts3, N, pts, ray_in, X0, ldx, Y8, ldy, H4, ldh);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_ray_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, const int* off_in, const int* off_out,
                  int* slot, float* pts, int* ray_in, float* X0, int ld_x0, float* Y8, int ld_y8, float* H4, int ld_h4,
                  float* XN, int ld_xn, float* H5, int ld_h5, float* FV, int ld_fv, float* dist_out, int* ray_out, void* stream) {
  if (R <= 0) return NERO_OK;
  const FillParams q{rays_o, rays_d, z_vals, R, S, off_in, off_out, slot, pts, ray_in, X0, ld_x0, Y8, ld_y8, H4, ld_h4, XN, ld_xn, H5, ld_h5,
                     FV, ld_fv, dist_out, ray_out};
  ray_fill_kernel<<<blocks_for(long(R) * 32, 128), 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_dact_times_row(const float* H, int ldh, const float* row, float* V, int ldv, int ncol, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  dact_times_row_kernel<<<kNumSMs * 8, 256, 0, (cudaStream_t)stream>>>(H, ldh, row, V, ldv, ncol, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_row_axpy(const float* a, int lda, const float* X, int ldx, float* Y, int ldy, int ncol, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  if ((ncol & 3) || (ldx & 3) || (ldy & 3)) return NERO_ERR_ARG;
  row_axpy_kernel<<<kNumSMs * 8, 256, 0, (cudaStream_t)stream>>>(a, lda, X, ldx, Y, ldy, ncol, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_pe_grad(const float* X0, int ldx, const float* U0, int ldu, const float* US, int lds, float* G, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  pe_grad_kernel<<<blocks_for(m_cap, 128), 128, 0, (cudaStream_t)stream>>>(X0, ldx, U0, ldu, US, lds, G, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_pe_tangent(const float* X0, int ldx, const float* DG, float* UB0, int ld0, float* UB4, int ld4, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  pe_tangent_kernel<<<blocks_for(m_cap, 128), 128, 0, (cudaStream_t)stream>>>(X0, ldx, DG, UB0, ld0, UB4, ld4, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_sdf_alpha_fwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, float* alpha, float* gerr, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  sdf_alpha_fwd_kernel<<<blocks_for(m_cap, 256), 256, 0, (cudaStream_t)stream>>>(Y8, ldy, sdf_col, G, pts, ray_in, rays_d, variance, car, alpha,
                                                                                 gerr, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_sdf_alpha_bwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, const float* dalpha, const float* dgerr, float* dY8, int lddy, float* DG,
                       float* d_inv_s, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const int nb = blocks_for(m_cap, 256);
  if (nb > kDinvsMaxBlocks) return NERO_ERR_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  sdf_alpha_bwd_kernel<<<nb, 256, 0, st>>>(Y8, ldy, sdf_col, G, pts, ray_in, rays_d, variance, car, dalpha, dgerr, dY8, lddy, DG, d_inv_s, m_ptr, m_cap);
  sdf_alpha_bwd_finish_kernel<<<1, 256, 0, st>>>(nb, d_inv_s);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_nerf_post_fwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, float* alpha, float* color,
                       const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  nerf_post_fwd_kernel<<<blocks_for(m_cap, 256), 256, 0, (cudaStream_t)stream>>>(dens, ldd, rgb, ldr, dist, alpha, color, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_nerf_post_bwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, const float* dalpha, const float* dcolor,
                       float* ddens, int lddd, float* drgb, int lddr, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  nerf_post_bwd_kernel<<<blocks_for(m_cap, 256), 256, 0, (cudaStream_t)stream>>>(dens, ldd, rgb, ldr, dist, dalpha, dcolor, ddens, lddd, drgb,
                                                                                 lddr, m_ptr, m_cap);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_composite_fwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       float* rgb, float* weights, void* stream) {
  if (R <= 0) return NERO_OK;
  if (S > 256) return NERO_ERR_ARG;
  composite_kernel<false><<<blocks_for(long(R) * 32, 128), 128, 0, (cudaStream_t)stream>>>(slot, R, S, a_in, c_in, a_out, c_out, rgb, weights,
                                                                                           nullptr, nullptr, nullptr, nullptr, nullptr);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_composite_bwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       const float* drgb, float* da_in, float* dc_in, float* da_out, float* dc_out, void* stream) {
  if (R <= 0) return NERO_OK;
  if (S > 256) return NERO_ERR_ARG;
  composite_kernel<true><<<blocks_for(long(R) * 32, 128), 128, 0, (cudaStream_t)stream>>>(slot, R, S, a_in, c_in, a_out, c_out, nullptr, nullptr,
                                                                                          drgb, da_in, dc_in, da_out, dc_out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
