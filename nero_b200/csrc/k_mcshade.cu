// Stage II Monte-Carlo shading (MCShadingNetwork.shade_mixed / get_lights, network/field.py:858-1003) around the light
// MLPs: direction sampling, hit/miss compaction + input encodings, the estimator reduction, and their backward passes.
//
// Ray j of point p is ray index p*S + j; j < Sd are the cosine-weighted (diffuse) samples, the rest GGX (specular).
// Rays that escape the mesh become rows of the OUTER list (outer_light [+ human_light]); rays that hit become rows of the
// INNER list (inner_light at the hit point).  Both lists keep ray order (deterministic block scan), so row r of the outer
// list is the r-th miss exactly like `points[miss_mask]` in the reference.
#include "common.cuh"
#include "math_enc.cuh"
#include "math_shade.cuh"
#include "tile_io.cuh"
#include "math_mc.cuh"

namespace nero {

__constant__ IdeTable c_ide_mc;

int set_ide_table_mc(const float* mat17x36_host) {
  IdeTable t;
  int i = 0;
  for (int e = 0; e < 5; ++e) {
    const int l = 1 << e;
    for (int m = 0; m <= l; ++m) { t.m[i] = m; t.l[i] = l; ++i; }
  }
  for (int k = 0; k < 17; ++k)
    for (int j = 0; j < 36; ++j) { t.mat[k][j] = double(mat17x36_host[k * 36 + j]); t.matf[k][j] = mat17x36_host[k * 36 + j]; }
  NERO_CUDA_TRY(cudaMemcpyToSymbol(c_ide_mc, &t, sizeof(IdeTable)));
  return NERO_OK;
}

using McParams = ::nero_mc_params;

__device__ __forceinline__ void ray_direction(const McParams& q, const McPoint& pt, int p, int j, float a, float* d) {
  if (j < q.Sd) {
    const float az = mc_azimuth(q.tab_d[2 * j], q.rand_d ? q.rand_d[p] : 0.f, q.rand_d != nullptr);
    mc_diffuse_dir(pt, az, q.tab_d[2 * j + 1], d);
  } else {
    const int k = j - q.Sd;
    const float phi = mc_azimuth(q.tab_s[2 * k], q.rand_s ? q.rand_s[p] : 0.f, q.rand_s != nullptr);
    mc_specular_dir<float>(pt, phi, q.tab_s[2 * k + 1], a, d);
  }
}

// ------------------------------------------------------------------ directions + secondary-ray origins
__global__ void mc_sample_kernel(const McParams q) {
  const int S = q.Sd + q.Ss;
  const long i = long(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= long(q.P) * S) return;
  const int p = int(i / S), j = int(i % S);
  const McPoint pt = mc_point(q.normals + 3 * p, q.view + 3 * p);
  float d[3];
  ray_direction(q, pt, p, j, q.rough[p], d);
  const float* x = q.pts + 3 * p;
  *reinterpret_cast<float4*>(q.dir + i * 4) = make_float4(d[0], d[1], d[2], 0.f);
  *reinterpret_cast<float4*>(q.org + i * 4) = make_float4(x[0] + d[0] * 1e-5f, x[1] + d[1] * 1e-5f, x[2] + d[2] * 1e-5f, 0.f);
}

// ------------------------------------------------------------------ hit / miss compaction (deterministic)
constexpr int kClsBlock = 256;
__global__ void mc_count_kernel(const McParams q, long N) {
  __shared__ int s_cnt;
  if (threadIdx.x == 0) s_cnt = 0;
  __syncthreads();
  const long i = long(blockIdx.x) * kClsBlock + threadIdx.x;
  const bool hit = i < N && reinterpret_cast<const float4*>(q.nrm_hit)[i].w > 0.5f;
  const unsigned b = __ballot_sync(0xffffffffu, hit);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_cnt, __popc(b));
  __syncthreads();
  if (threadIdx.x == 0) q.blk_cnt[blockIdx.x] = s_cnt;
}
__global__ void mc_scan_kernel(const McParams q, int nblk, long N) {   // one block of 1024 threads
  __shared__ int s_part[1024];
  const int per = (nblk + 1023) / 1024;
  const int b0 = threadIdx.x * per;
  int sum = 0;
  for (int k = 0; k < per; ++k) if (b0 + k < nblk) sum += q.blk_cnt[b0 + k];
  s_part[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {
    const int v = threadIdx.x >= off ? s_part[threadIdx.x - off] : 0;
    __syncthreads();
    s_part[threadIdx.x] += v;
    __syncthreads();
  }
  int run = s_part[threadIdx.x] - sum;
  for (int k = 0; k < per; ++k)
    if (b0 + k < nblk) { q.blk_off[b0 + k] = run; run += q.blk_cnt[b0 + k]; }
  if (threadIdx.x == 1023) { q.counts[0] = s_part[1023]; q.counts[1] = int(N - s_part[1023]); }
}

// rows + encodings.  Outer row: IDE(dir, 0) [+ IDE(sphere point, 0)] and the human-light IPE; inner row: PE8(hit point) at
// columns 0..50, IDE(reflection of -dir about the hit normal, 0) at 52..123 (field.py:814-820, 822-856).
// The compaction keeps ray order, so the misses of a warp are consecutive rows of the outer matrices and its hits consecutive
// rows of the inner one: each group is staged in a per-warp tile and stored as whole rows (tile_io.cuh).  Per-thread 16-byte
// stores into 32 different rows wrote 2.6x the algorithmic bytes to DRAM (half-filled sectors evicted from L2).
constexpr int kMcTileLd = 73;
constexpr int kMcFillSmem = (kClsBlock / 32) * 32 * kMcTileLd * 4;
__global__ void __launch_bounds__(kClsBlock) mc_fill_kernel(const McParams q, long N) {
  extern __shared__ float s_mc_tiles[];
  __shared__ int s_warp[kClsBlock / 32];
  const int S = q.Sd + q.Ss;
  const long i = long(blockIdx.x) * kClsBlock + threadIdx.x;
  const bool valid = i < N;
  const float4 nh = valid ? reinterpret_cast<const float4*>(q.nrm_hit)[i] : make_float4(0, 0, 0, 0);
  const bool hit = valid && nh.w > 0.5f, miss = valid && !hit;
  const unsigned b = __ballot_sync(0xffffffffu, hit), bm = __ballot_sync(0xffffffffu, miss);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_warp[wid] = __popc(b);
  __syncthreads();
  int wbefore = q.blk_off[blockIdx.x];                  // hits before this warp
  for (int k = 0; k < wid; ++k) wbefore += s_warp[k];
  const unsigned lt = (1u << lane) - 1u;
  const int n_hit = __popc(b), n_miss = __popc(bm);
  const int rank = hit ? __popc(b & lt) : __popc(bm & lt);
  const long row_i0 = wbefore;                          // first inner row of the warp
  const long row_o0 = (i - lane) - wbefore;             // first outer row of the warp
  float (*tile)[kMcTileLd] = reinterpret_cast<float (*)[kMcTileLd]>(s_mc_tiles + size_t(wid) * 32 * kMcTileLd);
  float d[3] = {0.f, 0.f, 1.f};
  int p = 0;
  if (valid) {
    const float4 d4 = *reinterpret_cast<const float4*>(q.dir + i * 4);
    d[0] = d4.x; d[1] = d4.y; d[2] = d4.z;
    p = int(i / S);
  }
  // ---- misses -> outer rows
  if (n_miss) {
    if (miss) {
      q.slot[i] = int(row_o0 + rank);
      ide_forward(c_ide_mc, d, 0.f, tile[rank]);
    }
    float* eo = q.EO + row_o0 * q.ldeo;
    warp_rows_store4<kMcTileLd, 18>(tile, eo, q.ldeo, n_miss, lane);
    if (q.sphere_dir) {
      if (miss) {
        float sp[3], pu[3];
        mc_sphere_point(q.pts + 3 * p, d, sp, pu);
        ide_forward(c_ide_mc, sp, 0.f, tile[rank]);
      }
      warp_rows_store4<kMcTileLd, 18>(tile, eo + 72, q.ldeo, n_miss, lane);
    }
    if (q.human) {
      if (miss) {
        const HumanGeo h = human_geo_fwd(q.pts + 3 * p, d, q.poses + 12 * p, 0.f);
        const float var[2] = {0.f, 0.f};
        ipe_forward(h.mean, var, tile[rank]);
        q.hhit[row_o0 + rank] = h.hit;
      }
      warp_rows_store4<kMcTileLd, 6>(tile, q.EH + row_o0 * q.ldeh, q.ldeh, n_miss, lane);
    }
  }
  // ---- hits -> inner rows
  if (n_hit) {
    float* ei = q.EI + row_i0 * q.ldei;
    if (hit) {
      q.slot[i] = ~int(row_i0 + rank);
      const float4 pd = reinterpret_cast<const float4*>(q.pos_depth)[i];
      const float x[3] = {pd.x, pd.y, pd.z};
      pe_encode<3>(x, 8, tile[rank]);
      tile[rank][51] = 0.f;
    }
    warp_rows_store4<kMcTileLd, 13>(tile, ei, q.ldei, n_hit, lane);
    if (hit) {
      float n[3], v[3], nv[3] = {-d[0], -d[1], -d[2]};
      const float nr[3] = {nh.x, nh.y, nh.z};
      normalize3(nr, n);
      normalize3(nv, v);
      const float vn = v[0] * n[0] + v[1] * n[1] + v[2] * n[2];
      const float rf[3] = {vn * n[0] * 2.f - v[0], vn * n[1] * 2.f - v[1], vn * n[2] * 2.f - v[2]};
      ide_forward(c_ide_mc, rf, 0.f, tile[rank]);
    }
    warp_rows_store4<kMcTileLd, 18>(tile, ei + 52, q.ldei, n_hit, lane);
  }
}

// ------------------------------------------------------------------ light of one ray from the MLP outputs
struct RayLight { float L[3]; float ol[3]; float hl[3]; float hw_raw, hw, hhit; };
__device__ __forceinline__ RayLight ray_light(const McParams& q, int slot) {
  RayLight r;
  r.hw_raw = r.hw = r.hhit = 0.f;
  if (slot >= 0) {
    const float4 o = *reinterpret_cast<const float4*>(q.OUT_O + size_t(slot) * 4);
    r.ol[0] = o.x; r.ol[1] = o.y; r.ol[2] = o.z;
    r.hl[0] = r.hl[1] = r.hl[2] = 0.f;
    if (q.human) {
      const float4 h = *reinterpret_cast<const float4*>(q.OUT_H + size_t(slot) * 4);
      r.hhit = q.hhit[slot];
      r.hl[0] = h.x * r.hhit; r.hl[1] = h.y * r.hhit; r.hl[2] = h.z * r.hhit;
      r.hw_raw = h.w * r.hhit;
      r.hw = fminf(fmaxf(r.hw_raw, 0.f), 1.f);
    }
    for (int c = 0; c < 3; ++c) r.L[c] = r.ol[c] * (1.f - r.hw) + r.hl[c] * r.hw;
  } else {
    const float4 o = *reinterpret_cast<const float4*>(q.OUT_I + size_t(~slot) * 4);
    r.L[0] = o.x; r.L[1] = o.y; r.L[2] = o.z;
    r.ol[0] = r.ol[1] = r.ol[2] = 0.f; r.hl[0] = r.hl[1] = r.hl[2] = 0.f;
  }
  return r;
}

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ------------------------------------------------------------------ estimator: one warp per point
// LD = mean over diffuse samples of L;  LS = mean over all samples of L*w;  LSF = mean of L*w*(1-HoV)^5
// (specular colour = F0*LS + (1-F0)*LSF; diffuse colour = albedo*(1-metallic)*LD -- assembled by the caller).
__global__ void mc_combine_fwd_kernel(const McParams q) {
  const int S = q.Sd + q.Ss;
  const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (p >= q.P) return;
  const McPoint pt = mc_point(q.normals + 3 * p, q.view + 3 * p);
  const float a = q.rough[p];
  const float fd = float(q.Sd) / float(S), fs = float(q.Ss) / float(S);
  float acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = lane; j < S; j += 32) {
    const long i = long(p) * S + j;
    const float4 d4 = *reinterpret_cast<const float4*>(q.dir + i * 4);
    const float d[3] = {d4.x, d4.y, d4.z};
    float w, f5;
    mc_weights<float>(pt, d, a, j >= q.Sd, fd, fs, q.ggx_smith, w, f5);
    const RayLight rl = ray_light(q, q.slot[i]);
    const float near = reinterpret_cast<const float4*>(q.pos_depth)[i].w > 1e-5f ? 1.f : 0.f;
    for (int c = 0; c < 3; ++c) {
      const float L = rl.L[c] * near;
      if (j < q.Sd) acc[c] += L;
      acc[3 + c] += L * w;
      acc[6 + c] += L * w * f5;
    }
  }
  for (int k = 0; k < 9; ++k) acc[k] = warp_sum(acc[k]);
  if (lane == 0) {
    for (int c = 0; c < 3; ++c) {
      q.LD[3 * p + c] = acc[c] / float(q.Sd);
      q.LS[3 * p + c] = acc[3 + c] / float(S);
      q.LSF[3 * p + c] = acc[6 + c] / float(S);
    }
  }
}

// backward of the estimator w.r.t. the MLP outputs (pre-activation) and, through the weights, the roughness
__global__ void mc_combine_bwd_kernel(const McParams q) {
  const int S = q.Sd + q.Ss;
  const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (p >= q.P) return;
  const McPoint pt = mc_point(q.normals + 3 * p, q.view + 3 * p);
  const Dual a = mk(q.rough[p], 1.f);
  const float fd = float(q.Sd) / float(S), fs = float(q.Ss) / float(S);
  const float emax_o = expf(q.exp_max_o), emax_i = expf(q.exp_max_i);
  float gd[3], gs[3], gf[3];
  for (int c = 0; c < 3; ++c) { gd[c] = q.dLD[3 * p + c] / float(q.Sd); gs[c] = q.dLS[3 * p + c] / float(S); gf[c] = q.dLSF[3 * p + c] / float(S); }
  float da = 0.f;
  for (int j = lane; j < S; j += 32) {
    const long i = long(p) * S + j;
    Dual d[3];
    if (j < q.Sd) {
      const float4 d4 = *reinterpret_cast<const float4*>(q.dir + i * 4);
      d[0] = mk(d4.x); d[1] = mk(d4.y); d[2] = mk(d4.z);
    } else {
      const int k = j - q.Sd;
      const float phi = mc_azimuth(q.tab_s[2 * k], q.rand_s ? q.rand_s[p] : 0.f, q.rand_s != nullptr);
      mc_specular_dir<Dual>(pt, phi, q.tab_s[2 * k + 1], a, d);
    }
    Dual w, f5;
    mc_weights<Dual>(pt, d, a, j >= q.Sd, fd, fs, q.ggx_smith, w, f5);
    const int slot = q.slot[i];
    const RayLight rl = ray_light(q, slot);
    const float near = reinterpret_cast<const float4*>(q.pos_depth)[i].w > 1e-5f ? 1.f : 0.f;
    float dL[3];
    const Dual wf = w * f5;
    for (int c = 0; c < 3; ++c) {
      const float L = rl.L[c] * near;
      dL[c] = ((j < q.Sd ? gd[c] : 0.f) + gs[c] * w.v + gf[c] * wf.v) * near;
      da += L * (gs[c] * w.d + gf[c] * wf.d);
    }
    if (slot >= 0) {
      float4 po, ph = make_float4(0, 0, 0, 0);
      float* pov = reinterpret_cast<float*>(&po);
      for (int c = 0; c < 3; ++c) pov[c] = rl.ol[c] < emax_o ? dL[c] * (1.f - rl.hw) * rl.ol[c] : 0.f;
      po.w = 0.f;
      *reinterpret_cast<float4*>(q.DPRE_O + size_t(slot) * 4) = po;
      if (q.human) {
        const float4 h = *reinterpret_cast<const float4*>(q.OUT_H + size_t(slot) * 4);   // raw exp outputs (exp_max = 0)
        const float hv[4] = {h.x, h.y, h.z, h.w};
        float* phv = reinterpret_cast<float*>(&ph);
        float dhw = 0.f;
        for (int c = 0; c < 3; ++c) {
          phv[c] = hv[c] < 1.0f ? dL[c] * rl.hw * rl.hhit * hv[c] : 0.f;
          dhw += dL[c] * (rl.hl[c] - rl.ol[c]);
        }
        const float pass = (rl.hw_raw >= 0.f && rl.hw_raw <= 1.f) ? 1.f : 0.f;
        ph.w = hv[3] < 1.0f ? dhw * pass * rl.hhit * hv[3] : 0.f;
        *reinterpret_cast<float4*>(q.DPRE_H + size_t(slot) * 4) = ph;
      }
    } else {
      float4 pi;
      float* piv = reinterpret_cast<float*>(&pi);
      for (int c = 0; c < 3; ++c) piv[c] = rl.L[c] < emax_i ? dL[c] * rl.L[c] : 0.f;
      pi.w = 0.f;
      *reinterpret_cast<float4*>(q.DPRE_I + size_t(~slot) * 4) = pi;
    }
  }
  da = warp_sum(da);
  if (lane == 0) q.dA[p] = da;
}

// gradient that reaches the roughness through the sampled specular directions: encoding-input gradients of the light MLPs
// -> d(direction) -> <., d(direction)/d(roughness)>.  Diffuse directions do not depend on any learnable quantity.
__global__ void mc_dir_bwd_kernel(const McParams q) {
  const int S = q.Sd + q.Ss;
  const int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (p >= q.P) return;
  const McPoint pt = mc_point(q.normals + 3 * p, q.view + 3 * p);
  const Dual a = mk(q.rough[p], 1.f);
  float da = 0.f;
  for (int k = lane; k < q.Ss; k += 32) {
    const int j = q.Sd + k;
    const long i = long(p) * S + j;
    const float phi = mc_azimuth(q.tab_s[2 * k], q.rand_s ? q.rand_s[p] : 0.f, q.rand_s != nullptr);
    Dual dd[3];
    mc_specular_dir<Dual>(pt, phi, q.tab_s[2 * k + 1], a, dd);
    const float d[3] = {dd[0].v, dd[1].v, dd[2].v};
    const int slot = q.slot[i];
    float g[3] = {0.f, 0.f, 0.f};
    float ge[72];
    if (slot >= 0) {
      const float* e = q.dEO + size_t(slot) * q.ldeo;
      for (int c = 0; c < 72; ++c) ge[c] = e[c];
      ide_backward(c_ide_mc, d, 0.f, ge, g);
      if (q.sphere_dir) {
        float sp[3], pu[3], gsp[3] = {0.f, 0.f, 0.f};
        mc_sphere_point(q.pts + 3 * p, d, sp, pu);
        for (int c = 0; c < 72; ++c) ge[c] = e[72 + c];
        ide_backward(c_ide_mc, sp, 0.f, ge, gsp);
        mc_sphere_point_bwd(pu, d, gsp, g);
      }
      if (q.human) {
        const HumanGeo h = human_geo_fwd(q.pts + 3 * p, d, q.poses + 12 * p, 0.f);
        if (h.hit > 0.5f) {
          const float* eh = q.dEH + size_t(slot) * q.ldeh;
          float gh[24], dmean[2], dvar[2];
          const float var[2] = {0.f, 0.f};
          for (int c = 0; c < 24; ++c) gh[c] = eh[c];
          ipe_backward(h.mean, var, gh, dmean, dvar);
          human_geo_bwd(q.pts + 3 * p, d, q.poses + 12 * p, 0.f, dmean, 0.f, g);
        }
      }
    } else {
      const float* e = q.dEI + size_t(~slot) * q.ldei + 52;
      for (int c = 0; c < 72; ++c) ge[c] = e[c];
      const float4 nh = reinterpret_cast<const float4*>(q.nrm_hit)[i];
      float n[3], v[3];
      const float nr[3] = {nh.x, nh.y, nh.z}, nv[3] = {-d[0], -d[1], -d[2]};
      normalize3(nr, n);
      normalize3(nv, v);
      const float vn = v[0] * n[0] + v[1] * n[1] + v[2] * n[2];
      const float rf[3] = {vn * n[0] * 2.f - v[0], vn * n[1] * 2.f - v[1], vn * n[2] * 2.f - v[2]};
      float gr[3] = {0.f, 0.f, 0.f};
      ide_backward(c_ide_mc, rf, 0.f, ge, gr);
      // r = 2 (v.n) n - v  ->  dv = 2 n (n.gr) - gr ;  v = u/|u|, u = -d
      const float ngr = n[0] * gr[0] + n[1] * gr[1] + n[2] * gr[2];
      float gv[3];
      for (int c = 0; c < 3; ++c) gv[c] = 2.f * n[c] * ngr - gr[c];
      const float un = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
      const float vg = v[0] * gv[0] + v[1] * gv[1] + v[2] * gv[2];
      for (int c = 0; c < 3; ++c) g[c] -= (gv[c] - v[c] * vg) / un;
    }
    da += g[0] * dd[0].d + g[1] * dd[1].d + g[2] * dd[2].d;
  }
  da = warp_sum(da);
  if (lane == 0) q.dA2[p] = da;
}

static inline int blocks_for_l(long n, int per) { return int((n + per - 1) / per); }

extern "C" {

int nero_mc_sample(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  const long N = long(q->P) * (q->Sd + q->Ss);
  if (N <= 0) return NERO_OK;
  mc_sample_kernel<<<blocks_for_l(N, 128), 128, 0, (cudaStream_t)stream>>>(*q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_mc_classify(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  const long N = long(q->P) * (q->Sd + q->Ss);
  if (N <= 0) return NERO_OK;
  const int nblk = blocks_for_l(N, kClsBlock);
  const cudaStream_t st = (cudaStream_t)stream;
  mc_count_kernel<<<nblk, kClsBlock, 0, st>>>(*q, N);
  NERO_LAUNCH_CHECK();
  mc_scan_kernel<<<1, 1024, 0, st>>>(*q, nblk, N);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_mc_fill(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  const long N = long(q->P) * (q->Sd + q->Ss);
  if (N <= 0) return NERO_OK;
  static const cudaError_t attr = cudaFuncSetAttribute(mc_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMcFillSmem);
  if (attr != cudaSuccess) return NERO_ERR_CUDA;
  mc_fill_kernel<<<blocks_for_l(N, kClsBlock), kClsBlock, kMcFillSmem, (cudaStream_t)stream>>>(*q, N);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_mc_combine_fwd(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  if (q->P <= 0) return NERO_OK;
  mc_combine_fwd_kernel<<<blocks_for_l(long(q->P) * 32, 128), 128, 0, (cudaStream_t)stream>>>(*q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_mc_combine_bwd(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  if (q->P <= 0) return NERO_OK;
  mc_combine_bwd_kernel<<<blocks_for_l(long(q->P) * 32, 128), 128, 0, (cudaStream_t)stream>>>(*q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_mc_dir_bwd(const nero_mc_params* q, void* stream) {
  if (!q) return NERO_ERR_ARG;
  if (q->P <= 0) return NERO_OK;
  mc_dir_bwd_kernel<<<blocks_for_l(long(q->P) * 32, 128), 128, 0, (cudaStream_t)stream>>>(*q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

// PE8 rows of the material network input (MaterialFeatsNetwork, field.py:660-689): X [M,ldx] cols 0..50, the same 51
// columns at CAT[:, 256..306] (skip concat before module1) and the raw xyz at Y[:, 256..258] (predictor input cat(feats, pts)).
__global__ void mat_prep_kernel(const float* __restrict__ pts, int M, float* X, int ldx, float* CAT, int ldc, float* Y, int ldy) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float p[3] = {pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]};
  float pe[51];
  pe_encode<3>(p, 8, pe);
  for (int c = 0; c < 51; ++c) { X[size_t(i) * ldx + c] = pe[c]; CAT[size_t(i) * ldc + 256 + c] = pe[c]; }
  for (int c = 0; c < 3; ++c) Y[size_t(i) * ldy + 256 + c] = p[c];
}
extern "C" int nero_mat_prep(const float* pts, int M, float* X, int ldx, float* CAT, int ldc, float* Y, int ldy, void* stream) {
  if (M <= 0) return NERO_OK;
  mat_prep_kernel<<<(M + 127) / 128, 128, 0, (cudaStream_t)stream>>>(pts, M, X, ldx, CAT, ldc, Y, ldy);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
