// Per-sample kernels of the split-sum shading network (AppShadingNetwork.forward, network/field.py:591-651):
//   shade_prep  fwd/bwd : normalize / reflect / NoV, PE6(r), PE8(x), IDE(r, roughness), IDE(n, 1)
//                         (utils/ref_utils.py:85-115), human-light plane intersection + IPE (field.py:536-547)
//   shade_combine fwd/bwd : occlusion blend of the light predictions, FG-LUT lookup (nvdiffrast.texture,
//                         field.py:610-613), diffuse + specular, sRGB, clamp; produces PRE-activation gradients
//                         of every predictor head for the backward GEMMs.
// Buffer layouts (mirrored in nero_b200/shape_renderer.py):
//   E    [N, 240] : PE6(r) @0 (39) | PE8(x) @40 (51) | IDE(r,rough) @92 (72) | IDE(n,1) @164 (72)
//   E    [N, 384] with sphere_direction (field.py:560-563, 583-586: outer_light reads 144 columns):
//                   PE6(r) @0 | PE8(x) @40 | IDE(r,rough) @92 | IDE(s_r,rough) @164 | IDE(n,1) @236 | IDE(s_n,1) @308,
//                   s_d = the direction of the unit-sphere exit point of the ray (x, d)
//   OUTS [N, 32]  : metallic @0 | roughness @4 | albedo @8 | Ldiffuse @12 | Ldirect @16 | Lindirect @20 | inner_weight @24 | human @28 (4)
//   GEO  [N, 8]   : n(3) NoV r(3) hit
#include "common.cuh"
#include "math_shade.cuh"
#include "tile_io.cuh"

namespace nero {

constexpr int E_PE6R = 0, E_PE8X = 40, E_IDER = 92, E_IDEN = 164;
constexpr int ES_IDESR = 164, ES_IDEN = 236, ES_IDESN = 308;   // sphere_direction layout
constexpr int O_MET = 0, O_ROUGH = 4, O_ALB = 8, O_LD = 12, O_LDIR = 16, O_LI = 20, O_IW = 24, O_HUM = 28, O_LDIM = 32;

__constant__ IdeTable c_ide;

int set_ide_table(const float* mat17x36_host) {
  IdeTable t;
  int i = 0;
  for (int e = 0; e < 5; ++e) {
    const int l = 1 << e;
    for (int m = 0; m <= l; ++m) { t.m[i] = m; t.l[i] = l; ++i; }
  }
  for (int k = 0; k < 17; ++k)
    for (int j = 0; j < 36; ++j) { t.mat[k][j] = double(mat17x36_host[k * 36 + j]); t.matf[k][j] = mat17x36_host[k * 36 + j]; }
  NERO_CUDA_TRY(cudaMemcpyToSymbol(c_ide, &t, sizeof(IdeTable)));
  return NERO_OK;
}

__device__ __forceinline__ int load_count2(const int* p, int cap) {
  int m = p ? *p : cap;
  return m > cap ? cap : m;
}

struct ShadePrepParams {
  const float* G; const float* pts; const int* ray_in; const float* rays_d;
  const float* OUTS; float* E; int lde; float* GEO;
  const float* human_poses; float* EH; int ldeh;   // human light (null when disabled)
  int pos_freq;
  const int* m_ptr; int m_cap;
  int sphere;
};

// One thread computes one sample; the wide rows (E: 222-366 floats, the dE inputs of the backward kernel) move through a
// per-warp shared-memory tile (tile_io.cuh) so that global memory sees whole rows.
constexpr int kPrepTileLd = 73;     // 72 columns + 1
struct PrepTile { float t[4][32][kPrepTileLd]; };
#define tile_store_rows warp_rows_store<kPrepTileLd>

__global__ void __launch_bounds__(128) shade_prep_fwd_kernel(const ShadePrepParams q) {
  __shared__ PrepTile sm;
  const int M = load_count2(q.m_ptr, q.m_cap);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int base = blockIdx.x * blockDim.x + warp * 32;
  if (base >= M) return;                       // whole warp
  const int rows = min(32, M - base);
  const int i = min(base + lane, M - 1);       // lanes past the end recompute the last sample and store nothing
  const bool ok = base + lane < M;
  float (*tile)[kPrepTileLd] = sm.t[warp];
  float* mine = tile[lane];
  const int r = q.ray_in[i];
  const float4 g4 = *reinterpret_cast<const float4*>(q.G + size_t(i) * 4);
  const float4 p4 = *reinterpret_cast<const float4*>(q.pts + size_t(i) * 4);
  const float g[3] = {g4.x, g4.y, g4.z}, x[3] = {p4.x, p4.y, p4.z};
  float d[3] = {q.rays_d[r * 3], q.rays_d[r * 3 + 1], q.rays_d[r * 3 + 2]};
  const float dn = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
  const float view[3] = {-d[0] / dn, -d[1] / dn, -d[2] / dn};
  float n[3], v[3], rf[3], NoV;
  shade_geometry_fwd(g, view, n, v, rf, &NoV);
  const float rough = q.OUTS[size_t(i) * O_LDIM + O_ROUGH];
  float* e = q.E + size_t(base) * q.lde;
  pe_encode<3>(rf, 6, mine);
  tile_store_rows(tile, e + E_PE6R, q.lde, 39, rows, lane);
  pe_encode<3>(x, q.pos_freq, mine);
  tile_store_rows(tile, e + E_PE8X, q.lde, 3 + 6 * q.pos_freq, rows, lane);
  ide_forward(c_ide, rf, rough, mine);
  warp_rows_store4<kPrepTileLd, 18>(tile, e + E_IDER, q.lde, rows, lane);
  ide_forward(c_ide, n, 1.0f, mine);
  warp_rows_store4<kPrepTileLd, 18>(tile, e + (q.sphere ? ES_IDEN : E_IDEN), q.lde, rows, lane);
  if (q.sphere) {
    float sd[3];
    sphere_dir_fwd(x, rf, sd);
    ide_forward(c_ide, sd, rough, mine);
    warp_rows_store4<kPrepTileLd, 18>(tile, e + ES_IDESR, q.lde, rows, lane);
    sphere_dir_fwd(x, n, sd);
    ide_forward(c_ide, sd, 1.0f, mine);
    warp_rows_store4<kPrepTileLd, 18>(tile, e + ES_IDESN, q.lde, rows, lane);
  }
  float hit = 0.f;
  if (q.human_poses) {
    const HumanGeo h = human_geo_fwd(x, rf, q.human_poses + size_t(r) * 12, rough);
    const float var2[2] = {h.var, h.var};
    ipe_forward(h.mean, var2, mine);
    warp_rows_store4<kPrepTileLd, 6>(tile, q.EH + size_t(base) * q.ldeh, q.ldeh, rows, lane);
    hit = h.hit;
  }
  if (ok) {
    float* geo = q.GEO + size_t(i) * 8;
    *reinterpret_cast<float4*>(geo) = make_float4(n[0], n[1], n[2], NoV);
    *reinterpret_cast<float4*>(geo + 4) = make_float4(rf[0], rf[1], rf[2], hit);
  }
}

struct ShadePrepBwdParams {
  const float* G; const float* pts; const int* ray_in; const float* rays_d; const float* OUTS; const float* GEO;
  const float* dE_dir; int ld_dir;   // d IDE(r,rough) from outer_light(direct)   cols [0,72)  [+ d IDE(s_r,rough) cols [72,144)]
  const float* dE_inn; int ld_inn;   // d IDE(r,rough) from inner_light          cols [0,72)
  const float* dE_dif; int ld_dif;   // d IDE(n,1)     from outer_light(diffuse) cols [0,72)  [+ d IDE(s_n,1) cols [72,144)]
  const float* dEH; int ld_eh;       // d IPE (24)     from the human predictor  (null when disabled)
  const float* human_poses;
  const float* dNoV;
  float* DOUTS; float* DG;
  const int* m_ptr; int m_cap;
  int sphere;
};

// (row reads stay per thread -- see pe_grad_kernel; this kernel only writes 5 floats per sample)
__global__ void shade_prep_bwd_kernel(const ShadePrepBwdParams q) {
  const int M = load_count2(q.m_ptr, q.m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int r = q.ray_in[i];
  const float4 g4 = *reinterpret_cast<const float4*>(q.G + size_t(i) * 4);
  const float4 p4 = *reinterpret_cast<const float4*>(q.pts + size_t(i) * 4);
  const float g[3] = {g4.x, g4.y, g4.z}, x[3] = {p4.x, p4.y, p4.z};
  float d[3] = {q.rays_d[r * 3], q.rays_d[r * 3 + 1], q.rays_d[r * 3 + 2]};
  const float dn_ = fmaxf(sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]), 1e-12f);
  const float view[3] = {-d[0] / dn_, -d[1] / dn_, -d[2] / dn_};
  float n[3], v[3], rf[3], NoV;
  shade_geometry_fwd(g, view, n, v, rf, &NoV);
  const float rough = q.OUTS[size_t(i) * O_LDIM + O_ROUGH];
  float dide[72];
  for (int c = 0; c < 72; ++c) dide[c] = q.dE_dir[size_t(i) * q.ld_dir + c] + q.dE_inn[size_t(i) * q.ld_inn + c];
  float dr[3] = {0.f, 0.f, 0.f}, dnrm[3] = {0.f, 0.f, 0.f};
  float drough = ide_backward(c_ide, rf, rough, dide, dr);
  for (int c = 0; c < 72; ++c) dide[c] = q.dE_dif[size_t(i) * q.ld_dif + c];
  ide_backward(c_ide, n, 1.0f, dide, dnrm);
  if (q.sphere) {      // the second halves of the two outer_light inputs: encodings of the sphere exit directions
    float sd[3], dsd[3] = {0.f, 0.f, 0.f};
    sphere_dir_fwd(x, rf, sd);
    for (int c = 0; c < 72; ++c) dide[c] = q.dE_dir[size_t(i) * q.ld_dir + 72 + c];
    drough += ide_backward(c_ide, sd, rough, dide, dsd);
    sphere_dir_bwd(x, rf, dsd, dr);
    sphere_dir_fwd(x, n, sd);
    dsd[0] = dsd[1] = dsd[2] = 0.f;
    for (int c = 0; c < 72; ++c) dide[c] = q.dE_dif[size_t(i) * q.ld_dif + 72 + c];
    ide_backward(c_ide, sd, 1.0f, dide, dsd);
    sphere_dir_bwd(x, n, dsd, dnrm);
  }
  if (q.human_poses) {
    const float* pose = q.human_poses + size_t(r) * 12;
    const HumanGeo h = human_geo_fwd(x, rf, pose, rough);
    if (h.hit > 0.f) {
      float deh[24], dmean[2], dvar[2];
      for (int c = 0; c < 24; ++c) deh[c] = q.dEH[size_t(i) * q.ld_eh + c];
      const float var2[2] = {h.var, h.var};
      ipe_backward(h.mean, var2, deh, dmean, dvar);
      drough += human_geo_bwd(x, rf, pose, rough, dmean, dvar[0] + dvar[1], dr);
    }
  }
  q.DOUTS[size_t(i) * O_LDIM + O_ROUGH] += drough * rough * (1.0f - rough);
  float dg[3] = {0.f, 0.f, 0.f};
  shade_geometry_bwd(g, n, v, NoV, dnrm, dr, q.dNoV[i], dg);
  *reinterpret_cast<float4*>(q.DG + size_t(i) * 4) = make_float4(dg[0], dg[1], dg[2], 0.f);
}

struct ShadeCombineParams {
  const float* OUTS; const float* GEO; const float* lut; float exp_max; int human;
  float* color; float* occ_prob; float* refl;           // fwd outputs: [N,4], [N], [N,4]
  const float* dcolor; const float* docc; float* DOUTS; float* dNoV;   // bwd
  const int* m_ptr; int m_cap;
};

__device__ __forceinline__ ShadeIn load_shade_in(const float* o, const float* geo, int human) {
  ShadeIn s;
  s.metallic = o[O_MET]; s.roughness = o[O_ROUGH];
  for (int c = 0; c < 3; ++c) { s.albedo[c] = o[O_ALB + c]; s.Ld[c] = o[O_LD + c]; s.Ldir[c] = o[O_LDIR + c]; s.Li[c] = o[O_LI + c]; }
  s.iw = o[O_IW];
  const float hit = human ? geo[7] : 0.f;
  for (int c = 0; c < 3; ++c) s.Lh[c] = human ? o[O_HUM + c] * hit : 0.f;
  s.wh = human ? o[O_HUM + 3] * hit : 0.f;
  s.NoV = geo[3];
  return s;
}

__global__ void shade_combine_fwd_kernel(const ShadeCombineParams q) {
  const int M = load_count2(q.m_ptr, q.m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float* geo = q.GEO + size_t(i) * 8;
  const ShadeIn s = load_shade_in(q.OUTS + size_t(i) * O_LDIM, geo, q.human);
  float c[3];
  shade_combine_fwd(s, q.lut, c);
  *reinterpret_cast<float4*>(q.color + size_t(i) * 4) = make_float4(c[0], c[1], c[2], 0.f);
  q.occ_prob[i] = s.iw * 0.5f + 0.5f;
  *reinterpret_cast<float4*>(q.refl + size_t(i) * 4) = make_float4(geo[4], geo[5], geo[6], 0.f);
}

__global__ void shade_combine_bwd_kernel(const ShadeCombineParams q) {
  const int M = load_count2(q.m_ptr, q.m_cap);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float* geo = q.GEO + size_t(i) * 8;
  const float* o = q.OUTS + size_t(i) * O_LDIM;
  const ShadeIn s = load_shade_in(o, geo, q.human);
  ShadeGrad d;
  const float4 dc4 = *reinterpret_cast<const float4*>(q.dcolor + size_t(i) * 4);
  const float dc[3] = {dc4.x, dc4.y, dc4.z};
  shade_combine_bwd(s, q.lut, dc, d);
  float* dout = q.DOUTS + size_t(i) * O_LDIM;
  const float emax = expf(q.exp_max);
  dout[O_MET] = d.metallic * s.metallic * (1.0f - s.metallic);
  dout[O_ROUGH] = d.roughness * s.roughness * (1.0f - s.roughness);
  for (int c = 0; c < 3; ++c) {
    dout[O_ALB + c] = d.albedo[c] * s.albedo[c] * (1.0f - s.albedo[c]);
    dout[O_LD + c] = s.Ld[c] < emax ? d.Ld[c] * s.Ld[c] : 0.f;
    dout[O_LDIR + c] = s.Ldir[c] < emax ? d.Ldir[c] * s.Ldir[c] : 0.f;
    dout[O_LI + c] = s.Li[c] < emax ? d.Li[c] * s.Li[c] : 0.f;
  }
  dout[O_IW] = d.iw + (q.docc ? 0.5f * q.docc[i] : 0.f);
  if (q.human) {
    const float hit = geo[7];
    for (int c = 0; c < 3; ++c) { const float y = o[O_HUM + c]; dout[O_HUM + c] = y < 1.0f ? d.Lh[c] * hit * y : 0.f; }
    const float y = o[O_HUM + 3];
    dout[O_HUM + 3] = y < 1.0f ? d.wh * hit * y : 0.f;
  }
  q.dNoV[i] = d.NoV;
}

constexpr int kEncBlock = 128;
// out[i, 0:72] = IDE(dirs[i, 0:3], kappa_inv[i * kstride])   (kappa == nullptr: kappa_scalar for every row)
__global__ void __launch_bounds__(kEncBlock) ide_kernel(const float* __restrict__ dirs, int ldd, const float* __restrict__ kappa, int kstride,
                                                       float kappa_scalar, int M, float* __restrict__ out, int ldo) {
  __shared__ float s_rows[kEncBlock * 73];
  const int i0 = blockIdx.x * kEncBlock;
  const int i = i0 + threadIdx.x;
  if (i < M) {
    const float d[3] = {dirs[size_t(i) * ldd], dirs[size_t(i) * ldd + 1], dirs[size_t(i) * ldd + 2]};
    ide_forward(c_ide, d, kappa ? kappa[size_t(i) * kstride] : kappa_scalar, s_rows + threadIdx.x * 73);
  }
  __syncthreads();
  const int rows = min(kEncBlock, M - i0);
  if (ldo == 72) {
    float* dst = out + size_t(i0) * 72;
    for (int e = threadIdx.x; e < rows * 72; e += kEncBlock) dst[e] = s_rows[(e / 72) * 73 + e % 72];
  } else {
    for (int r = threadIdx.x >> 5; r < rows; r += kEncBlock / 32)
      for (int c = threadIdx.x & 31; c < 72; c += 32) out[size_t(i0 + r) * ldo + c] = s_rows[r * 73 + c];
  }
}

static inline int blocks_for(long n, int per) { return int((n + per - 1) / per); }

extern "C" {

int nero_ide(const float* dirs, int ldd, const float* kappa_inv, int kstride, float kappa_scalar, int M, float* out, int ldo, void* stream) {
  if (!dirs || !out || ldd < 3 || ldo < 72) return NERO_ERR_ARG;
  if (M <= 0) return NERO_OK;
  ide_kernel<<<(M + kEncBlock - 1) / kEncBlock, kEncBlock, 0, (cudaStream_t)stream>>>(dirs, ldd, kappa_inv, kstride, kappa_scalar, M, out, ldo);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_shade_prep_fwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, float* E, int lde,
                        float* GEO, const float* human_poses, float* EH, int ldeh, int pos_freq, const int* m_ptr, int m_cap, int sphere, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const ShadePrepParams q{G, pts, ray_in, rays_d, OUTS, E, lde, GEO, human_poses, EH, ldeh, pos_freq, m_ptr, m_cap, sphere};
  shade_prep_fwd_kernel<<<blocks_for(m_cap, 128), 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_shade_prep_bwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, const float* GEO,
                        const float* dE_dir, int ld_dir, const float* dE_inn, int ld_inn, const float* dE_dif, int ld_dif,
                        const float* dEH, int ld_eh, const float* human_poses, const float* dNoV, float* DOUTS, float* DG,
                        const int* m_ptr, int m_cap, int sphere, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const ShadePrepBwdParams q{G, pts, ray_in, rays_d, OUTS, GEO, dE_dir, ld_dir, dE_inn, ld_inn, dE_dif, ld_dif, dEH, ld_eh, human_poses, dNoV,
                             DOUTS, DG, m_ptr, m_cap, sphere};
  shade_prep_bwd_kernel<<<blocks_for(m_cap, 128), 128, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_shade_combine_fwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, float* color,
                           float* occ_prob, float* refl, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const ShadeCombineParams q{OUTS, GEO, lut, exp_max, human, color, occ_prob, refl, nullptr, nullptr, nullptr, nullptr, m_ptr, m_cap};
  shade_combine_fwd_kernel<<<blocks_for(m_cap, 256), 256, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}
int nero_shade_combine_bwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, const float* dcolor,
                           const float* docc, float* DOUTS, float* dNoV, const int* m_ptr, int m_cap, void* stream) {
  if (m_cap <= 0) return NERO_OK;
  const ShadeCombineParams q{OUTS, GEO, lut, exp_max, human, nullptr, nullptr, nullptr, dcolor, docc, DOUTS, dNoV, m_ptr, m_cap};
  shade_combine_bwd_kernel<<<blocks_for(m_cap, 256), 256, 0, (cudaStream_t)stream>>>(q);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
