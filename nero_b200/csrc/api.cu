// extern "C" entry points of libnero_b200 (declared in include/nero_b200.h).
#include "common.cuh"
#include "../../include/nero_b200.h"

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
struct WgradParams {
  const float* dY; int ldy; const float* X; int ldx;
  const float* dY2; int ldy2; const float* X2; int ldx2;
  int n0; int n_valid; int k0; int k_valid;
  float* partial; int ld_partial; int rows_partial;
  float* bias_partial;
  const int* m_ptr; int m_cap;
};
int linear_dispatch(const LinearParams& p, cudaStream_t stream);
int wgrad_dispatch(WgradParams p, int n_rows_pad, int k_pad, int P, cudaStream_t stream);
int prep_weight(const float* v, const float* g, int K, int row0, int nrows, const int* kmap, float in_scale,
                uint8_t* img_f, int rows_pad_f, uint8_t* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff, int ld_weff,
                cudaStream_t stream);
int wgrad_finish(const float* partial, int P, int rows_partial, int ld_partial, const float* bias_partial, int K,
                 int row0, int nrows, const int* kmap, float in_scale, const float* v, const float* g, float* grad_w,
                 float* grad_g, float* grad_b, const float* extra_row, float extra_scale, cudaStream_t stream);
int colsum(const float* X, int ldx, int ncol, const float* w, int ldw, const int* m_ptr, int m_cap, float* out, cudaStream_t stream);
int wgrad_finish_batch(const void* jobs_dev, int n_jobs, int max_rows, int max_k, cudaStream_t stream);
int prep_weight_batch(const void* jobs_dev, int n_jobs, int max_rows, cudaStream_t stream);
int adam_flat(float* p, const float* g, float* m, float* v, long n, float lr_over_bc1, float b1, float b2, float eps, float inv_sqrt_bc2,
              float wd, cudaStream_t st);
}  // namespace nero


namespace nero {
struct IdeTable;
int set_ide_table(const float* mat17x36_host);
int ray_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, int* cnt_in, int* cnt_out,
                int* off_in, int* off_out, int* n_in, int* n_out, cudaStream_t st);
struct FillParams {
  const float* rays_o; const float* rays_d; const float* z_vals; int R; int S;
  const int* off_in; const int* off_out;
  int* slot; float* pts; int* ray_in;
  float* X0; int ld_x0; float* Y8; int ld_y8; float* H4; int ld_h4;
  float* XN; int ld_xn; float* H5; int ld_h5; float* FV; int ld_fv;
  float* dist_out; int* ray_out;
};
int ray_fill(const FillParams& q, cudaStream_t st);
int dact_times_row(const float* H, int ldh, const float* row, float* V, int ldv, int ncol, const int* m_ptr, int m_cap, cudaStream_t st);
int pe_grad(const float* X0, int ldx, const float* U0, int ldu, const float* US, int lds, float* G, const int* m_ptr, int m_cap, cudaStream_t st);
int pe_tangent_launch(const float* X0, int ldx, const float* DG, float* UB0, int ld0, float* UB4, int ld4, const int* m_ptr, int m_cap, cudaStream_t st);
int sdf_alpha_forward(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                      const float* variance, const float* car, float* alpha, float* gerr, const int* m_ptr, int m_cap, cudaStream_t st);
int sdf_alpha_backward(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, const float* dalpha, const float* dgerr, float* dY8, int lddy, float* DG,
                       float* d_inv_s, const int* m_ptr, int m_cap, cudaStream_t st);
int nerf_post_forward(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, float* alpha, float* color, const int* m_ptr, int m_cap, cudaStream_t st);
int nerf_post_backward(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, const float* dalpha, const float* dcolor,
                       float* ddens, int lddd, float* drgb, int lddr, const int* m_ptr, int m_cap, cudaStream_t st);
int composite_forward(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                      float* rgb, float* weights, cudaStream_t st);
int composite_backward(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       const float* drgb, float* da_in, float* dc_in, float* da_out, float* dc_out, cudaStream_t st);
struct ShadePrepParams {
  const float* G; const float* pts; const int* ray_in; const float* rays_d;
  const float* OUTS; float* E; int lde; float* GEO;
  const float* human_poses; float* EH; int ldeh;
  int pos_freq;
  const int* m_ptr; int m_cap;
  int sphere;
};
struct ShadePrepBwdParams {
  const float* G; const float* pts; const int* ray_in; const float* rays_d; const float* OUTS; const float* GEO;
  const float* dE_dir; int ld_dir; const float* dE_inn; int ld_inn; const float* dE_dif; int ld_dif;
  const float* dEH; int ld_eh; const float* human_poses; const float* dNoV;
  float* DOUTS; float* DG;
  const int* m_ptr; int m_cap;
  int sphere;
};
struct ShadeCombineParams {
  const float* OUTS; const float* GEO; const float* lut; float exp_max; int human;
  float* color; float* occ_prob; float* refl;
  const float* dcolor; const float* docc; float* DOUTS; float* dNoV;
  const int* m_ptr; int m_cap;
};
int shade_prep_forward(const ShadePrepParams& q, cudaStream_t st);
int shade_prep_backward(const ShadePrepBwdParams& q, cudaStream_t st);
int shade_combine_forward(const ShadeCombineParams& q, cudaStream_t st);
int shade_combine_backward(const ShadeCombineParams& q, cudaStream_t st);
struct SampleInitParams {
  const float* rays_o; const float* rays_d; const float* near; const float* far; int R;
  int n; int nb;
  const float* lin_inner; const float* bg_base; const float* bg_lower; const float* bg_upper;
  const float* rand_inner; const float* rand_bg;
  float* z; int ldz; float* z_bg; int ldzb;
  float* X0; int ldx; float* HC; int ldh;
};
struct UpsampleParams {
  const float* rays_o; const float* rays_d; int R;
  const float* z; int ldz; const float* sdf; int lds; int n;
  int n_new;
  const float* variance; float inv_s_cap; int clip;
  int surface_variant;
  float* new_z; int ldn;
  float* X0; int ldx; float* HC; int ldh;
  float* wsum;
  const float* origins;
};
int sample_init(const SampleInitParams& q, cudaStream_t st);
int upsample(const UpsampleParams& q, cudaStream_t st);
int merge_samples(const float* z, int ldz, const float* sdf, int lds, int n, const float* nz, int ldn, const float* nsdf, int ldns,
                  int m, float* oz, int ldoz, float* osdf, int ldos, int R, cudaStream_t st);
int occ_init(const float* pts, const float* refl, const int* sel, const int* p_ptr, int p_cap, int sn0, const float* lin,
             float* o_out, float* d_out, float* z, int ldz, float* X0, int ldx, float* HC, int ldh, cudaStream_t st);
int occ_select(const float* pts, const float* Y8, int ldy, int sdf_col, const float* G, const int* ray_in, const float* rays_d,
               float sdf_thresh, const int* m_ptr, int m_cap, int* sel, int* count, cudaStream_t st);
int row_axpy(const float* a, int lda, const float* X, int ldx, float* Y, int ldy, int ncol, const int* m_ptr, int m_cap, cudaStream_t st);
int reg_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, int* cnt, int* cnt_dummy,
                int* off, int* off_dummy, int* n, int* n_dummy, cudaStream_t st);
int reg_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, const int* off, float* pts,
             float* X0, int ldx, float* H4, int ldh, cudaStream_t st);
int points_fill(const float* pts3, int N, float* pts, int* ray_in, float* X0, int ldx, float* Y8, int ldy, float* H4, int ldh, cudaStream_t st);
struct ChainParams;
int set_ide_table_mc(const float* mat17x36_host);
int bvh_build_host(const float* verts, int V, const int* tris, int T, void* nodes_out, float* tri_out, int* tri_id_out, int* n_nodes);
struct BvhNode;
struct TraceParams {
  const BvhNode* nodes; const float4* tris; int n_rays;
  const float* org; int ldo; const float* dir; int ldd;
  float4* pos_depth; float4* nrm_hit;
  float miss_depth; int flip;
};
int bvh_trace(const TraceParams& q, cudaStream_t st);
int mc_sample(const ::nero_mc_params& q, cudaStream_t st);
int mc_classify(const ::nero_mc_params& q, cudaStream_t st);
int mc_fill(const ::nero_mc_params& q, cudaStream_t st);
int mc_combine_fwd(const ::nero_mc_params& q, cudaStream_t st);
int mc_combine_bwd(const ::nero_mc_params& q, cudaStream_t st);
int mc_dir_bwd(const ::nero_mc_params& q, cudaStream_t st);
int mat_prep(const float* pts, int M, float* X, int ldx, float* CAT, int ldc, float* Y, int ldy, cudaStream_t st);
int chain_dispatch(const ChainParams& p, cudaStream_t stream);
int pe_standalone(const float* x, int d, int ldx, int M, int L, float scale, float* out, int ldo, cudaStream_t st);
int ide_standalone(const float* dirs, int ldd, const float* kappa, int kstride, float kappa_scalar, int M, float* out, int ldo, cudaStream_t st);
int occ_loss(const float* occ_prob, const float* gt, const int* sel, const int* p_ptr, int p_cap, float* loss_sum, float* docc_sign,
             cudaStream_t st);
int mcubes_count(const float* u, int nx, int ny, int nz, float iso, int* blk_cnt, long long* blk_off, long long* totals, cudaStream_t st);
int mcubes_emit(const float* u, int nx, int ny, int nz, float iso, const long long* blk_off, long long V, long long T, int* emap,
                float* verts, int* tris, cudaStream_t st);
int relight_render(const ::nero_relight_params& q, cudaStream_t st);
int depth_render(const ::nero_depth_params& q, cudaStream_t st);
int depth_points_count(const float* depth, int n_views, int height, int width, float lo, float hi, int* blk_cnt, long long* blk_off,
                       long long* total, cudaStream_t st);
int depth_points_emit(const float* depth, int n_views, int height, int width, float lo, float hi, const double* cams,
                      const long long* blk_off, long long n, float* pts, cudaStream_t st);
int voxel_keys(const double* pts, long long n, const double* bounds, double voxel, long long* keys, cudaStream_t st);
int voxel_mean(const double* pts, const long long* order, const long long* ends, long long m, double* out, cudaStream_t st);
int nearest_dist(const float* q, long long n, const float* t, long long m, float* dist, cudaStream_t st);
}  // namespace nero

using namespace nero;

extern "C" {

int nero_version(void) { return 100; }

int nero_prep_weight(const float* v, const float* g, int K, int row0, int nrows, const int* kmap, float in_scale,
                     void* img_f, int rows_pad_f, void* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff, int ld_weff,
                     void* stream) {
  return prep_weight(v, g, K, row0, nrows, kmap, in_scale, (uint8_t*)img_f, rows_pad_f, (uint8_t*)img_t, rows_pad_t, t_c0, t_ncols,
                     w_eff, ld_weff, (cudaStream_t)stream);
}

int nero_linear(const float* A, int lda, int k_valid, const void* wimg, int n_pad, int k_chunks, const float* bias, int n_bias,
                float* out, int ldo, int ncol_out, float oscale, int mode, int act, float act_param,
                const float* H, int ldh, float hscale, int dact, const float* V, int ldv, float* out2, int ldo2,
                const float* addend, int ldadd, int ncol_main, float* tail, int ldt,
                const int* m_ptr, int m_cap, void* stream) {
  LinearParams p{A, lda, k_valid, (const uint8_t*)wimg, n_pad, k_chunks, bias, n_bias, out, ldo, ncol_out, oscale, mode, act, act_param,
                 H, ldh, hscale, dact, V, ldv, out2, ldo2, addend, ldadd, ncol_main, tail, ldt, m_ptr, m_cap};
  if (!A || !wimg || !out || ncol_out > n_pad) return NERO_ERR_ARG;
  return linear_dispatch(p, (cudaStream_t)stream);
}

int nero_wgrad(const float* dY, int ldy, int n_valid, const float* X, int ldx, int k_valid,
               const float* dY2, int ldy2, const float* X2, int ldx2,
               float* partial, int ld_partial, int rows_partial, float* bias_partial,
               int n_rows_pad, int k_pad, int P, const int* m_ptr, int m_cap, void* stream) {
  WgradParams p{dY, ldy, X, ldx, dY2, ldy2, X2, ldx2, 0, n_valid, 0, k_valid, partial, ld_partial, rows_partial, bias_partial,
                m_ptr, m_cap};
  if (!dY || !X || !partial || (dY2 && !X2)) return NERO_ERR_ARG;
  return wgrad_dispatch(p, n_rows_pad, k_pad, P, (cudaStream_t)stream);
}

int nero_wgrad_finish(const float* partial, int P, int rows_partial, int ld_partial, const float* bias_partial, int K,
                      int row0, int nrows, const int* kmap, float in_scale, const float* v, const float* g,
                      float* grad_w, float* grad_g, float* grad_b, const float* extra_row, float extra_scale, void* stream) {
  return wgrad_finish(partial, P, rows_partial, ld_partial, bias_partial, K, row0, nrows, kmap, in_scale, v, g, grad_w, grad_g,
                      grad_b, extra_row, extra_scale, (cudaStream_t)stream);
}

int nero_colsum(const float* X, int ldx, int ncol, const float* w, int ldw, const int* m_ptr, int m_cap, float* out,
                void* stream) {
  return colsum(X, ldx, ncol, w, ldw, m_ptr, m_cap, out, (cudaStream_t)stream);
}

int nero_set_ide_table(const float* mat17x36_host) {
  const int rc = set_ide_table(mat17x36_host);
  return rc != NERO_OK ? rc : set_ide_table_mc(mat17x36_host);
}
int nero_bvh_build_host(const float* verts, int V, const int* tris, int T, void* nodes_out, float* tri_out, int* tri_id_out, int* n_nodes) {
  if (!verts || !tris || !nodes_out || !tri_out || !tri_id_out || !n_nodes) return NERO_ERR_ARG;
  return bvh_build_host(verts, V, tris, T, nodes_out, tri_out, tri_id_out, n_nodes);
}
int nero_bvh_trace(const void* nodes, const float* tris, int n_rays, const float* org, int ldo, const float* dir, int ldd,
                   float* pos_depth, float* nrm_hit, float miss_depth, int flip, void* stream) {
  if (!nodes || !tris || (n_rays > 0 && (!org || !dir || !pos_depth || !nrm_hit))) return NERO_ERR_ARG;
  TraceParams q{reinterpret_cast<const BvhNode*>(nodes), reinterpret_cast<const float4*>(tris), n_rays, org, ldo, dir, ldd,
                reinterpret_cast<float4*>(pos_depth), reinterpret_cast<float4*>(nrm_hit), miss_depth, flip};
  return bvh_trace(q, (cudaStream_t)stream);
}
int nero_mc_sample(const nero_mc_params* q, void* stream) { return q ? mc_sample(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mc_classify(const nero_mc_params* q, void* stream) { return q ? mc_classify(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mc_fill(const nero_mc_params* q, void* stream) { return q ? mc_fill(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mc_combine_fwd(const nero_mc_params* q, void* stream) { return q ? mc_combine_fwd(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mc_combine_bwd(const nero_mc_params* q, void* stream) { return q ? mc_combine_bwd(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mc_dir_bwd(const nero_mc_params* q, void* stream) { return q ? mc_dir_bwd(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_mcubes_count(const float* u, int nx, int ny, int nz, float iso, int* blk_cnt, long long* blk_off, long long* totals,
                      void* stream) {
  return mcubes_count(u, nx, ny, nz, iso, blk_cnt, blk_off, totals, (cudaStream_t)stream);
}
int nero_mcubes_emit(const float* u, int nx, int ny, int nz, float iso, const long long* blk_off, long long V, long long T, int* emap,
                     float* verts, int* tris, void* stream) {
  return mcubes_emit(u, nx, ny, nz, iso, blk_off, V, T, emap, verts, tris, (cudaStream_t)stream);
}
int nero_relight_render(const nero_relight_params* q, void* stream) {
  return q ? relight_render(*q, (cudaStream_t)stream) : NERO_ERR_ARG;
}
int nero_depth_render(const nero_depth_params* q, void* stream) { return q ? depth_render(*q, (cudaStream_t)stream) : NERO_ERR_ARG; }
int nero_depth_points_count(const float* depth, int n_views, int height, int width, float lo, float hi, int* blk_cnt,
                            long long* blk_off, long long* total, void* stream) {
  return depth_points_count(depth, n_views, height, width, lo, hi, blk_cnt, blk_off, total, (cudaStream_t)stream);
}
int nero_depth_points_emit(const float* depth, int n_views, int height, int width, float lo, float hi, const double* cams,
                           const long long* blk_off, long long n, float* pts, void* stream) {
  return depth_points_emit(depth, n_views, height, width, lo, hi, cams, blk_off, n, pts, (cudaStream_t)stream);
}
int nero_voxel_keys(const double* pts, long long n, const double* bounds_host, double voxel, long long* keys, void* stream) {
  return voxel_keys(pts, n, bounds_host, voxel, keys, (cudaStream_t)stream);
}
int nero_voxel_mean(const double* pts, const long long* order, const long long* ends, long long m, double* out, void* stream) {
  return voxel_mean(pts, order, ends, m, out, (cudaStream_t)stream);
}
int nero_nearest_dist(const float* q, long long n, const float* t, long long m, float* dist, void* stream) {
  return nearest_dist(q, n, t, m, dist, (cudaStream_t)stream);
}
int nero_abi_sizeof(int which) {
  switch (which) {
    case 0: return int(sizeof(nero_chain_layer));
    case 1: return int(sizeof(nero_chain_params));
    case 2: return int(sizeof(nero_mc_params));
    case 3: return 104;   /* finish job record (k_weights.cu FinishJob) */
    case 4: return 88;    /* prep job record (k_weights.cu PrepJob) */
    case 5: return int(sizeof(nero_relight_params));
    case 6: return int(sizeof(nero_depth_params));
    default: return -1;
  }
}
int nero_prep_weight_batch(const void* jobs_dev, int n_jobs, int max_rows, void* stream) {
  return prep_weight_batch(jobs_dev, n_jobs, max_rows, (cudaStream_t)stream);
}
int nero_wgrad_finish_batch(const void* jobs_dev, int n_jobs, int max_rows, int max_k, void* stream) {
  return wgrad_finish_batch(jobs_dev, n_jobs, max_rows, max_k, (cudaStream_t)stream);
}
int nero_adam_flat(float* p, const float* g, float* m, float* v, long long n, float lr_over_bc1, float b1, float b2, float eps,
                   float inv_sqrt_bc2, float weight_decay, void* stream) {
  if (!p || !g || !m || !v) return NERO_ERR_ARG;
  return adam_flat(p, g, m, v, long(n), lr_over_bc1, b1, b2, eps, inv_sqrt_bc2, weight_decay, (cudaStream_t)stream);
}
int nero_mat_prep(const float* pts, int M, float* X, int ldx, float* CAT, int ldc, float* Y, int ldy, void* stream) {
  return mat_prep(pts, M, X, ldx, CAT, ldc, Y, ldy, (cudaStream_t)stream);
}

int nero_pe(const float* x, int d, int ldx, int M, int L, float scale, float* out, int ldo, void* stream) {
  return pe_standalone(x, d, ldx, M, L, scale, out, ldo, (cudaStream_t)stream);
}
int nero_ide(const float* dirs, int ldd, const float* kappa_inv, int kstride, float kappa_scalar, int M, float* out, int ldo, void* stream) {
  return ide_standalone(dirs, ldd, kappa_inv, kstride, kappa_scalar, M, out, ldo, (cudaStream_t)stream);
}

int nero_chain(const void* chain_params_host, void* stream) {
  if (!chain_params_host) return NERO_ERR_ARG;
  return chain_dispatch(*reinterpret_cast<const ChainParams*>(chain_params_host), (cudaStream_t)stream);
}
int nero_reg_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, int* cnt, int* cnt_dummy,
                     int* off, int* off_dummy, int* n, int* n_dummy, void* stream) {
  return reg_prepare(rays_o, rays_d, z_vals, R, S, radius, cnt, cnt_dummy, off, off_dummy, n, n_dummy, (cudaStream_t)stream);
}
int nero_reg_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, const int* off, float* pts,
                  float* X0, int ldx, float* H4, int ldh, void* stream) {
  return reg_fill(rays_o, rays_d, z_vals, R, S, radius, off, pts, X0, ldx, H4, ldh, (cudaStream_t)stream);
}
int nero_points_fill(const float* pts3, int N, float* pts, int* ray_in, float* X0, int ldx, float* Y8, int ldy, float* H4, int ldh, void* stream) {
  return points_fill(pts3, N, pts, ray_in, X0, ldx, Y8, ldy, H4, ldh, (cudaStream_t)stream);
}
int nero_row_axpy(const float* a, int lda, const float* X, int ldx, float* Y, int ldy, int ncol, const int* m_ptr, int m_cap, void* stream) {
  return row_axpy(a, lda, X, ldx, Y, ldy, ncol, m_ptr, m_cap, (cudaStream_t)stream);
}

int nero_ray_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, int* cnt_in, int* cnt_out,
                     int* off_in, int* off_out, int* n_in, int* n_out, void* stream) {
  return ray_prepare(rays_o, rays_d, z_vals, R, S, cnt_in, cnt_out, off_in, off_out, n_in, n_out, (cudaStream_t)stream);
}
int nero_ray_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, const int* off_in, const int* off_out,
                  int* slot, float* pts, int* ray_in, float* X0, int ld_x0, float* Y8, int ld_y8, float* H4, int ld_h4,
                  float* XN, int ld_xn, float* H5, int ld_h5, float* FV, int ld_fv, float* dist_out, int* ray_out, void* stream) {
  FillParams q{rays_o, rays_d, z_vals, R, S, off_in, off_out, slot, pts, ray_in, X0, ld_x0, Y8, ld_y8, H4, ld_h4, XN, ld_xn, H5, ld_h5,
               FV, ld_fv, dist_out, ray_out};
  return ray_fill(q, (cudaStream_t)stream);
}
int nero_dact_times_row(const float* H, int ldh, const float* row, float* V, int ldv, int ncol, const int* m_ptr, int m_cap, void* stream) {
  return dact_times_row(H, ldh, row, V, ldv, ncol, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_pe_grad(const float* X0, int ldx, const float* U0, int ldu, const float* US, int lds, float* G, const int* m_ptr, int m_cap, void* stream) {
  return pe_grad(X0, ldx, U0, ldu, US, lds, G, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_pe_tangent(const float* X0, int ldx, const float* DG, float* UB0, int ld0, float* UB4, int ld4, const int* m_ptr, int m_cap, void* stream) {
  return pe_tangent_launch(X0, ldx, DG, UB0, ld0, UB4, ld4, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_sdf_alpha_fwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, float* alpha, float* gerr, const int* m_ptr, int m_cap, void* stream) {
  return sdf_alpha_forward(Y8, ldy, sdf_col, G, pts, ray_in, rays_d, variance, car, alpha, gerr, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_sdf_alpha_bwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, const float* dalpha, const float* dgerr, float* dY8, int lddy, float* DG,
                       float* d_inv_s, const int* m_ptr, int m_cap, void* stream) {
  return sdf_alpha_backward(Y8, ldy, sdf_col, G, pts, ray_in, rays_d, variance, car, dalpha, dgerr, dY8, lddy, DG, d_inv_s, m_ptr, m_cap,
                            (cudaStream_t)stream);
}
int nero_nerf_post_fwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, float* alpha, float* color,
                       const int* m_ptr, int m_cap, void* stream) {
  return nerf_post_forward(dens, ldd, rgb, ldr, dist, alpha, color, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_nerf_post_bwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, const float* dalpha, const float* dcolor,
                       float* ddens, int lddd, float* drgb, int lddr, const int* m_ptr, int m_cap, void* stream) {
  return nerf_post_backward(dens, ldd, rgb, ldr, dist, dalpha, dcolor, ddens, lddd, drgb, lddr, m_ptr, m_cap, (cudaStream_t)stream);
}
int nero_composite_fwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       float* rgb, float* weights, void* stream) {
  return composite_forward(slot, R, S, a_in, c_in, a_out, c_out, rgb, weights, (cudaStream_t)stream);
}
int nero_composite_bwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       const float* drgb, float* da_in, float* dc_in, float* da_out, float* dc_out, void* stream) {
  return composite_backward(slot, R, S, a_in, c_in, a_out, c_out, drgb, da_in, dc_in, da_out, dc_out, (cudaStream_t)stream);
}
int nero_shade_prep_fwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, float* E, int lde,
                        float* GEO, const float* human_poses, float* EH, int ldeh, int pos_freq, const int* m_ptr, int m_cap, int sphere, void* stream) {
  ShadePrepParams q{G, pts, ray_in, rays_d, OUTS, E, lde, GEO, human_poses, EH, ldeh, pos_freq, m_ptr, m_cap, sphere};
  return shade_prep_forward(q, (cudaStream_t)stream);
}
int nero_shade_prep_bwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, const float* GEO,
                        const float* dE_dir, int ld_dir, const float* dE_inn, int ld_inn, const float* dE_dif, int ld_dif,
                        const float* dEH, int ld_eh, const float* human_poses, const float* dNoV, float* DOUTS, float* DG,
                        const int* m_ptr, int m_cap, int sphere, void* stream) {
  ShadePrepBwdParams q{G, pts, ray_in, rays_d, OUTS, GEO, dE_dir, ld_dir, dE_inn, ld_inn, dE_dif, ld_dif, dEH, ld_eh, human_poses, dNoV,
                       DOUTS, DG, m_ptr, m_cap, sphere};
  return shade_prep_backward(q, (cudaStream_t)stream);
}
int nero_shade_combine_fwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, float* color,
                           float* occ_prob, float* refl, const int* m_ptr, int m_cap, void* stream) {
  ShadeCombineParams q{OUTS, GEO, lut, exp_max, human, color, occ_prob, refl, nullptr, nullptr, nullptr, nullptr, m_ptr, m_cap};
  return shade_combine_forward(q, (cudaStream_t)stream);
}
int nero_shade_combine_bwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, const float* dcolor,
                           const float* docc, float* DOUTS, float* dNoV, const int* m_ptr, int m_cap, void* stream) {
  ShadeCombineParams q{OUTS, GEO, lut, exp_max, human, nullptr, nullptr, nullptr, dcolor, docc, DOUTS, dNoV, m_ptr, m_cap};
  return shade_combine_backward(q, (cudaStream_t)stream);
}
int nero_sample_init(const float* rays_o, const float* rays_d, const float* near, const float* far, int R, int n, int nb,
                     const float* lin_inner, const float* bg_base, const float* bg_lower, const float* bg_upper,
                     const float* rand_inner, const float* rand_bg, float* z, int ldz, float* z_bg, int ldzb,
                     float* X0, int ldx, float* HC, int ldh, void* stream) {
  SampleInitParams q{rays_o, rays_d, near, far, R, n, nb, lin_inner, bg_base, bg_lower, bg_upper, rand_inner, rand_bg, z, ldz, z_bg, ldzb,
                     X0, ldx, HC, ldh};
  return sample_init(q, (cudaStream_t)stream);
}
int nero_upsample(const float* rays_o, const float* rays_d, int R, const float* z, int ldz, const float* sdf, int lds, int n, int n_new,
                  const float* variance, float inv_s_cap, int clip, int surface_variant, float* new_z, int ldn,
                  float* X0, int ldx, float* HC, int ldh, float* wsum, void* stream) {
  UpsampleParams q{rays_o, rays_d, R, z, ldz, sdf, lds, n, n_new, variance, inv_s_cap, clip, surface_variant, new_z, ldn, X0, ldx, HC, ldh,
                   wsum, nullptr};
  return upsample(q, (cudaStream_t)stream);
}
int nero_merge_samples(const float* z, int ldz, const float* sdf, int lds, int n, const float* nz, int ldn, const float* nsdf, int ldns,
                       int m, float* oz, int ldoz, float* osdf, int ldos, int R, void* stream) {
  return merge_samples(z, ldz, sdf, lds, n, nz, ldn, nsdf, ldns, m, oz, ldoz, osdf, ldos, R, (cudaStream_t)stream);
}
int nero_occ_init(const float* pts, const float* refl, const int* sel, const int* p_ptr, int p_cap, int sn0, const float* lin,
                  float* o_out, float* d_out, float* z, int ldz, float* X0, int ldx, float* HC, int ldh, void* stream) {
  return occ_init(pts, refl, sel, p_ptr, p_cap, sn0, lin, o_out, d_out, z, ldz, X0, ldx, HC, ldh, (cudaStream_t)stream);
}
int nero_occ_select(const float* pts, const float* Y8, int ldy, int sdf_col, const float* G, const int* ray_in, const float* rays_d,
                    float sdf_thresh, const int* m_ptr, int m_cap, int* sel, int* count, void* stream) {
  return occ_select(pts, Y8, ldy, sdf_col, G, ray_in, rays_d, sdf_thresh, m_ptr, m_cap, sel, count, (cudaStream_t)stream);
}
int nero_occ_loss(const float* occ_prob, const float* gt, const int* sel, const int* p_ptr, int p_cap, float* loss_sum, float* docc_sign,
                  void* stream) {
  return occ_loss(occ_prob, gt, sel, p_ptr, p_cap, loss_sum, docc_sign, (cudaStream_t)stream);
}

}  // extern "C"
