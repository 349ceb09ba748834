/* libnero_b200 -- C ABI of the H100-native (sm_90a) NeRO stage-I volume-rendering hot path.
 *
 * There is no FFI in the reference (it is pure PyTorch); the boundary this library sits behind is the Python
 * nn.Module contract of network/renderer.py (NeROShapeRenderer.render / render_core) -- see INTEGRATION.md.
 * Each entry point below replaces a group of PyTorch op sites of the reference; the file:line it replaces is
 * cited per function.  Conventions: all pointers are DEVICE pointers unless marked host; fp32 row-major
 * matrices with an explicit leading dimension (in floats); `stream` is a cudaStream_t passed as void*;
 * no allocation and no host synchronisation inside; data-dependent row counts are read from device memory
 * (`m_ptr`, clamped to the host-known capacity `m_cap`); the return value is 0 on success, non-zero on a bad
 * argument (1) or a CUDA launch error (2).
 */
#ifndef NERO_B200_H_
#define NERO_B200_H_
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* activation codes */
#define NERO_ACT_NONE 0
#define NERO_ACT_SOFTPLUS100 1 /* nn.Softplus(beta=100), network/field.py:124 */
#define NERO_ACT_RELU 2
#define NERO_ACT_SIGMOID 3
#define NERO_ACT_EXPCLAMP 4    /* exp(min(x, p)), network/field.py:302-308 */
/* epilogue modes of nero_linear */
#define NERO_EPI_BIAS_ACT 0
#define NERO_EPI_MUL_DACT 1
#define NERO_EPI_TANGENT 2

int nero_version(void);

/* ---- weights ------------------------------------------------------------------------------------------
 * Fold weight_norm (network/field.py:118-119, 324-331: W = g * v/||v||) and build the tensor-core operand images
 * (split-bf16, K-major SWIZZLE_128B, one 64-wide K chunk = [hi plane | lo plane]).  g == NULL: plain weight
 * (NeRFNetwork, field.py:239-256).  kmap (device, may be NULL) maps reference input column -> layout column.
 * img_t (for input-gradient GEMMs) only covers layout columns [t_c0, t_c0+t_ncols). */
int nero_prep_weight(const float* v, const float* g, int K, int row0, int nrows, const int* kmap, float in_scale,
                     void* img_f, int rows_pad_f, void* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff, int ld_weff,
                     void* stream);

/* ---- fused linear layer on wgmma tensor cores ------------------------------------------------------------
 * out = epilogue(A[M,K] * W^T).  Replaces nn.Linear + activation of SDFNetwork.forward (field.py:130-147),
 * NeRFNetwork.forward (field.py:258-283), make_predictor (field.py:310-346) and the autograd input-gradient /
 * double-backward GEMMs of SDFNetwork.gradient (field.py:155-167).
 *   mode BIAS_ACT : out = oscale * act(acc + bias)
 *   mode MUL_DACT : out[:, :ncol_main] = oscale * act'(H*hscale) * acc (+ addend);  tail[:, :] = oscale * acc[:, ncol_main:]
 *   mode TANGENT  : as MUL_DACT, plus out2 = 100 * (1 - act'(H*hscale)) * V * acc   (softplus'' term)
 * A is 16-byte aligned; H, V and addend (when given) are 8-byte aligned with even leading dimensions (else NERO_ERR_ARG). */
int nero_linear(const float* A, int lda, int k_valid, const void* wimg, int n_pad, int k_chunks, const float* bias, int n_bias,
                float* out, int ldo, int ncol_out, float oscale, int mode, int act, float act_param,
                const float* H, int ldh, float hscale, int dact, const float* V, int ldv, float* out2, int ldo2,
                const float* addend, int ldadd, int ncol_main, float* tail, int ldt,
                const int* m_ptr, int m_cap, void* stream);

/* ---- fused MLP chain on wgmma (A operand kept in shared memory across layers) -----------------------------------
 * Runs up to 10 consecutive layers of SDFNetwork / make_predictor / NeRFNetwork (network/field.py:130-147, 310-346,
 * 258-283) or of their gradient sweeps on each 128-row tile without writing the inter-layer activations' A operand
 * to HBM.  `chain_params_host` points to a HOST struct nero_chain_params (layout below, natural alignment).  A0 is 16-byte
 * aligned; every layer's H, V and addend (when given) are 8-byte aligned with even leading dimensions (else NERO_ERR_ARG). */
typedef struct nero_chain_layer {
  const void* wimg; const float* bias;
  float* save; const float* H; const float* addend; const float* V; float* out2; float* tail;
  int n_pad, k_chunks, n_bias, ncol_out, ncol_main, kind, act;   /* kind: 0 bias+softplus100, 1 bias+relu, 2 bias+act(generic), */
  int ld_save, ldh, ldadd, ldv, ldo2, ldt;                        /*       3 dsoftplus*acc, 4 drelu*acc, 5 acc, 6 tangent        */
  float oscale, hscale, act_param;
  int write_a, a_blocks;      /* write_a: the output becomes the next A operand; a_blocks: 16-col blocks of it to define */
  const float* csrc; int ld_csrc;   /* skip-concat source: columns >= ncol_out of the next A operand come from csrc[row, col] */
  int pad_;
} nero_chain_layer;
typedef struct nero_chain_params {
  const float* A0; int lda0; int k_valid0;
  int n_layers; const int* m_ptr; int m_cap;
  nero_chain_layer L[10];
  /* phase_clk: NULL, except with the diagnostic build compiled with NERO_CHAIN_PHASES (tools/chain_phases.py), where it
   * points to zeroed device memory of 132 * (2 * 10 * 5 + 2) counters: the SM cycles each warpgroup spent in each phase
   * of each layer, then per CTA its cycles and globaltimer nanoseconds (k_gemm_chain.cu).  The product build ignores it. */
  unsigned long long* phase_clk;
} nero_chain_params;
int nero_chain(const void* chain_params_host, void* stream);
/* Y[i,:] += a[i*lda] * X[i,:] */
int nero_row_axpy(const float* a, int lda, const float* X, int ldx, float* Y, int ldy, int ncol, const int* m_ptr, int m_cap, void* stream);

/* ---- weight gradients -------------------------------------------------------------------------------------
 * partial = dY^T X (+ dY2^T X2) split over sample rows: P CTAs per 128-row output tile each contract a slice of the sample
 * rows and store their tile into their own slice p of the [P x rows_partial x ld_partial] fp32 array `partial` (and the
 * column sums of dY into `bias_partial` [P x rows_partial]).  Every slice's rows [0, 128 * ceil(n_rows_pad / 128)) (clipped
 * to rows_partial) x columns [0, k_pad) are stored, zeros included, so the caller need not initialise either array.  No
 * atomics: the result is the same every run.
 * Replaces the autograd weight-gradient GEMMs; nero_wgrad_finish is then called with the same P. */
int nero_wgrad(const float* dY, int ldy, int n_valid, const float* X, int ldx, int k_valid,
               const float* dY2, int ldy2, const float* X2, int ldx2,
               float* partial, int ld_partial, int rows_partial, float* bias_partial,
               int n_rows_pad, int k_pad, int P, const int* m_ptr, int m_cap, void* stream);
/* reduce partials, undo kmap, weight-norm chain rule, accumulate into grads (g == NULL: plain weight) */
int nero_wgrad_finish(const float* partial, int P, int rows_partial, int ld_partial, const float* bias_partial, int K,
                      int row0, int nrows, const int* kmap, float in_scale, const float* v, const float* g,
                      float* grad_w, float* grad_g, float* grad_b, const float* extra_row, float extra_scale, void* stream);
/* out[j] += sum_m w[m*ldw] * X[m, j]  (w NULL = 1) */
int nero_colsum(const float* X, int ldx, int ncol, const float* w, int ldw, const int* m_ptr, int m_cap, float* out,
                void* stream);

/* ---- stand-alone encodings (fused into their consumers on the training path) --------------------------------
 * nero_pe : out[i, 0:d(1+2L)] = scale * [x, sin(2^0 x), cos(2^0 x), ..., sin(2^(L-1) x), cos(2^(L-1) x)], d in {3,4}
 *           (Embedder / get_embedder, network/field.py:14-58).
 * nero_ide: out[i, 0:72] = integrated directional encoding [Re(36) | Im(36)] of dirs[i, 0:3] with
 *           kappa_inv[i*kstride] (kappa_inv == NULL: kappa_scalar)   (generate_ide_fn(5), utils/ref_utils.py:53-117;
 *           needs nero_set_ide_table first). */
int nero_pe(const float* x, int d, int ldx, int M, int L, float scale, float* out, int ldo, void* stream);
int nero_ide(const float* dirs, int ldd, const float* kappa_inv, int kstride, float kappa_scalar, int M, float* out, int ldo, void* stream);

/* ---- encodings --------------------------------------------------------------------------------------------
 * Upload the IDE coefficient table mat[17][36] (HOST pointer; fp32-rounded like utils/ref_utils.py:77-82). */
int nero_set_ide_table(const float* mat17x36_host);

/* ---- render_core sample bookkeeping (network/renderer.py:554-572) -----------------------------------------
 * ray_prepare: per-ray inner/outer counts + exclusive scan -> off_in/off_out, totals n_in/n_out (device ints).
 * ray_fill: ordered compaction; writes slot[R,S] (inner i >= 0, outer -1-io), pts[i]=(x,y,z,dist), ray ids,
 * PE6(p) rows (X0, and /sqrt2 into H4[:,217:256] for the skip concat of field.py:139-140), p into Y8[:,256:259],
 * PE10([p/|p|,1/|p|]) rows (XN and H5[:, :84]), PE4(-dir) into FV[:,256:283], dist_out. */
int nero_ray_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, int* cnt_in, int* cnt_out,
                     int* off_in, int* off_out, int* n_in, int* n_out, void* stream);
int nero_ray_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, const int* off_in, const int* off_out,
                  int* slot, float* pts, int* ray_in, float* X0, int ld_x0, float* Y8, int ld_y8, float* H4, int ld_h4,
                  float* XN, int ld_xn, float* H5, int ld_h5, float* FV, int ld_fv, float* dist_out, int* ray_out, void* stream);

/* init-sdf regulariser points (network/renderer.py:591-594): ordered compaction of samples with |p| < radius + PE rows */
int nero_reg_prepare(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, int* cnt, int* cnt_dummy,
                     int* off, int* off_dummy, int* n, int* n_dummy, void* stream);
int nero_reg_fill(const float* rays_o, const float* rays_d, const float* z_vals, int R, int S, float radius, const int* off, float* pts,
                  float* X0, int ldx, float* H4, int ldh, void* stream);

/* arbitrary query points (validation render network/renderer.py:465-482; grid query network/field.py:1090-1117 via
 * sdf_network.sdf, extract_mesh.py:27): PE rows into X0 and the layer-4 skip tail; optionally PTS, identity ray ids and
 * xyz into Y8 (each may be NULL) */
int nero_points_fill(const float* pts3, int N, float* pts, int* ray_in, float* X0, int ldx, float* Y8, int ldy, float* H4, int ldh, void* stream);

/* ---- analytic SDF gradient helpers (SDFNetwork.gradient, network/field.py:155-167) ------------------------- */
int nero_dact_times_row(const float* H, int ldh, const float* row, float* V, int ldv, int ncol, const int* m_ptr, int m_cap, void* stream);
int nero_pe_grad(const float* X0, int ldx, const float* U0, int ldu, const float* US, int lds, float* G, const int* m_ptr, int m_cap, void* stream);
int nero_pe_tangent(const float* X0, int ldx, const float* DG, float* UB0, int ld0, float* UB4, int ld4, const int* m_ptr, int m_cap, void* stream);

/* ---- NeuS SDF -> alpha + eikonal term (compute_sdf_alpha, network/renderer.py:484-512, :574) ---------------- */
int nero_sdf_alpha_fwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, float* alpha, float* gerr, const int* m_ptr, int m_cap, void* stream);
int nero_sdf_alpha_bwd(const float* Y8, int ldy, int sdf_col, const float* G, const float* pts, const int* ray_in, const float* rays_d,
                       const float* variance, const float* car, const float* dalpha, const float* dgerr, float* dY8, int lddy, float* DG,
                       float* d_inv_s, const int* m_ptr, int m_cap, void* stream);

/* ---- outer NeRF activations (compute_density_alpha, network/renderer.py:346-347, 514-520) ------------------- */
int nero_nerf_post_fwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, float* alpha, float* color,
                       const int* m_ptr, int m_cap, void* stream);
int nero_nerf_post_bwd(const float* dens, int ldd, const float* rgb, int ldr, const float* dist, const float* dalpha, const float* dcolor,
                       float* ddens, int lddd, float* drgb, int lddr, const int* m_ptr, int m_cap, void* stream);

/* ---- alpha compositing, warp per ray (network/renderer.py:578-579) ------------------------------------------ */
int nero_composite_fwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       float* rgb, float* weights, void* stream);
int nero_composite_bwd(const int* slot, int R, int S, const float* a_in, const float* c_in, const float* a_out, const float* c_out,
                       const float* drgb, float* da_in, float* dc_in, float* da_out, float* dc_out, void* stream);

/* ---- split-sum shading (AppShadingNetwork.forward, network/field.py:591-651; IDE utils/ref_utils.py:85-115) - */
int nero_shade_prep_fwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, float* E, int lde,
                        float* GEO, const float* human_poses, float* EH, int ldeh, int pos_freq, const int* m_ptr, int m_cap, int sphere, void* stream);
int nero_shade_prep_bwd(const float* G, const float* pts, const int* ray_in, const float* rays_d, const float* OUTS, const float* GEO,
                        const float* dE_dir, int ld_dir, const float* dE_inn, int ld_inn, const float* dE_dif, int ld_dif,
                        const float* dEH, int ld_eh, const float* human_poses, const float* dNoV, float* DOUTS, float* DG,
                        const int* m_ptr, int m_cap, int sphere, void* stream);
int nero_shade_combine_fwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, float* color,
                           float* occ_prob, float* refl, const int* m_ptr, int m_cap, void* stream);
int nero_shade_combine_bwd(const float* OUTS, const float* GEO, const float* lut, float exp_max, int human, const float* dcolor,
                           const float* docc, float* DOUTS, float* dNoV, const int* m_ptr, int m_cap, void* stream);

/* ---- NeuS hierarchical sampling (sample_ray / upsample / cat_z_vals, network/renderer.py:355-443;
 *      sample_pdf network/field.py:399-429) and the occlusion march (get_weights/get_intersection, field.py:432-484) */
int nero_sample_init(const float* rays_o, const float* rays_d, const float* near, const float* far, int R, int n, int nb,
                     const float* lin_inner, const float* bg_base, const float* bg_lower, const float* bg_upper,
                     const float* rand_inner, const float* rand_bg, float* z, int ldz, float* z_bg, int ldzb,
                     float* X0, int ldx, float* HC, int ldh, void* stream);
int nero_upsample(const float* rays_o, const float* rays_d, int R, const float* z, int ldz, const float* sdf, int lds, int n, int n_new,
                  const float* variance, float inv_s_cap, int clip, int surface_variant, float* new_z, int ldn,
                  float* X0, int ldx, float* HC, int ldh, float* wsum, void* stream);
int nero_merge_samples(const float* z, int ldz, const float* sdf, int lds, int n, const float* nz, int ldn, const float* nsdf, int ldns,
                       int m, float* oz, int ldoz, float* osdf, int ldos, int R, void* stream);
int nero_occ_init(const float* pts, const float* refl, const int* sel, const int* p_ptr, int p_cap, int sn0, const float* lin,
                  float* o_out, float* d_out, float* z, int ldz, float* X0, int ldx, float* HC, int ldh, void* stream);
int nero_occ_select(const float* pts, const float* Y8, int ldy, int sdf_col, const float* G, const int* ray_in, const float* rays_d,
                    float sdf_thresh, const int* m_ptr, int m_cap, int* sel, int* count, void* stream);
int nero_occ_loss(const float* occ_prob, const float* gt, const int* sel, const int* p_ptr, int p_cap, float* loss_sum, float* docc_sign,
                  void* stream);

/* ------------------------------------------------------------------------------------------------------------------
 * Stage II (material estimation).  Replaces MCShadingNetwork.shade_mixed / get_lights (network/field.py:858-1003) around
 * the light MLPs and the third-party ray tracer called at network/renderer.py:676,720.
 * ------------------------------------------------------------------------------------------------------------------ */
/* Host-side BVH build (init time).  verts [V,3] fp32 and tris [T,3] int32 in HOST memory; outputs in caller-allocated
 * HOST memory: nodes_out 2*T records of 32 bytes, tri_out T*12 floats (v0,e1,e2 as float4), tri_id_out T ints. */
int nero_bvh_build_host(const float* verts, int V, const int* tris, int T, void* nodes_out, float* tri_out, int* tri_id_out, int* n_nodes);
/* Closest hit of n_rays rays (device pointers).  pos_depth [n,4] = (hit position, depth; depth = miss_depth on a miss),
 * nrm_hit [n,4] = (unit face normal, hit flag); flip != 0 negates the normal (renderer.py:722-723). */
int nero_bvh_trace(const void* nodes, const float* tris, int n_rays, const float* org, int ldo, const float* dir, int ldd,
                   float* pos_depth, float* nrm_hit, float miss_depth, int flip, void* stream);

typedef struct nero_mc_params {
  const float* pts; const float* normals; const float* view; const float* rough;   /* per point [P,3] x3, [P]            */
  const float* poses;                                                               /* [P,12] capturer poses or NULL     */
  const float* rand_d; const float* rand_s;                                         /* [P] azimuth draws or NULL         */
  const float* tab_d; const float* tab_s;                                           /* [Sd,2], [Ss,2] (az, el) in [0,1]  */
  int P, Sd, Ss;
  int ggx_smith, sphere_dir, human;
  float* org; float* dir;                                                           /* per ray [N,4], N = P*(Sd+Ss)      */
  const float* pos_depth; const float* nrm_hit;                                     /* nero_bvh_trace outputs            */
  int* slot;                                                                        /* >= 0 outer row, < 0 ~inner row    */
  int* blk_cnt; int* blk_off; int* counts;                                          /* [ceil(N/256)] x2, [2]=(hit,miss)  */
  float* EO; int ldeo; float* EH; int ldeh; float* hhit; float* EI; int ldei;       /* MLP input rows                    */
  const float* OUT_O; const float* OUT_H; const float* OUT_I;                       /* MLP outputs [.,4]                 */
  float exp_max_o, exp_max_i;
  float* LD; float* LS; float* LSF;                                                 /* estimator means [P,3]             */
  const float* dLD; const float* dLS; const float* dLSF;
  float* DPRE_O; float* DPRE_H; float* DPRE_I;                                      /* pre-activation output grads [.,4] */
  float* dA;                                                                        /* [P] d/d roughness (weights part)  */
  const float* dEO; const float* dEH; const float* dEI;                             /* MLP input grads                   */
  float* dA2;                                                                       /* [P] d/d roughness via directions  */
} nero_mc_params;
/* sample_diffuse_directions / sample_specular_directions (field.py:768-812): dir, org = pts + 1e-5*dir */
int nero_mc_sample(const nero_mc_params* q, void* stream);
/* hit/miss counts per 256-ray block + exclusive scan + totals (deterministic compaction, field.py:866-879 masks) */
int nero_mc_classify(const nero_mc_params* q, void* stream);
/* row assignment + encodings: outer IDE(dir,0) [+IDE(sphere point)] (+ human IPE), inner PE8(hit) | IDE(reflection) */
int nero_mc_fill(const nero_mc_params* q, void* stream);
/* LD / LS / LSF means over the samples (field.py:941-984) */
int nero_mc_combine_fwd(const nero_mc_params* q, void* stream);
int nero_mc_combine_bwd(const nero_mc_params* q, void* stream);
/* gradient reaching the roughness through the specular directions (IDE / IPE / reflection backward) */
int nero_mc_dir_bwd(const nero_mc_params* q, void* stream);
/* MaterialFeatsNetwork inputs (field.py:660-689): PE8 rows, skip-concat tail, xyz for the predictor input */
int nero_mat_prep(const float* pts, int M, float* X, int ldx, float* CAT, int ldc, float* Y, int ldy, void* stream);

/* ---- marching cubes (mcubes.marching_cubes in extract_geometry, network/field.py:1110-1117; extract_mesh.py) --------------
 * u: [nx,ny,nz] fp32 C-contiguous, u[i,j,k] at index point (i,j,k); a corner is below iff u <= iso.  One vertex per grid edge
 * (p, p+e_a) whose ends lie on different sides, at p + t e_a with t = (iso-u(p)) / (u(p+e_a)-u(p)), ordered by (linear index of
 * p, a); triangles ordered by the linear index of their cube, then table order (nero_b200/csrc/mc_tables.cuh), wound so that
 * cross(v1-v0, v2-v0) points to the below side.  Placement is count -> exclusive scan -> emit: the same input gives
 * bit-identical output.  Workspaces, with nblk = ceil(nx*ny*nz / 1024): blk_cnt int[2*nblk], blk_off int64[2*nblk],
 * totals int64[2], emap int[3*nx*ny*nz] (written at sign-change edges only; needs no initialisation).
 * nero_mcubes_count: block counts, their scan and totals = (V, T) in device memory.
 * nero_mcubes_emit: V, T are those totals read back by the caller; writes verts [V,3] fp32 (index space), tris [T,3] int32.
 * Both return 1 if a dimension is < 2; emit also if V or T does not fit in int32. */
int nero_mcubes_count(const float* u, int nx, int ny, int nz, float iso, int* blk_cnt, long long* blk_off, long long* totals,
                      void* stream);
int nero_mcubes_emit(const float* u, int nx, int ny, int nz, float iso, const long long* blk_off, long long V, long long T, int* emap,
                     float* verts, int* tris, void* stream);

/* ---- relighting (the Blender Cycles render of relight.py / blender_backend/relight_backend.py) ---------------------------
 * Path-traces one image of a triangle mesh with per-vertex NeRO materials under an equirectangular environment map
 * (k_relight.cu; the scene is stated in nero_b200/relight.py).  One thread per pixel adds the radiance of samples
 * [spp0, spp0 + spp) in order into accum[pixel] = (r, g, b, number of samples that hit the mesh); every random number is a
 * hash of (seed, pixel, sample, bounce, dimension), so any split of the samples over calls gives the same bits.
 * rays (may be NULL) receives the number of rays traced (camera + shadow + continuation).  All pointers are device pointers. */
typedef struct nero_relight_params {
  const void* nodes; const float* tris;           /* nero_bvh_build_host outputs (nodes, tri)                              */
  const int* tri_ids; const int* faces;           /* [T] BVH order -> input triangle, [T,3] vertex indices                 */
  const float* vmat;                              /* [V,8] albedo rgb, metallic, roughness (linear values), 3 unused       */
  const float* env;                               /* [H,W,4] radiance rgb + unused, rows from the bottom (v = 0) up        */
  const float* env_p;                             /* [H,W] probability of each texel for the light sampler                 */
  const float* cdf_rows; const float* cdf_cols;   /* [H+1] marginal CDF over rows, [H,W+1] conditional CDF per row         */
  float* accum;                                   /* [height*width,4] running sums                                         */
  unsigned long long* rays;
  float pose[12];                                 /* world -> camera [R | t], row-major, OpenCV axes (x right, y down)     */
  float K[4];                                     /* fx, fy, cx, cy in pixels                                              */
  int env_w, env_h, width, height;
  int spp0, spp, max_bounces, ggx_smith;
  unsigned int seed; int pad_;
} nero_relight_params;
int nero_relight_render(const nero_relight_params* q, void* stream);

/* ---- shape evaluation (eval_synthetic_shape.py / eval_real_shape.py; the protocol is stated in nero_b200/evaluate.py) ------
 * nero_depth_render: depth map of a triangle mesh as the reference's nvdiffrast call produces it (w = 1): per pixel (x, y) the
 * closest hit of the ray through (x + 1/2, y + 1/2), depth = sum b_i z_i^2 / sum b_i z_i from its 3-D barycentrics b and the
 * camera depths z of the input vertices; 0 on a miss or outside [near_z, far_z].  K must have zero skew and last row (0, 0, 1). */
typedef struct nero_depth_params {
  const void* nodes; const float* tris;           /* nero_bvh_build_host outputs (nodes, tri)                              */
  const int* tri_ids; const int* faces;           /* [T] BVH order -> input triangle, [T,3] vertex indices                 */
  const float* verts;                             /* [V,3]                                                                 */
  float* depth;                                   /* [height,width] output                                                 */
  float pose[12];                                 /* world -> camera [R | t], row-major, OpenCV axes (x right, y down)     */
  float K[9];                                     /* 3x3 row-major intrinsics in pixels                                    */
  int width, height;
  float near_z, far_z;
} nero_depth_params;
int nero_depth_render(const nero_depth_params* q, void* stream);
/* Ordered compaction of the pixels with lo < depth < hi of n_views stacked [height,width] depth maps, in (view, row, column)
 * order, each unprojected at its integer pixel coordinates, X_cam = d ((x - cx)/fx, (y - cy)/fy, 1), and moved to world
 * space, X = R_c2w X_cam + c, in fp64; written as fp32 pts [n,3].  cams: [n_views,16] fp64 = R_c2w (row-major 3x3), camera
 * centre c, fx, fy, cx, cy.  Count -> exclusive scan -> emit; workspaces with nblk = ceil(n_views*height*width / 1024):
 * blk_cnt int[nblk], blk_off int64[nblk], total int64[1].  emit takes n = *total read back by the caller. */
int nero_depth_points_count(const float* depth, int n_views, int height, int width, float lo, float hi, int* blk_cnt,
                            long long* blk_off, long long* total, void* stream);
int nero_depth_points_emit(const float* depth, int n_views, int height, int width, float lo, float hi, const double* cams,
                           const long long* blk_off, long long n, float* pts, void* stream);
/* Open3D VoxelDownSample in fp64.  nero_voxel_keys: key = i << 42 | j << 21 | k with (i, j, k) = floor((p - min) / voxel);
 * bounds_host (HOST) = (min_x, min_y, min_z, max_x, max_y, max_z) with min = the cloud's minimum - voxel/2; returns 1 if an
 * index along any axis can reach 2^21.  nero_voxel_mean: given order = a stable key sort of the points and ends = inclusive
 * cumulative counts of the m distinct keys, out[v] = mean of the points of voxel v, summed in input order. */
int nero_voxel_keys(const double* pts, long long n, const double* bounds_host, double voxel, long long* keys, void* stream);
int nero_voxel_mean(const double* pts, const long long* order, const long long* ends, long long m, double* out, void* stream);
/* dist[i] = min_j |q_i - t_j| over t [m,3] (m >= 1), q [n,3], fp32: ((dx*dx + dy*dy) + dz*dz) rounded to nearest without
 * contraction, minimum, correctly rounded square root.  The result does not depend on the launch shape. */
int nero_nearest_dist(const float* q, long long n, const float* t, long long m, float* dist, void* stream);

/* sizeof() of the structures that cross this ABI, for bindings to verify their layouts against the library:
 * 0 nero_chain_layer, 1 nero_chain_params, 2 nero_mc_params, 3 nero_finish_job, 4 nero_prep_job, 5 nero_relight_params,
 * 6 nero_depth_params. */
int nero_abi_sizeof(int which);

/* nero_prep_weight for many layers in ONE launch.  jobs_dev: device array of n_jobs records (same meaning as the
 * nero_prep_weight arguments). */
typedef struct nero_prep_job {
  const float* v; const float* g; const int* kmap; void* img_f; void* img_t; float* w_eff;
  int K, row0, nrows, rows_pad_f, rows_pad_t, t_c0, t_ncols, ld_weff;
  float in_scale; int pad_;
} nero_prep_job;
int nero_prep_weight_batch(const void* jobs_dev, int n_jobs, int max_rows, void* stream);

/* nero_wgrad_finish for many layers in ONE launch.  jobs_dev: device array of n_jobs records (same meaning as the
 * nero_wgrad_finish arguments).  Jobs of one launch must not share destination rows. */
typedef struct nero_finish_job {
  const float* partial; const float* bias_partial; const int* kmap; const float* v; const float* g;
  float* grad_w; float* grad_g; float* grad_b; const float* extra_row;
  int P, rows_partial, ld_partial, K, row0, nrows;
  float in_scale, extra_scale;
} nero_finish_job;
int nero_wgrad_finish_batch(const void* jobs_dev, int n_jobs, int max_rows, int max_k, void* stream);

/* Adam step over one flat fp32 parameter buffer (torch.optim.Adam semantics; replaces the multi-tensor optimizer launch of
 * train/trainer.py:73-76,160-166).  lr_over_bc1 = lr / (1 - b1^t), inv_sqrt_bc2 = 1 / sqrt(1 - b2^t); buffers 16-byte aligned. */
int nero_adam_flat(float* p, const float* g, float* m, float* v, long long n, float lr_over_bc1, float b1, float b2, float eps,
                   float inv_sqrt_bc2, float weight_decay, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_B200_H_ */
