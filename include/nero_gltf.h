/* libnero_b200 -- C ABI of the glTF 2.0 export of a textured mesh: welded vertices, tangent frames, the tangent-space normal
 * map and the metallic-roughness texture (nero_b200/gltf.py sequences it and writes the container; oracle/nero_oracle_gltf.py
 * restates it in numpy).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.  No
 * kernel uses atomics, and every sum runs in a fixed order, so two runs give identical bytes.
 *
 * Inputs are the textured OBJ as relight.load_textured_obj reads it: verts [V,3] fp32, tris [T,3] int32 (wound with
 * cross(e1, e2) pointing into the solid, include/nero_normalmap.h), vt [N,2] fp32 as the file stores it (v points up in the
 * image), ft [T,3] int32 into vt.  (vt_ptr [V+1], vt_tri [3T]) is each vertex's triangles in ascending order, the CSR of
 * nero_b200.simplify._vertex_triangles: a triangle that names a vertex twice is listed twice.
 *
 * Corner walk of a position vertex p.  The CSR entries of p in ascending order; an entry equal to the one before it is
 * skipped (the triangle was walked already); within a triangle t, the slots s = 0, 1, 2 with tris[3t+s] = p in ascending
 * order.  Every corner of p is visited exactly once.
 *
 * Weld.  A glTF vertex is one distinct (position index, uv index) pair.  One thread per position vertex p: the distinct uv
 * indices ft[3t+s] of its corners, in the order of the corner walk, get local ids 0, 1, ... by first occurrence.  The
 * per-vertex counts go through the ordered scan of compact.cuh (blocks of 256 vertices), so the welded vertices are ordered by
 * position vertex, then by local id.  Outputs: wv [W] (position index), wt [W] (uv index), wf [T,3] (the welded vertex of each
 * corner, in the OBJ's corner order).  Vertices with no triangle get no welded vertex; W = the number of distinct pairs.
 *
 * Tangent frames.  One thread per welded vertex i = (p, k); n = normals[p] (nero_normalmap_vertex_normals).  fp32, every
 * operation rounded on its own (_rn); dot(a, b) = (a0 b0 + a1 b1) + a2 b2; normalize(s) = s / sqrt(dot(s, s)).  Over the
 * corners (t, s) of p's corner walk with ft[3t+s] = k, in that order:
 *   P0, P1, P2 = the positions of slots s, s+1, s+2 (mod 3); e1 = P1 - P0, e2 = P2 - P0;
 *   uv0, uv1, uv2 = vt of the same slots (the file's convention); d1 = uv1 - uv0, d2 = uv2 - uv0;
 *   det = d1u d2v - d2u d1v;  t_f = (d2v e1 - d1v e2) / det;  b_f = (d1u e2 - d2u e1) / det (per component, products first);
 *   t_p = normalize(t_f - n dot(n, t_f));
 *   the corner is skipped when det = 0, e1 or e2 is zero, or t_f - n dot(n, t_f) is zero;
 *   a = acosf(clamp(dot(e1 / |e1|, e2 / |e2|), -1, 1)), the corner angle (MikkTSpace's weight);
 *   S += a t_p;  h += a if dot(cross(n, t_f), b_f) >= 0 else h -= a.
 * Then T = normalize(S - n dot(n, S)) and w = -1 if h < 0 else +1.  A vertex with no usable corner, or whose S projects to
 * zero: T = normalize(cross(a, n)) with a the unit axis of the smallest |n component| (ties to the lowest index), w = +1.  A
 * zero normal: n = (0, 0, 1), T = (1, 0, 0), w = +1.  Outputs: wnormal [W,3] (n as written), wtangent [W,4] = (T, w).
 *
 * Tangent-space conversion.  One thread per covered texel of the raster of the atlas (u, 1 - v) at the normal map's size
 * (texel [n], owner: nero_tex_raster / nero_tex_compact_* of include/nero_texmap.h), with the texel's barycentrics b exactly as
 * the texture export computes them (texel_bary.cuh).  For its triangle t, with n_i, (t_i, w_i) the welded frames of wf[3t+i]:
 *   N = normalize(Σ b_i n_i), T = normalize(Σ b_i t_i), B = normalize(Σ b_i w_i cross(n_i, t_i)), each sum ((i0 + i1) + i2),
 *   the frame the glTF 2.0 sample viewer interpolates per fragment;
 *   m = normalize(2 k / 255 - 1) per channel of the object-space map's bytes at the texel (fp32: (2k) / 255, then - 1);
 *   det = dot(T, cross(B, N));  x = (dot(m, cross(B, N)), dot(m, cross(N, T)), dot(m, cross(T, B))) / det, normalised;
 *   bytes = floor((x 0.5 + 0.5) 255 + 0.5) clamped to [0, 255] (include/nero_normalmap.h's encoding).
 * m zero, det zero or any result not finite writes the bytes of (0, 0, 1), i.e. (128, 128, 255).  The three bytes go to
 * channels 0-2 of img [width*height, 5] at the texel; channels 3-4 and every uncovered texel are 0, the layout
 * nero_tex_inpaint fills the seam band of.
 *
 * Metallic-roughness texture.  One thread per texel: out [n,3] = (255, lut_r[roughness[i]], lut_m[metallic[i]]), glTF's
 * (occlusion, roughness, metallic) channel order with no occlusion.  The tables are built on the host from the relighter's
 * decoding (nero_b200/gltf.py): lut_m[k] = round(255 srgb_to_linear(k / 255)), lut_r[k] = round(255 sqrt(srgb_to_linear(k /
 * 255))), since the texture export stores alpha and glTF's roughness is sqrt(alpha).
 */
#ifndef NERO_GLTF_H_
#define NERO_GLTF_H_

#include "nero_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Weld, step 1: per-block counts of welded vertices (blk_cnt [nblk], nblk = ceil(V / 256)), their exclusive offsets blk_off
 * [nblk] and *total = W, on the device.  Returns 1 for V, T < 0, NULL buffers (V > 0) or V >= 2^31 - 255. */
int nero_gltf_weld_count(const int* tris, const int* ft, int T, int V, const int* vt_ptr, const int* vt_tri, int* blk_cnt,
                         long long* blk_off, long long* total, void* stream);

/* Weld, step 2: wv [W], wt [W], wf [T,3] with W = *total of step 1.  Returns 1 for NULL buffers or W outside [0, 3T]. */
int nero_gltf_weld_emit(const int* tris, const int* ft, int T, int V, const int* vt_ptr, const int* vt_tri, const long long* blk_off,
                        long long W, int* wv, int* wt, int* wf, void* stream);

/* Tangent frames of the W welded vertices -> wnormal [W,3], wtangent [W,4] fp32.  normals [V,3].  Returns 1 for NULL buffers
 * (W > 0) or W < 0. */
int nero_gltf_tangents(const float* verts, const int* tris, const float* vt, const int* ft, const int* vt_ptr, const int* vt_tri,
                       const float* normals, const int* wv, const int* wt, int W, float* wnormal, float* wtangent, void* stream);

/* Tangent-space conversion of the object-space map omap [width*height,3] uint8 (row 0 at v = 0 of the atlas) -> img
 * [width*height,5] uint8.  atlas [N,2]: (u, 1 - v) of the file's vt; faces [T,3] the uv triangles (ft); wf, wnormal, wtangent
 * as above.  Returns 1 for NULL required buffers, a bad size or n outside [0, width*height]. */
int nero_gltf_tangent_space(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* atlas,
                            const int* faces, const int* wf, const float* wnormal, const float* wtangent, const unsigned char* omap,
                            unsigned char* img, void* stream);

/* Metallic-roughness texture: metallic [n], roughness [n] uint8 (the red channel of feat1 / feat2), lut_m [256], lut_r [256]
 * -> out [n,3] uint8.  Returns 1 for NULL buffers (n > 0) or n < 0. */
int nero_gltf_metal_rough(const unsigned char* metallic, const unsigned char* roughness, long long n, const unsigned char* lut_m,
                          const unsigned char* lut_r, unsigned char* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_GLTF_H_ */
