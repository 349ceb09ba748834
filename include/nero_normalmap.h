/* libnero_b200 -- C ABI of the normal-map bake: the fine mesh's shading baked onto the UV atlas of its simplification
 * (nero_b200/normalmap.py sequences it; oracle/nero_oracle_normalmap.py restates it in numpy).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 *
 * Convention.  Object-space maps: a texel holds the outward unit normal in the OBJ's own coordinates.  Meshes are wound
 * like marching-cubes meshes, cross(v1 - v0, v2 - v0) pointing into the solid, so a triangle's outward area vector is
 * -cross(e1, e2).  Byte encoding per channel: k = floor((n 0.5 + 0.5) 255 + 0.5) clamped to [0, 255] (fp32, each operation
 * rounded on its own); decoding is linear, 2k/255 - 1, with no sRGB transfer.
 *
 * Vertex normals.  n_v = normalize(sum of -cross(e1, e2) over v's triangles in ascending triangle order), e1 = v1 - v0,
 * e2 = v2 - v0, every fp32 operation rounded on its own (_rn, no contraction); |s| = sqrt((x x + y y) + z z), n = s / |s|; a
 * zero sum gives (0, 0, 0).  One thread per vertex, so the result does not depend on scheduling.
 *
 * Bake.  One thread per covered texel of the atlas (texel [n]: covered texels in row-major order, owner: the raster's owner
 * map).  With the texel's barycentrics b and point p exactly as nero_tex_compact_emit computes them (texel_bary.cuh):
 *   c = normalize(b0 n0 + b1 n1 + b2 n2) from the low mesh's vertex normals (fp32 _rn, ((b0 n0 + b1 n1) + b2 n2));
 *   one ray from p + distance c along -c; the closest hit on the detail BVH with t in (0, 2 distance):
 *     hit  -> normalize(w0 m_a + u m_b + v m_c), the detail vertex normals of the hit triangle (through tri_ids and
 *             detail_faces) interpolated with the hit's barycentrics (w0 = 1 - u - v), fp32 _rn;
 *     miss -> c (also when c is zero: then the normal is zero).
 * The three bytes go to channels 0-2 of img [width*height, 5] at the texel, channels 3-4 are 0 and so is every uncovered
 * texel (the layout nero_tex_inpaint and nero_tex_downsample take).  hit [n] gets 1 / 0.  point, cage and normal [n,3] fp32
 * receive p, c and the baked float normal when they are not NULL.
 */
#ifndef NERO_NORMALMAP_H_
#define NERO_NORMALMAP_H_

#include "nero_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* verts [V,3] fp32, tris [T,3] int32, (vt_ptr [V+1], vt_tri [3T]): each vertex's triangles in ascending order (the CSR of
 * nero_b200.simplify._vertex_triangles) -> normals [V,3] fp32.  Returns 1 for NULL buffers (with V, T > 0) or V, T < 0. */
int nero_normalmap_vertex_normals(const float* verts, int V, const int* tris, int T, const int* vt_ptr, const int* vt_tri, float* normals,
                                  void* stream);

/* The bake of the low mesh (vt, ft, verts, faces, low_normals) against the detail mesh's BVH (nodes, bvh_tris, tri_ids as
 * nero_bvh_build_host writes them, detail_faces [T',3], detail_normals [V',3]).  distance > 0 in scene units.  Returns 1 for
 * NULL required buffers, a bad atlas size, n outside [0, width*height] or distance <= 0 or not finite. */
int nero_normalmap_bake(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* vt, const int* ft,
                        const float* verts, const int* faces, const float* low_normals, const float* nodes, const float* bvh_tris,
                        const int* tri_ids, const int* detail_faces, const float* detail_normals, float distance, unsigned char* img,
                        unsigned char* hit, float* point, float* cage, float* normal, void* stream);

/* nero_relight_render_textured and nero_relight_render_textured_aov (include/nero_denoise.h) with an object-space normal map
 * in texel channels 5-7: tex [tex_h,tex_w,8] = (albedo rgb, metallic, roughness, nx, ny, nz), the outward unit normal in the
 * mesh's own coordinates (the convention above).  The texel's second float4 is loaded whole; the normal is filtered
 * bilinearly like the other channels, then normalised.  Shading rule at a hit:
 *   n_g = the flat normal, -cross(e1, e2) normalised, flipped to face the incoming ray (the rule of the other instances);
 *   n_s = the filtered map normal / its length, flipped by the same sign as n_g; a length below 1e-6 gives n_s = n_g;
 *   if dot(n_s, wo) <= 0 (wo = -ray direction), n_s = n_g;
 *   the BRDF, its pdf and both lobe samplers use n_s;
 *   a light direction l with dot(n_g, l) <= 0 carries nothing, and a continuation with dot(n_g, l) <= 0 ends the path;
 *   ray offsets stay along n_g;
 *   the AOV instance's normal guide is n_s.
 * Arguments and return codes are those of the unmapped pair. */
int nero_relight_render_textured_nmap(const nero_relight_params* q, const float* vt, const int* ft, int n_uv, const float* tex, int tex_w,
                                      int tex_h, void* stream);
int nero_relight_render_textured_nmap_aov(const nero_relight_params* q, const float* vt, const int* ft, int n_uv, const float* tex,
                                          int tex_w, int tex_h, float* aov, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_NORMALMAP_H_ */
