/* libnero_b200 -- C ABI of the ambient-occlusion bake: cosine-weighted visibility within a distance, counted per point or per
 * texel of the UV atlas (nero_b200/occlusion.py sequences it; oracle/nero_oracle_occlusion.py restates it in numpy).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 *
 * Stored value.  From a point q with unit normal n_g, N rays over the cosine-weighted hemisphere of n_g; a ray is unoccluded
 * if it hits no occluder triangle with t in (0, distance).  The value is the unoccluded count c of N.
 *
 * Sampler (a Hammersley set with a per-point Cranley-Patterson rotation; a pure function of (seed, key, i, N), fp32, every
 * operation rounded on its own):
 *   xi1 = rl_uniform(seed, key, 0, 0, 0), xi2 = rl_uniform(seed, key, 0, 0, 1)        (math_relight.cuh)
 *   a = (2i + 1) / (2N) + xi1,                  r1 = a if a < 1 else a - 1               (i in [0, N))
 *   b = (__brev(i) >> 8) 2^-24 + xi2,            r2 = b if b < 1 else b - 1
 *   l = rl_sample_diffuse(n_g, r1, r2)                                                  (math_relight.cuh)
 * Ray: origin q + kRelightEps n_g (1e-4, fp32 _rn per component), direction l, t in (0, distance), any hit on the occluder
 * BVH (bvh_traverse<true>, nodes and triangles as nero_bvh_build_host writes them).  A row whose n_g is (0, 0, 0) counts
 * c = N without casting.  One warp per row, lanes striding the rays, the count summed with __reduce_add_sync: integers only,
 * so the result does not depend on scheduling.
 *
 * Byte: k = (510 c + N) div (2N) in integers, round-half-up of 255 c / N, linear (no sRGB transfer).
 *
 * Texel points.  Meshes are wound with cross(e1, e2) pointing into the solid, so the flat outward normal of a triangle is
 * normalize(-cross(e1, e2)) with e1 = v1 - v0, e2 = v2 - v0, each fp32 operation rounded on its own and |s| =
 * sqrt((x x + y y) + z z); a zero cross product gives (0, 0, 0).  One thread per covered texel L (texel [n]: covered texels in
 * row-major order, owner: the raster's owner map), key = L, and with b, p exactly as nero_tex_compact_emit computes them
 * (texel_bary.cuh):
 *   self   (detail nodes NULL): q = p, n_g = the flat outward normal of the owner triangle, hit = 1;
 *   detail (the normal bake's cage ray, include/nero_normalmap.h): c = normalize(b0 n0 + b1 n1 + b2 n2) from the low mesh's
 *          vertex normals, o = p + cage_distance c, the closest hit with t in (0, 2 cage_distance) along -c on the detail
 *          BVH.  Hit: q = o + t (-c) (fp32 _rn), n_g = normalize(-cross(e1, e2)) of the hit triangle from the BVH's e1, e2,
 *          hit = 1.  Miss, or c zero: q = p, n_g = (0, 0, 0) (so the count is N and the byte 255), hit = 0.
 */
#ifndef NERO_OCCLUSION_H_
#define NERO_OCCLUSION_H_

#include "nero_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* The counting kernel on arbitrary rows: points [n,3], normals [n,3] fp32 (unit, or zero), keys [n] uint32 (NULL: the row
 * index) -> counts [n] int32 in [0, rays].  nodes / bvh_tris: the occluder BVH.  Returns 1 for NULL required buffers, n < 0,
 * rays outside [1, 65536] or distance <= 0 or not finite. */
int nero_occlusion_points(const float* points, const float* normals, const unsigned int* keys, long long n, const float* nodes,
                          const float* bvh_tris, int rays, float distance, unsigned int seed, int* counts, void* stream);

/* The points, normals, keys and hit flags of the covered texels (texel [n] of a width x height raster of the low mesh: vt, ft,
 * verts, faces).  Self source: nodes, bvh_tris and low_normals may be NULL (nodes NULL selects it).  Detail source: nodes,
 * bvh_tris of the detail mesh's BVH and low_normals [V,3] (nero_normalmap_vertex_normals of the low mesh), cage_distance > 0.
 * points / normals [n,3], keys [n], hit [n] are required; surface [n,3] (p) and cage [n,3] (c, zero for the self source)
 * receive the texel's point and cage direction when they are not NULL.  Returns 1 for NULL required buffers, a bad atlas
 * size, n outside [0, width*height] or, with a detail mesh, cage_distance <= 0 or not finite. */
int nero_occlusion_texels(const unsigned int* owner, int width, int height, const int* texel, long long n, const float* vt, const int* ft,
                          const float* verts, const int* faces, const float* low_normals, const float* nodes, const float* bvh_tris,
                          float cage_distance, float* points, float* normals, unsigned int* keys, unsigned char* hit, float* surface,
                          float* cage, void* stream);

/* The bytes of counts [n] of texel [n]: k to channels 0-2 of img [width*height, 5], channels 3-4 and every uncovered texel 0
 * (the layout nero_tex_inpaint and nero_tex_downsample take).  Returns 1 for NULL required buffers, a bad atlas size, n
 * outside [0, width*height] or rays outside [1, 65536]. */
int nero_occlusion_bytes(const int* texel, long long n, const int* counts, int rays, int width, int height, unsigned char* img,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_OCCLUSION_H_ */
