/* libnero_b200 -- C ABI of relighting with UV-textured materials (the textured OBJ that
 * tools/extract_materials_texture_map.py writes, relit by tools/relight.py --obj).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument, 2 on a CUDA launch error.
 * The scene is stated in nero_b200/relight.py.
 */
#ifndef NERO_RELIGHT_TEX_H_
#define NERO_RELIGHT_TEX_H_

#include "nero_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* nero_relight_render with the materials read from textures instead of q->vmat, which must be NULL; every other field of q
 * means what it means there.  vt [n_uv,2] fp32 uv; ft [T,3] int32 indices into vt, in input-triangle order, read through
 * q->tri_ids as q->faces is; tex [tex_h,tex_w,8] fp32 linear values laid out like vmat (albedo rgb, metallic, roughness, 3
 * unused), row 0 the top row of the image file.  Material at a hit with barycentrics (u, v), w0 = 1 - u - v:
 *   uv = w0 uv0 + u uv1 + v uv2 (fp32);  s = uv.x tex_w - 1/2,  t = (1 - uv.y) tex_h - 1/2  (v = 0 is the bottom row);
 *   x0 = floor(s), fx = s - x0 (y likewise); the taps x0, x0 + 1 and y0, y0 + 1 wrap (repeat, positive modulo);
 *   bilinear in lerp form, a + f (b - a), per channel, x first; no mip-mapping.
 *   albedo and metallic are the filtered values; alpha = the filtered roughness, NOT squared (the texture export stores the
 *   rescaled roughness NeRO's shading takes; the per-vertex export stores its square root).
 * Returns 1 also for NULL vt, ft or tex, n_uv < 1, tex_w < 1 or tex_h < 1.  ft is not range-checked here. */
int nero_relight_render_textured(const nero_relight_params* q, const float* vt, const int* ft, int n_uv, const float* tex, int tex_w,
                                 int tex_h, void* stream);

/* The normal-mapped instances, nero_relight_render_textured_nmap and _nmap_aov, are declared in include/nero_normalmap.h. */

#ifdef __cplusplus
}
#endif
#endif /* NERO_RELIGHT_TEX_H_ */
