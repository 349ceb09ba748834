/* libnero_b200 -- C ABI of the UV texture-map export (the GPU replacement of the reference's
 * extract_materials_texture_map.py: xatlas, the nvdiffrast rasteriser, scipy's morphology and sklearn's kd-tree).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless marked host, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument,
 * 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in nero_b200/texmap.py.
 *
 * Raster conventions: the atlas is `width` x `height` texels; texel (x, y) samples uv = ((x + 1/2) / width,
 * (y + 1/2) / height), row 0 is v = 0.  Images are row-major [height, width, 5] uint8 (albedo rgb, metallic, roughness).
 */
#ifndef NERO_TEXMAP_H_
#define NERO_TEXMAP_H_

#ifdef __cplusplus
extern "C" {
#endif

/* Host UV unwrapper (init-time host code, runs without a GPU).  verts [V,3] fp32, tris [T,3] int32 (host).  Charts grow
 * breadth-first from seeds in triangle order across edges used by exactly two triangles in opposite directions, within a
 * 60 degree normal cone, while the projection onto the plane normal to the seed stays injective (exact predicates).
 * Charts are turned to their principal axes and shelf-packed at one texel density, the largest that fits with `gutter`
 * texels between charts and from the border.  Outputs (host, caller-allocated): vt_out [3T,2] fp32 in [0,1], ft_out [T,3]
 * int32 indices into vt_out, *n_uv rows of vt_out used, *n_charts.  Returns 1 if the charts cannot fit the atlas. */
int nero_uv_atlas_host(const float* verts, int V, const int* tris, int T, int width, int height, int gutter, float* vt_out,
                       int* ft_out, int* n_uv, int* n_charts);

/* One thread per uv triangle over its texel bounding box.  uv is snapped to 1/256 texel; exact int64 edge functions with the
 * top-left rule decide coverage, so a texel centre on a shared edge belongs to one triangle.  owner [W*H] is filled with
 * 0xffffffff (uncovered) and then atomicMin'ed with the covering triangle ids; cover [W*H] counts covering triangles. */
int nero_tex_raster(const float* vt, const int* ft, int T, int width, int height, unsigned int* owner, int* cover, void* stream);

/* Ordered compaction of the covered texels in row-major order: count -> one-block scan (blk_cnt [nblk], blk_off [nblk],
 * *total on the device) -> emit.  nblk = ceil(W*H / 1024).  emit writes texel [n] (row-major index) and xyz [n,3] = the
 * positions verts[faces] interpolated in fp32 with the barycentrics of the raster's edge functions. */
int nero_tex_compact_count(const unsigned int* owner, int width, int height, int* blk_cnt, long long* blk_off, long long* total,
                           void* stream);
int nero_tex_compact_emit(const unsigned int* owner, int width, int height, const float* vt, const int* ft, const float* verts,
                          const int* faces, const long long* blk_off, long long n, int* texel, float* xyz, void* stream);

/* img [W*H,5] uint8 = 0, then img[texel[i]] = (uint8)(linear_to_srgb(mat[i]) * 255) per channel, the transfer evaluated in
 * fp64 as numpy evaluates it (utils/raw_utils.py:11-15) and truncated.  mat [n,5] fp32. */
int nero_tex_encode(const float* mat, const int* texel, long long n, int width, int height, unsigned char* img, void* stream);

/* Seam inpainting (extract_materials_texture_map.py:136-149).  search [W*H] = covered texels within Manhattan distance 3 of
 * an uncovered texel or the border; tile_occ [ceil(H/16)*ceil(W/16)] marks 16x16 tiles holding a search texel.  Every
 * uncovered texel with a covered texel within Manhattan distance 32 copies the 5 bytes of its Euclidean-nearest search texel
 * (smallest squared distance, then smallest row-major index); src [W*H] is that texel's index, -1 elsewhere.  out = img
 * with those copies. */
int nero_tex_inpaint(const unsigned char* img, const unsigned int* owner, int width, int height, unsigned char* search, int* tile_occ,
                     unsigned char* out, int* src, void* stream);

/* 2x down-sample of [H,W,5] uint8 (W, H even): (a + b + c + d + 2) >> 2 per channel -> [H/2, W/2, 5]. */
int nero_tex_downsample(const unsigned char* img, int width, int height, unsigned char* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_TEXMAP_H_ */
