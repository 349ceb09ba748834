/* libnero_b200 -- C ABI of mesh clean-up and area-uniform surface sampling (region crop, connected components, component
 * selection, compaction, sampling of N points).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in
 * nero_b200/evaluate.py, and restated in numpy by oracle/nero_oracle_meshpts.py.
 *
 * A mesh is float32 verts [V,3] and int32 tris [T,3], row-major.  Blocks of the compaction hold NERO_MESHPTS_BLOCK elements:
 * the triangle blocks come first, ceil(T / 256) of them, then the vertex blocks, ceil(V / 256).
 */
#ifndef NERO_MESHPTS_H_
#define NERO_MESHPTS_H_

#define NERO_MESHPTS_BLOCK 256     /* elements per compaction block */
#define NERO_MESHPTS_CHUNK 256     /* triangles per sequential chunk of the cumulative areas */

#ifdef __cplusplus
extern "C" {
#endif

/* area[t] = 0.5 sqrt((cx cx + cy cy) + cz cz), c = (v1 - v0) x (v2 - v0), in uncontracted fp64 from the fp32 vertices; 0 for
 * a triangle with an index outside [0, V).  keep (may be NULL) [T] = 1 iff the indices are in range and all three vertices
 * lie inside the crop, else 0.  sphere (HOST pointer, may be NULL) = cx, cy, cz, r with r > 0: inside iff
 * (dx dx + dy dy) + dz dz <= r r in fp64.  box (HOST pointer, may be NULL) = x0, y0, z0, x1, y1, z1 with x0 <= x1, ...:
 * inside iff x0 <= x <= x1 on every axis.  With both, a vertex must be inside both. */
int nero_meshpts_areas(const float* verts, int V, const int* tris, int T, const double* sphere, const double* box, double* area,
                       unsigned char* keep, void* stream);

/* Connected components of the kept triangles: two triangles are connected when they share a vertex index.  tri_label[t] =
 * the smallest vertex index of t's component for a kept triangle, V for the others.  parent [V] is workspace (it ends
 * holding each vertex's label; unreferenced vertices are their own).  Union-find: hooks to the smaller root by CAS, then
 * ceil(log2 V) + 1 rounds of pointer jumping, enough for any tree depth below V. */
int nero_meshpts_components(const int* tris, int T, const unsigned char* keep, int V, int* parent, int* tri_label, void* stream);

/* Component c (of m) is the kept triangles order[ends[c-1] .. ends[c]) (ends[-1] = 0), listed in ascending triangle index,
 * with label comp_label[c].  comp_area[c] = the fp64 sum of their areas in that order.  root_keep[comp_label[c]] = 1 iff
 * comp_area[c] >= frac * max comp_area (frac in [0, 1]), else 0; other entries of root_keep [V] are not written. */
int nero_meshpts_component_areas(const double* area, const long long* order, const long long* ends, const int* comp_label, int m,
                                 double frac, double* comp_area, unsigned char* root_keep, void* stream);

/* tri_flag[t] = keep[t] && root_keep[tri_label[t]]; vert_flag[v] = 1 iff a flagged triangle references v.  blk_cnt, blk_off
 * [ceil(T/256) + ceil(V/256)]: per-block counts and their exclusive prefix in block order (triangle and vertex blocks each
 * from 0); totals [2] = kept vertices, kept triangles. */
int nero_meshpts_compact_count(const int* tris, int T, const unsigned char* keep, const int* tri_label, const unsigned char* root_keep,
                               int V, unsigned char* tri_flag, unsigned char* vert_flag, int* blk_cnt, long long* blk_off,
                               long long* totals, void* stream);

/* Flagged vertices in their original order -> verts_out [nv,3], remap [V] = each flagged vertex's new index; flagged
 * triangles in their original order with remapped indices -> tris_out [nt,3].  nv, nt: the totals of compact_count. */
int nero_meshpts_compact_emit(const float* verts, int V, const int* tris, int T, const unsigned char* tri_flag,
                              const unsigned char* vert_flag, const long long* blk_off, long long nv, long long nt, int* remap,
                              float* verts_out, int* tris_out, void* stream);

/* Inclusive prefix of area [T] in fp64: chunk k (triangles [256 k, 256 k + 256)) is summed sequentially, partial[t]; the
 * chunk sums s_k are prefixed sequentially, O_k = O_(k-1) + s_(k-1) with O_0 = 0; cdf[t] = O_k + partial[t].
 * chunk [ceil(T/256)] is workspace. */
int nero_meshpts_cdf(const double* area, int T, double* chunk, double* cdf, void* stream);

/* Samples i0 .. i0 + n - 1 -> out [n,3] fp64.  Sample i draws h_d = hash(seed, i, d), d = 0..3 (rl_mix chain of
 * math_relight's form); u0 = ((h_0 >> 5) 2^26 + (h_1 >> 6)) 2^-53, r1 = h_2 2^-32, r2 = h_3 2^-32.  Its triangle is the first t
 * with cdf[t] > u0 cdf[T-1] (the last one if none), found by binary search, so a zero-area triangle is never chosen; with
 * s = sqrt(r1) the point is (b0 v0 + b1 v1) + b2 v2, b = (1 - s, s (1 - r2), s r2), in uncontracted fp64.  A sample
 * depends on (seed, i) and the mesh only. */
int nero_meshpts_sample(const float* verts, int V, const int* tris, int T, const double* cdf, unsigned int seed, long long i0,
                        long long n, double* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_MESHPTS_H_ */
