/* libnero_b200 -- C ABI of custom-object preparation: the crop of a COLMAP point cloud, RANSAC hypotheses of the support
 * plane and their inlier counts, least-squares refit sums, and object isolation by voxel connected components.
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in
 * nero_b200/objprep.py, and restated in numpy by oracle/nero_oracle_objprep.py.
 *
 * A cloud is fp64 pts [n,3], row-major, n < 2^31.  A plane is 4 fp64 (nx, ny, nz, d); the signed distance of p is
 * r = ((nx px + ny py) + nz pz) + d, and every such expression is evaluated in uncontracted fp64 (no FMA).
 */
#ifndef NERO_OBJPREP_H_
#define NERO_OBJPREP_H_

#define NERO_OBJPREP_BLOCK 256     /* elements per compaction block */
#define NERO_OBJPREP_CHUNK 4096    /* points per block of the refit sums (256 threads x 16 points) */
#define NERO_OBJPREP_MOMENTS 10    /* refit sums per block: count, sum d (3), sum d d^T (xx, xy, xz, yy, yz, zz) */

#ifdef __cplusplus
extern "C" {
#endif

/* keep [n] = 1 iff pts[i] lies inside the crop, else 0.  sphere (HOST pointer, may be NULL) = cx, cy, cz, r with r > 0:
 * inside iff (dx dx + dy dy) + dz dz <= r r.  box (HOST pointer, may be NULL) = x0, y0, z0, x1, y1, z1 with x0 <= x1, ...:
 * inside iff x0 <= x <= x1 on every axis.  With both, a point must be inside both; with neither, every point is kept.  The
 * semantics of nero_meshpts_areas, on fp64 points. */
int nero_objprep_crop(const double* pts, long long n, const double* sphere, const double* box, unsigned char* keep, void* stream);

/* Ordered compaction, step 1: blk_cnt [ceil(n/256)] = flagged elements per 256-element block, blk_off = their exclusive
 * prefix in block order, *total (device) = the flagged count. */
int nero_objprep_compact_count(const unsigned char* flag, long long n, int* blk_cnt, long long* blk_off, long long* total, void* stream);

/* Ordered compaction, step 2: the m flagged points in their original order -> idx [m] (int32 original index) and, if out is
 * not NULL, out [m,3] (their coordinates).  m: the total of compact_count. */
int nero_objprep_compact_emit(const double* pts, const unsigned char* flag, long long n, const long long* blk_off, long long m, int* idx,
                              double* out, void* stream);

/* Plane hypotheses of the n kept points pts (compacted).  Hypothesis k < H draws h_d = hash(seed, k, d), d = 0, 1, 2, with
 * hash(s, k, d) = mix(mix(mix(s 0x9e3779b9 + 0x7f4a7c15) ^ k) ^ d) (mix: rl_mix of hash.cuh, uint32 arithmetic), and takes
 * the points j_d = (h_d n) >> 32 (64-bit product) -> sample [H,3] (int32).  With e1 = p1 - p0, e2 = p2 - p0 and
 * c = e1 x e2, it is valid iff |c|^2 > 1e-20 |e1|^2 |e2|^2 (squared norms as ((x x + y y) + z z)), i.e. the sine of the angle
 * at p0 exceeds 1e-10, so collinear and repeated points are invalid.  A valid plane is nhat = c / sqrt|c|^2 (per component),
 * d = -((nhat_x p0x + nhat_y p0y) + nhat_z p0z) -> planes [H,4]; an invalid one is (NaN, NaN, NaN, NaN), valid [H] = 1 / 0.
 * Needs n >= 3. */
int nero_objprep_hypotheses(const double* pts, long long n, int H, unsigned int seed, double* planes, int* sample, unsigned char* valid,
                            void* stream);

/* counts [H] (int64) = the number of points with |r_k(p)| <= tol for plane k of planes [H,4] (0 for a NaN plane).  Integer
 * sums only, so the counts do not depend on the launch configuration. */
int nero_objprep_counts(const double* pts, long long n, const double* planes, int H, double tol, long long* counts, void* stream);

/* Refit sums of the inliers |r(p)| <= tol of plane (HOST pointer, 4 doubles), with d = p - center (center: HOST pointer, 3
 * doubles).  Block b takes points [4096 b, 4096 b + 4096); thread t of it adds, in j order, the terms of its inlier points
 * 4096 b + 256 j + t, j = 0..15 (starting from 0); the 256 thread sums are combined by the tree s[t] += s[t + w],
 * w = 128, 64, .., 1 -> partial [ceil(n/4096), 10]; then out [10] = partial[0] + partial[1] + ... in block order.  The
 * ten sums are: count (as a double), d_x, d_y, d_z, d_x d_x, d_x d_y, d_x d_z, d_y d_y, d_y d_z, d_z d_z.  So the result
 * depends on (pts, n, plane, tol, center) only, bit for bit. */
int nero_objprep_moments(const double* pts, long long n, const double* plane, double tol, const double* center, double* partial, double* out,
                         void* stream);

/* flag [n] = keep[i] && r(p_i) >= above for plane (HOST pointer, 4 doubles).  keys [n] = the packed voxel key
 * (a << 42) | (b << 21) | c of a flagged point, a = floor((x - origin_x) / voxel) in fp64 (b, c likewise), and
 * 0x7fffffffffffffff for the others.  origin (HOST pointer, 3 doubles) and voxel > 0: the caller guarantees that every
 * flagged point has 0 <= a, b, c < 2^21. */
int nero_objprep_above(const double* pts, long long n, const unsigned char* keep, const double* plane, double above, const double* origin,
                       double voxel, unsigned char* flag, long long* keys, void* stream);

/* 26-connected components of the m occupied voxels ukeys [m] (strictly ascending packed keys).  Each voxel looks up its 13
 * neighbours with a larger key by binary search and unites with them: hooks to the smaller root by CAS, then
 * ceil(log2 m) + 1 rounds of pointer jumping.  label [m] = the smallest voxel index of the component; parent [m] is
 * workspace. */
int nero_objprep_voxel_components(const long long* ukeys, long long m, int* parent, int* label, void* stream);

/* comp_count [m] (int64): at index r, the sum of vcount [m] (points per voxel) over the voxels labelled r (0 for indices
 * that are no label).  voxel_keep [m] = 1 iff double(comp_count[label[v]]) >= frac * double(max comp_count), frac in
 * [0, 1]. */
int nero_objprep_component_select(const int* label, const long long* vcount, long long m, double frac, long long* comp_count,
                                  unsigned char* voxel_keep, void* stream);

/* out [n] = flag[i] && voxel_keep[v], v the index of keys[i] in ukeys [m] (binary search; it must be there). */
int nero_objprep_point_keep(const long long* keys, const unsigned char* flag, long long n, const long long* ukeys, long long m,
                            const unsigned char* voxel_keep, unsigned char* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_OBJPREP_H_ */
