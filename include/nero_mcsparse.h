/* libnero_b200 -- C ABI of brick-wise marching cubes on a narrow band of the grid: the same mesh as nero_mcubes_count /
 * nero_mcubes_emit (include/nero_b200.h) give on the dense field, from field values at the points of a list of bricks only.
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked before any launch), 2
 * on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in nero_b200/mesh.py (extract_sparse)
 * and restated in numpy by oracle/nero_oracle_mcsparse.py.
 *
 * The grid has nx x ny x nz points (each >= 2) at (ax[i], ay[j], az[k]); the linear index of a point is (i ny + j) nz + k, as
 * int64.  `brick` = B is 4, 8 or 16.  Axis a has nb_a = ceil((n_a - 1) / B) bricks and nb_a + 1 coarse points, coarse point g at
 * grid index min(g B, n_a - 1); bricks and coarse points are numbered like grid points ((bx nb_y + by) nb_z + bz).  Brick b
 * covers the (B+1)^3 grid points b B + d, d in [0, B]^3, clamped to the grid: P = (B+1)^3 values per brick, row
 * (dx (B+1) + dy) (B+1) + dz.  It owns the points with d_a < B or at the last grid index of axis a, the edges based at the
 * points it owns and the cubes based at them, so every edge and cube of the grid has one owner.
 * A corner is below iff u <= iso.
 */
#ifndef NERO_MCSPARSE_H_
#define NERO_MCSPARSE_H_

#define NERO_MCSPARSE_TILE 1024    /* flags per block of the brick compaction */

#ifdef __cplusplus
extern "C" {
#endif

/* rows [count,3] = the positions of coarse points first .. first + count - 1. */
int nero_mcsparse_coarse_points(const float* ax, const float* ay, const float* az, int nx, int ny, int nz, int brick,
                                long long first, long long count, float* rows, void* stream);

/* flag [nb_x nb_y nb_z] = 1 for a seed brick, else 0 (every entry is written).  cval [coarse points]: the raw field;
 * coutside (may be NULL) [coarse points]: 1 where the field is overridden by a constant above iso.  With d_c = cval - iso in
 * fp32 over the brick's 8 corners, a brick is a seed iff min |d_c| <= margin, or some but not all corners are outside and
 * min d_c <= margin. */
int nero_mcsparse_seed(const float* cval, const unsigned char* coutside, int nx, int ny, int nz, int brick, float iso, float margin,
                       unsigned char* flag, void* stream);

/* Flagged entries of flag [n] in ascending order: blk_cnt, blk_off [ceil(n / 1024)] = per-block counts and their exclusive
 * prefix in block order, total [1] = their number.  emit then appends them: list[base + r] = the r-th flagged index,
 * slot[that index] = base + r, and clears the flag. */
int nero_mcsparse_compact_count(const unsigned char* flag, long long n, int* blk_cnt, long long* blk_off, long long* total,
                                void* stream);
int nero_mcsparse_compact_emit(unsigned char* flag, long long n, const long long* blk_off, long long base, int* list, int* slot,
                               void* stream);

/* rows [count P, 3] = the positions of the points of bricks list[first .. first + count - 1], P rows per brick. */
int nero_mcsparse_brick_points(const float* ax, const float* ay, const float* az, int nx, int ny, int nz, int brick, const int* list,
                               long long first, long long count, float* rows, void* stream);

/* For bricks list[first .. first + count - 1], whose values are pool[j P .. j P + P) for list entry j: each of the six
 * neighbours that exists and has slot < 0 gets flag = 1 if a grid edge in the plane of points the two bricks share has its
 * ends on different sides of iso.  Other flags are not written. */
int nero_mcsparse_grow(const float* pool, const int* list, long long first, long long count, const int* slot, int nx, int ny, int nz,
                       int brick, float iso, unsigned char* flag, void* stream);

/* blk_cnt [2 n_bricks] = (vertices, triangles) owned by each listed brick, blk_off [2 n_bricks] their exclusive prefixes in
 * list order, totals [2] = V, T. */
int nero_mcsparse_count(const float* pool, const int* list, long long n_bricks, int nx, int ny, int nz, int brick, float iso,
                        int* blk_cnt, long long* blk_off, long long* totals, void* stream);

/* Vertex r: vkey [V] = 3 L + a for the edge (p, p + e_a), L the linear index of p; vpos [V,3] = p + t e_a in index space,
 * t = (iso - u(p)) / (u(p + e_a) - u(p)) in fp32.  Triangle r: tkey [T] = 5 C + s for the s-th triangle of the cube with
 * linear index C (table order of nero_b200/csrc/mc_tables.cuh), tedge [T,3] = the keys of its three vertices.  Rows are in
 * list order, then point order inside a brick; sorting by key gives the order of nero_mcubes_emit. */
int nero_mcsparse_emit(const float* pool, const int* list, long long n_bricks, int nx, int ny, int nz, int brick, float iso,
                       const long long* blk_off, long long* vkey, float* vpos, long long* tkey, long long* tedge, void* stream);

/* out[i] = the index of key[i] in the ascending array sorted [n_sorted] (binary search), -1 if it is not there; i < n. */
int nero_mcsparse_lookup(const long long* sorted, long long n_sorted, const long long* key, long long n, int* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_MCSPARSE_H_ */
