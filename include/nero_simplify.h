/* libnero_b200 -- C ABI of mesh simplification by deterministic parallel quadric edge collapse (input checks, locks and
 * quadrics; per round: edge placement, cost and validity, independent-set selection, collapse, triangle rewrite; output
 * compaction).
 *
 * Same library and conventions as include/nero_b200.h: pointers are DEVICE pointers unless stated otherwise, `stream` is a
 * cudaStream_t passed as void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked
 * before any launch), 2 on a CUDA launch error.  Plain arguments only (no records).  The protocol is stated in
 * nero_b200/simplify.py, and restated in numpy by oracle/nero_oracle_simplify.py.
 *
 * A mesh is int32 tris [T,3] over V vertices; positions are fp64 pos [V,3] and quadrics fp64 Q [V,10] (entries xx xy xz xw
 * yy yz yw zz zw ww).  Half-edge h = 3 t + k runs tris[t][k] -> tris[t][(k+1) % 3].  CSR rows are int32 (ptr [V+1]), so
 * 6 T must fit int32.  Keys are int64: float32(cost) bits << 32 | edge id, NERO_SIMPLIFY_KEY_INF for an edge that may not
 * collapse.  Blocks of the compactions hold NERO_SIMPLIFY_BLOCK elements.
 */
#ifndef NERO_SIMPLIFY_H_
#define NERO_SIMPLIFY_H_

#define NERO_SIMPLIFY_BLOCK 256                        /* elements per compaction block */
#define NERO_SIMPLIFY_KEY_INF 0x7fffffffffffffffLL     /* key of an edge that may not collapse; also "no error" */

#ifdef __cplusplus
extern "C" {
#endif

/* err [4] = KEY_INF, then err[0] = the smallest triangle with an index outside [0, V), err[1] = the smallest triangle that
 * repeats an index (among those in range). */
int nero_simplify_check_tris(const int* tris, int T, int V, long long* err, void* stream);

/* hkey [n] ascending: (min(s,d) V + max(s,d)) 2 + (s > d) of each half-edge s -> d, hidx [n] its half-edge id, n = 3 T.
 * err[2] = the smallest sorted position starting a run of >= 3 equal edges (an edge in more than two triangles), err[3] =
 * the smallest starting a run of 2 with equal directions (inconsistent winding); twin [n] = the half-edge running the other
 * way along the same edge, -1 on a boundary edge. */
int nero_simplify_check_edges(const long long* hkey, const long long* hidx, long long n, int* twin, long long* err, void* stream);

/* pos = the fp32 verts in fp64; Q = each vertex's triangle quadrics added from 0.0 in ascending triangle order (vt_ptr /
 * vt_tri: the CSR of each vertex's triangles, ascending); tri_q [T,10] is workspace.  locked [V] = 1 for an endpoint of a
 * boundary edge (twin -1) and for a vertex whose fan walk from its first triangle reaches fewer triangles than its degree. */
int nero_simplify_prepare(const float* verts, int V, const int* tris, int T, const int* vt_ptr, const int* vt_tri, const int* twin,
                          double* tri_q, double* pos, double* Q, unsigned char* locked, void* stream);

/* One thread per edge (ea[e] < eb[e], sorted): placement x [E,3] and clamped cost [E] from Q[a] + Q[b]; key [E] =
 * float32(cost) bits << 32 | e when the edge passes the validity tests (locks, link condition through the adjacency CSR
 * adj_ptr / adj with ascending rows, valences, no flip through the triangle CSR vt_ptr / vt_tri of the current tris), else
 * KEY_INF. */
int nero_simplify_edges(const double* pos, const double* Q, const unsigned char* locked, int V, const int* tris, int T,
                        const int* adj_ptr, const int* adj, const int* vt_ptr, const int* vt_tri, const int* ea, const int* eb, int E,
                        double* x, double* cost, long long* key, void* stream);

/* vmin [V] = the smallest key of the edges at each vertex (64-bit atomicMin); rmin [V] = the smallest vmin over the vertex
 * and its neighbours; selected [E] = key != KEY_INF && key == rmin[a] == rmin[b]. */
int nero_simplify_select(const int* ea, const int* eb, int E, const long long* key, const int* adj_ptr, const int* adj, int V,
                         long long* vmin, long long* rmin, unsigned char* selected, void* stream);

/* flag [E] = selected && key <= *thr (thr: one device int64); remap [V] = identity, then for every flagged edge (a, b):
 * pos[a] = x[e], Q[a] = Q[a] + Q[b], remap[b] = a.  The flagged edges share no vertex or triangle, so no write races. */
int nero_simplify_collapse(const int* ea, const int* eb, int E, const long long* key, const unsigned char* selected, const long long* thr,
                           const double* x, int V, double* pos, double* Q, int* remap, unsigned char* flag, void* stream);

/* Triangles rewritten through remap; those left with a repeated index are dropped.  blk_cnt, blk_off [ceil(T/256)]: the kept
 * count per block and its exclusive prefix in block order; total [1] = the kept triangles. */
int nero_simplify_rewrite_count(const int* tris, int T, const int* remap, int* blk_cnt, long long* blk_off, long long* total,
                                void* stream);

/* The kept triangles, rewritten, in their order -> out [nt,3] (nt: the total of rewrite_count). */
int nero_simplify_rewrite_emit(const int* tris, int T, const int* remap, const long long* blk_off, long long nt, int* out, void* stream);

/* vflag [V] = 1 iff a triangle references the vertex; blk_cnt, blk_off [ceil(V/256)] and total [1] as above, over vertices. */
int nero_simplify_output_count(const int* tris, int T, int V, unsigned char* vflag, int* blk_cnt, long long* blk_off, long long* total,
                               void* stream);

/* The flagged vertices in index order, rounded once to float32 -> verts_out [nv,3], remap [V] = their new index; the
 * triangles with remapped indices -> tris_out [T,3]. */
int nero_simplify_output_emit(const double* pos, int V, const int* tris, int T, const unsigned char* vflag, const long long* blk_off,
                              long long nv, int* remap, float* verts_out, int* tris_out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_SIMPLIFY_H_ */
