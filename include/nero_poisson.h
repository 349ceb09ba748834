/* libnero_b200 -- C ABI of screened Poisson surface reconstruction on a regular grid: cell binning of oriented samples, the
 * gather splats of the normal field and of the sample density, the right-hand side, the operator, the pieces of a
 * geometric-multigrid V-cycle, the fp64 dot-product partials and the CG vector updates, interpolation, and the trim test
 * (nero_b200/poisson.py sequences them; oracle/nero_oracle_poisson.py restates every kernel in numpy).
 *
 * Same library and conventions as include/nero_align.h: pointers are DEVICE pointers, `stream` is a cudaStream_t passed as
 * void*, no allocation and no host synchronisation inside, 0 on success, 1 on a bad argument (checked before any launch), 2
 * on a CUDA launch error.  Every fp32 operation is one correctly rounded __fadd_rn / __fsub_rn / __fmul_rn / __fdiv_rn, never
 * contracted into an FMA, in the order stated here, so numpy reproduces every bit.  No floating-point atomics anywhere.
 *
 * Grid.  N nodes per axis (3 <= N <= NERO_POISSON_MAX_N), node (i, j, k) at index (i N + j) N + k, unit spacing (grid
 * units).  Cell (i, j, k), i, j, k < N - 1, has key (i (N - 1) + j) (N - 1) + k.  The x-edge lattice has (N - 1) x N x N
 * entries, edge (i, j, k) joining nodes (i, j, k) and (i + 1, j, k) with its midpoint at (i + 1/2, j, k); the y and z
 * lattices likewise (N x (N - 1) x N and N x N x (N - 1), row-major).
 *
 * Hat weight.  For a sample at q and a lattice point c, w = (h(q.x - c.x) h(q.y - c.y)) h(q.z - c.z) with h(d) = 1 - |d|;
 * the sample contributes nothing when any factor is <= 0.  Samples are sorted by cell key (stable) and start [cells + 1]
 * holds the first sorted sample of each cell (start[cells] = n).  A gather visits its support cells with x outermost and z
 * innermost, each cell's samples in sorted order, and accumulates acc = acc + term from acc = 0.
 *
 * Stencils.  The neighbours of a node are visited in the order -x, +x, -y, +y, -z, +z, and only those inside the grid (Neumann
 * boundary).  L x at node n = the sum in that order of (x_n - x_m) over its neighbours m.
 */
#ifndef NERO_POISSON_H_
#define NERO_POISSON_H_

#include "nero_b200.h"

#define NERO_POISSON_BLOCK 256
#define NERO_POISSON_MAX_N 1025

#ifdef __cplusplus
extern "C" {
#endif

/* q [n,3] fp32 = fp32((p - o) / h) per axis in fp64 (one __dsub_rn, one __ddiv_rn, rounded to nearest), clamped to
 * [0, N - 1]; keys [n] = the key of cell min(floor(q), N - 2) per axis.  Returns 1 for n < 1, N out of range, h <= 0 or NaN,
 * or NULL buffers. */
int nero_poisson_keys(const double* points, long long n, double ox, double oy, double oz, double h, int N, float* q, int* keys,
                      void* stream);

/* start [cells + 1] = for each c in [0, cells] the first index i of the ascending keys [n] with keys[i] >= c (n if none).
 * Returns 1 for n < 1, cells < 1 or NULL buffers. */
int nero_poisson_cell_starts(const int* keys, long long n, int cells, int* start, void* stream);

/* The normal field: v_a [lattice a] = (gather over the 3 x 2 x 2 cells (i - 1 .. i + 1 along a, j - 1 .. j and k - 1 .. k
 * along the others, clipped to the grid) of w nrm_a) / sigma, with w the hat weight of the sorted sample q [n,3] at the
 * edge midpoint and nrm [n,3] the sorted unit normals.  Returns 1 for n < 1, N out of range, sigma <= 0 or NULL buffers. */
int nero_poisson_edge_splat(const float* q, const float* nrm, long long n, const int* start, int N, float sigma, float* vx, float* vy,
                            float* vz, void* stream);

/* density [N^3] = gather over the 2 x 2 x 2 cells i - 1 .. i, j - 1 .. j, k - 1 .. k (clipped) of w; diag [N^3] = the same
 * gather of w w.  Returns 1 for n < 1, N out of range or NULL buffers. */
int nero_poisson_node_splat(const float* q, long long n, const int* start, int N, float* density, float* diag, void* stream);

/* b [N^3] = G^T v: per axis x, y, z in turn, acc = acc + v_a[edge ending at the node] (if any), then acc = acc - v_a[edge
 * starting at the node] (if any).  Returns 1 for N out of range or NULL buffers. */
int nero_poisson_rhs(const float* vx, const float* vy, const float* vz, int N, float* b, void* stream);

/* out [m] = sum over the 8 corners of cell c = min(max(floor(q), 0), N - 2) (x outermost, z innermost) of w grid[corner], w
 * the hat weight of q [m,3] at the corner.  Returns 1 for m < 1, N out of range or NULL buffers. */
int nero_poisson_interp(const float* grid, int N, const float* q, long long m, float* out, void* stream);

/* y [N^3] = A x = L x + ws S^T S x: first sx [n] = interp(x, q) at the sorted samples (workspace), then per node
 * y = (L x) + ws t with t = the node-splat gather of w sx.  Returns 1 for n < 1, N out of range or NULL buffers. */
int nero_poisson_matvec(const float* x, int N, const float* q, long long n, const int* start, float ws, float* sx, float* y,
                        void* stream);

/* One colour of red-black Gauss-Seidel on the level operator s L + diag(d): every node with (i + j + k) mod 2 == colour gets
 * x = (b + s m) / (s deg + d), m = the sum of its neighbours' x in stencil order, deg = their number.  Returns 1 for N out
 * of range, colour not 0 or 1, s <= 0 or NULL buffers. */
int nero_poisson_smooth(float* x, const float* b, const float* d, int N, float s, int colour, void* stream);

/* r = b - ((s (L x)) + d x) on one level.  Returns 1 for N out of range, s <= 0 or NULL buffers. */
int nero_poisson_residual(const float* x, const float* b, const float* d, int N, float s, float* r, void* stream);

/* coarse [Nc^3], Nc = (Nf - 1) / 2 + 1, Nf odd: coarse[I] = the sum over the offsets (dx, dy, dz) in {-1, 0, 1}^3 (dx outermost)
 * with 2 I + d inside the fine grid of (wx wy) wz fine[2 I + d], w = 1 for 0 and 1/2 for +-1 (the transpose of
 * prolongation: full weighting times 8).  Returns 1 for Nf even or out of range, or NULL buffers. */
int nero_poisson_restrict(const float* fine, int Nf, float* coarse, void* stream);

/* fine [Nf^3] += trilinear prolongation of coarse [Nc^3]: fine[n] = fine[n] + sum over the coarse parents (one per axis at an
 * even index i, I = i / 2 with weight 1; two at an odd one, (i - 1) / 2 and (i + 1) / 2 with 1/2 each; x outermost) of
 * (wx wy) wz coarse[parent].  Returns 1 for Nc out of range or NULL buffers. */
int nero_poisson_prolong(const float* coarse, int Nc, float* fine, void* stream);

/* Partials [ceil(n / 256)] fp64 of (double) a[i] (double) b[i] (or (double) a[i] when b is NULL), each block summed by the
 * pairwise tree of include/nero_align.h; nero_align_reduce finishes the sum.  Returns 1 for n < 1 or NULL a, partial. */
int nero_poisson_dot(const float* a, const float* b, long long n, double* partial, void* stream);

/* The CG step: x = x + alpha p, r = r - alpha ap.  Returns 1 for n < 1 or NULL buffers. */
int nero_poisson_update(float* x, float* r, const float* p, const float* ap, float alpha, long long n, void* stream);

/* The CG direction: p = z + beta p.  Returns 1 for n < 1 or NULL buffers. */
int nero_poisson_direction(float* p, const float* z, float beta, long long n, void* stream);

/* keep [T] = 1 iff all three vertices of tris [T,3] have dens >= threshold, else 0.  Returns 1 for T < 1, V < 1 or NULL
 * buffers. */
int nero_poisson_trim(const float* dens, int V, const int* tris, int T, float threshold, unsigned char* keep, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERO_POISSON_H_ */
