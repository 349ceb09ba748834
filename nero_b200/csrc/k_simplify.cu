// Mesh simplification by parallel quadric edge collapse.  The protocol is stated in nero_b200/simplify.py, the ABI in
// include/nero_simplify.h, and oracle/nero_oracle_simplify.py restates every kernel in numpy.
//
//   check        one thread per triangle (index range, repeats); one thread per run of the sorted half-edge keys (edges in
//                more than two triangles, inconsistent winding, twins).  Errors keep the smallest offender by integer
//                atomicMin, which does not depend on order.
//   prepare      one thread per triangle: its quadric; one thread per vertex: the sum of its triangles' quadrics in
//                ascending triangle order, and the lock (boundary edge, or a fan walk that misses triangles).
//   edges        one thread per edge: the adjugate placement or the cheapest of a, b and the midpoint, the cost, and the
//                validity tests (locks, link condition by a merge of the two sorted adjacency rows, valences, no flip).
//   select       64-bit atomicMin of the keys at each vertex, the minimum over each closed 1-ring, the equality test.
//   collapse     one thread per flagged edge: disjoint vertices, so plain stores.
//   compaction   flags -> per-block counts -> one-block int64 scan -> emit in order (compact.cuh).
//
// Every fp64 product and sum is one rounded operation (__dmul_rn / __dadd_rn / ...), never contracted into an FMA, in the
// order the oracle writes; floating-point values are never combined by atomics, so every output is bit-identical from run
// to run.
#include "common.cuh"
#include "compact.cuh"
#include "../../include/nero_simplify.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_SIMPLIFY_BLOCK;
constexpr long long kKeyInf = NERO_SIMPLIFY_KEY_INF;
constexpr double kDetEps = 1e-10;

__device__ __forceinline__ double dm(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double da(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double ds(double a, double b) { return __dsub_rn(a, b); }

struct D3 {
  double x, y, z;
};

__device__ __forceinline__ D3 load3(const double* __restrict__ p, int i) {
  return D3{p[3 * (size_t)i], p[3 * (size_t)i + 1], p[3 * (size_t)i + 2]};
}

// (p1 - p0) x (p2 - p0)
__device__ __forceinline__ D3 cross3(const D3& p0, const D3& p1, const D3& p2) {
  const double e1x = ds(p1.x, p0.x), e1y = ds(p1.y, p0.y), e1z = ds(p1.z, p0.z);
  const double e2x = ds(p2.x, p0.x), e2y = ds(p2.y, p0.y), e2z = ds(p2.z, p0.z);
  return D3{ds(dm(e1y, e2z), dm(e1z, e2y)), ds(dm(e1z, e2x), dm(e1x, e2z)), ds(dm(e1x, e2y), dm(e1y, e2x))};
}

__device__ __forceinline__ double dot3(const D3& a, const D3& b) { return da(da(dm(a.x, b.x), dm(a.y, b.y)), dm(a.z, b.z)); }

// x^T M x + 2 g^T x + c
__device__ __forceinline__ double quadric_cost(const double* q, const D3& x) {
  const double mx0 = da(da(dm(q[0], x.x), dm(q[1], x.y)), dm(q[2], x.z));
  const double mx1 = da(da(dm(q[1], x.x), dm(q[4], x.y)), dm(q[5], x.z));
  const double mx2 = da(da(dm(q[2], x.x), dm(q[5], x.y)), dm(q[7], x.z));
  const double xmx = da(da(dm(x.x, mx0), dm(x.y, mx1)), dm(x.z, mx2));
  const double gx = da(da(dm(q[3], x.x), dm(q[6], x.y)), dm(q[8], x.z));
  return da(da(xmx, dm(2.0, gx)), q[9]);
}

// ------------------------------------------------------------------------------------------------ checks
__global__ void __launch_bounds__(kBlock) err_init_kernel(long long* err) {
  if (threadIdx.x < 4) err[threadIdx.x] = kKeyInf;
}

__global__ void __launch_bounds__(kBlock) check_tris_kernel(const int* __restrict__ tris, int T, int V, long long* err) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  const int i0 = __ldg(tris + 3 * (size_t)t), i1 = __ldg(tris + 3 * (size_t)t + 1), i2 = __ldg(tris + 3 * (size_t)t + 2);
  const bool in = i0 >= 0 && i0 < V && i1 >= 0 && i1 < V && i2 >= 0 && i2 < V;
  if (!in) atomicMin((unsigned long long*)err, (unsigned long long)t);
  else if (i0 == i1 || i1 == i2 || i0 == i2) atomicMin((unsigned long long*)(err + 1), (unsigned long long)t);
}

__global__ void __launch_bounds__(kBlock) check_edges_kernel(const long long* __restrict__ hkey, const long long* __restrict__ hidx,
                                                             long long n, int* __restrict__ twin, long long* err) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const long long e = hkey[i] >> 1;
  if (i > 0 && (hkey[i - 1] >> 1) == e) return;          // not the start of a run
  int len = 1;
  while (len < 3 && i + len < n && (hkey[i + len] >> 1) == e) ++len;
  if (len >= 3) {
    atomicMin((unsigned long long*)(err + 2), (unsigned long long)i);
    return;
  }
  if (len == 1) {
    twin[hidx[i]] = -1;
    return;
  }
  if ((hkey[i] & 1) == (hkey[i + 1] & 1)) {
    atomicMin((unsigned long long*)(err + 3), (unsigned long long)i);
    return;
  }
  twin[hidx[i]] = int(hidx[i + 1]);
  twin[hidx[i + 1]] = int(hidx[i]);
}

// ------------------------------------------------------------------------------------------------ quadrics and locks
__global__ void __launch_bounds__(kBlock) tri_quadric_kernel(const float* __restrict__ verts, const int* __restrict__ tris, int T,
                                                             double* __restrict__ tri_q) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  D3 p[3];
  for (int k = 0; k < 3; ++k) {
    const int v = __ldg(tris + 3 * (size_t)t + k);
    p[k] = D3{double(__ldg(verts + 3 * (size_t)v)), double(__ldg(verts + 3 * (size_t)v + 1)), double(__ldg(verts + 3 * (size_t)v + 2))};
  }
  const D3 n = cross3(p[0], p[1], p[2]);
  const double ln = __dsqrt_rn(dot3(n, n));
  double* q = tri_q + 10 * (size_t)t;
  if (!(ln > 0.0)) {
    for (int j = 0; j < 10; ++j) q[j] = 0.0;
    return;
  }
  const double nx = __ddiv_rn(n.x, ln), ny = __ddiv_rn(n.y, ln), nz = __ddiv_rn(n.z, ln);
  const double pp[4] = {nx, ny, nz, -da(da(dm(nx, p[0].x), dm(ny, p[0].y)), dm(nz, p[0].z))};
  const double A = dm(ln, 0.5);
  int j = 0;
  for (int a = 0; a < 4; ++a)
    for (int b = a; b < 4; ++b) q[j++] = dm(A, dm(pp[a], pp[b]));
}

__global__ void __launch_bounds__(kBlock) vertex_kernel(const float* __restrict__ verts, int V, const int* __restrict__ tris,
                                                        const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                        const int* __restrict__ twin, const double* __restrict__ tri_q,
                                                        double* __restrict__ pos, double* __restrict__ Q, unsigned char* __restrict__ locked) {
  const int v = blockIdx.x * kBlock + threadIdx.x;
  if (v >= V) return;
  for (int j = 0; j < 3; ++j) pos[3 * (size_t)v + j] = double(__ldg(verts + 3 * (size_t)v + j));
  const int r0 = vt_ptr[v], r1 = vt_ptr[v + 1];
  double s[10];
  for (int j = 0; j < 10; ++j) s[j] = 0.0;
  bool lock = false;
  for (int r = r0; r < r1; ++r) {
    const int t = vt_tri[r];
    const double* q = tri_q + 10 * (size_t)t;
    for (int j = 0; j < 10; ++j) s[j] = da(s[j], q[j]);
    for (int k = 0; k < 3; ++k)                  // v's outgoing and incoming half-edges in t
      if (__ldg(tris + 3 * (size_t)t + k) == v) lock = lock || twin[3 * t + k] < 0 || twin[3 * t + (k + 2) % 3] < 0;
  }
  for (int j = 0; j < 10; ++j) Q[10 * (size_t)v + j] = s[j];
  const int deg = r1 - r0;
  if (deg > 0 && !lock) {
    const int t0 = vt_tri[r0];
    int k0 = 0;
    while (__ldg(tris + 3 * (size_t)t0 + k0) != v) ++k0;
    int h = 3 * t0 + k0, cnt = 1;
    for (;;) {
      const int tw = twin[h];
      if (tw < 0) break;
      const int nt = tw / 3;
      if (nt == t0) break;
      if (++cnt > deg) break;
      h = 3 * nt + (tw % 3 + 1) % 3;
    }
    lock = cnt != deg;
  }
  locked[v] = lock ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ one round: edges
__global__ void __launch_bounds__(kBlock) edge_kernel(const double* __restrict__ pos, const double* __restrict__ Qv,
                                                      const unsigned char* __restrict__ locked, const int* __restrict__ tris,
                                                      const int* __restrict__ adj_ptr, const int* __restrict__ adj,
                                                      const int* __restrict__ vt_ptr, const int* __restrict__ vt_tri,
                                                      const int* __restrict__ ea, const int* __restrict__ eb, int E,
                                                      double* __restrict__ xo, double* __restrict__ co, long long* __restrict__ key) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e >= E) return;
  const int a = ea[e], b = eb[e];
  const D3 pa = load3(pos, a), pb = load3(pos, b);
  double q[10];
  for (int j = 0; j < 10; ++j) q[j] = da(Qv[10 * (size_t)a + j], Qv[10 * (size_t)b + j]);
  // placement: the adjugate solve of M x = -g when M is well conditioned and x stays near the edge
  const double c00 = ds(dm(q[4], q[7]), dm(q[5], q[5])), c01 = ds(dm(q[2], q[5]), dm(q[1], q[7]));
  const double c02 = ds(dm(q[1], q[5]), dm(q[2], q[4])), c11 = ds(dm(q[0], q[7]), dm(q[2], q[2]));
  const double c12 = ds(dm(q[1], q[2]), dm(q[0], q[5])), c22 = ds(dm(q[0], q[4]), dm(q[1], q[1]));
  const double det = da(da(dm(q[0], c00), dm(q[1], c01)), dm(q[2], c02));
  const double fro = __dsqrt_rn(da(da(da(dm(q[0], q[0]), dm(q[4], q[4])), dm(q[7], q[7])),
                                   dm(2.0, da(da(dm(q[1], q[1]), dm(q[2], q[2])), dm(q[5], q[5])))));
  const double g0 = q[3], g1 = q[6], g2 = q[8];
  const D3 xs{__ddiv_rn(-da(da(dm(c00, g0), dm(c01, g1)), dm(c02, g2)), det), __ddiv_rn(-da(da(dm(c01, g0), dm(c11, g1)), dm(c12, g2)), det),
              __ddiv_rn(-da(da(dm(c02, g0), dm(c12, g1)), dm(c22, g2)), det)};
  const D3 d{ds(pb.x, pa.x), ds(pb.y, pa.y), ds(pb.z, pa.z)};
  const double ln = __dsqrt_rn(dot3(d, d));
  const bool in_box = xs.x >= ds(fmin(pa.x, pb.x), ln) && xs.x <= da(fmax(pa.x, pb.x), ln) && xs.y >= ds(fmin(pa.y, pb.y), ln) &&
                      xs.y <= da(fmax(pa.y, pb.y), ln) && xs.z >= ds(fmin(pa.z, pb.z), ln) && xs.z <= da(fmax(pa.z, pb.z), ln);
  D3 x;
  double cost;
  if (fabs(det) > dm(kDetEps, dm(dm(fro, fro), fro)) && in_box) {
    x = xs;
    cost = quadric_cost(q, xs);
  } else {
    const D3 mid{dm(da(pa.x, pb.x), 0.5), dm(da(pa.y, pb.y), 0.5), dm(da(pa.z, pb.z), 0.5)};
    const double ca = quadric_cost(q, pa), cb = quadric_cost(q, pb), cm = quadric_cost(q, mid);
    x = pa;
    cost = ca;
    if (cb < cost) { x = pb; cost = cb; }
    if (cm < cost) { x = mid; cost = cm; }
  }
  cost = cost > 0.0 ? cost : 0.0;
  xo[3 * (size_t)e] = x.x;
  xo[3 * (size_t)e + 1] = x.y;
  xo[3 * (size_t)e + 2] = x.z;
  co[e] = cost;

  // validity
  bool ok = !locked[a] && !locked[b];
  const int a0 = adj_ptr[a], a1 = adj_ptr[a + 1], b0 = adj_ptr[b], b1 = adj_ptr[b + 1];
  if (ok) {
    int common = 0;
    bool low = false;
    for (int i = a0, j = b0; i < a1 && j < b1;) {       // both rows ascending
      const int u = adj[i], w = adj[j];
      if (u < w) ++i;
      else if (w < u) ++j;
      else {
        ++common;
        low = low || adj_ptr[u + 1] - adj_ptr[u] < 4;
        ++i;
        ++j;
      }
    }
    ok = common == 2 && !low && (a1 - a0) + (b1 - b0) - 4 >= 3;
  }
  for (int side = 0; side < 2 && ok; ++side) {
    const int me = side ? b : a, other = side ? a : b;
    for (int r = vt_ptr[me], r1 = vt_ptr[me + 1]; r < r1 && ok; ++r) {
      const int t = vt_tri[r];
      const int i0 = __ldg(tris + 3 * (size_t)t), i1 = __ldg(tris + 3 * (size_t)t + 1), i2 = __ldg(tris + 3 * (size_t)t + 2);
      if (i0 == other || i1 == other || i2 == other) continue;
      const D3 p0 = load3(pos, i0), p1 = load3(pos, i1), p2 = load3(pos, i2);
      const D3 no = cross3(p0, p1, p2);
      const D3 nn = cross3(i0 == me ? x : p0, i1 == me ? x : p1, i2 == me ? x : p2);
      const bool zero_new = nn.x == 0.0 && nn.y == 0.0 && nn.z == 0.0;
      const bool nz_old = no.x != 0.0 || no.y != 0.0 || no.z != 0.0;
      if (zero_new || (nz_old && !(dot3(nn, no) > 0.0))) ok = false;
    }
  }
  const unsigned bits = __float_as_uint(__double2float_rn(cost));
  key[e] = ok ? (long long)(((unsigned long long)bits << 32) | (unsigned)e) : kKeyInf;
}

// ------------------------------------------------------------------------------------------------ one round: selection
__global__ void __launch_bounds__(kBlock) fill_key_kernel(long long* __restrict__ p, int n) {
  const int i = blockIdx.x * kBlock + threadIdx.x;
  if (i < n) p[i] = kKeyInf;
}

__global__ void __launch_bounds__(kBlock) vmin_kernel(const int* __restrict__ ea, const int* __restrict__ eb, int E,
                                                      const long long* __restrict__ key, long long* vmin) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e >= E) return;
  const long long k = key[e];
  if (k == kKeyInf) return;
  atomicMin((unsigned long long*)(vmin + ea[e]), (unsigned long long)k);     // keys are < 2^63: the same order as signed
  atomicMin((unsigned long long*)(vmin + eb[e]), (unsigned long long)k);
}

__global__ void __launch_bounds__(kBlock) rmin_kernel(const int* __restrict__ adj_ptr, const int* __restrict__ adj, int V,
                                                      const long long* __restrict__ vmin, long long* __restrict__ rmin) {
  const int v = blockIdx.x * kBlock + threadIdx.x;
  if (v >= V) return;
  long long m = vmin[v];
  for (int r = adj_ptr[v], r1 = adj_ptr[v + 1]; r < r1; ++r) m = min(m, vmin[adj[r]]);
  rmin[v] = m;
}

__global__ void __launch_bounds__(kBlock) selected_kernel(const int* __restrict__ ea, const int* __restrict__ eb, int E,
                                                          const long long* __restrict__ key, const long long* __restrict__ rmin,
                                                          unsigned char* __restrict__ selected) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e >= E) return;
  const long long k = key[e];
  selected[e] = k != kKeyInf && k == rmin[ea[e]] && k == rmin[eb[e]] ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------ one round: collapse
__global__ void __launch_bounds__(kBlock) identity_kernel(int* __restrict__ remap, int V) {
  const int v = blockIdx.x * kBlock + threadIdx.x;
  if (v < V) remap[v] = v;
}

__global__ void __launch_bounds__(kBlock) collapse_kernel(const int* __restrict__ ea, const int* __restrict__ eb, int E,
                                                          const long long* __restrict__ key, const unsigned char* __restrict__ selected,
                                                          const long long* __restrict__ thr, const double* __restrict__ x,
                                                          double* __restrict__ pos, double* __restrict__ Q, int* __restrict__ remap,
                                                          unsigned char* __restrict__ flag) {
  const int e = blockIdx.x * kBlock + threadIdx.x;
  if (e >= E) return;
  const bool f = selected[e] && key[e] <= *thr;
  flag[e] = f ? 1 : 0;
  if (!f) return;
  const int a = ea[e], b = eb[e];
  for (int j = 0; j < 3; ++j) pos[3 * (size_t)a + j] = x[3 * (size_t)e + j];
  for (int j = 0; j < 10; ++j) Q[10 * (size_t)a + j] = da(Q[10 * (size_t)a + j], Q[10 * (size_t)b + j]);
  remap[b] = a;
}

// ------------------------------------------------------------------------------------------------ ordered compaction
__device__ __forceinline__ bool kept(const int* __restrict__ tris, const int* __restrict__ remap, int t, int* o) {
  for (int k = 0; k < 3; ++k) o[k] = remap[__ldg(tris + 3 * (size_t)t + k)];
  return o[0] != o[1] && o[1] != o[2] && o[0] != o[2];
}

__global__ void __launch_bounds__(kBlock) rewrite_count_kernel(const int* __restrict__ tris, int T, const int* __restrict__ remap,
                                                               int* __restrict__ blk_cnt) {
  __shared__ int s_w[kBlock / 32];
  const int t = blockIdx.x * kBlock + threadIdx.x;
  int o[3];
  int total;
  block_scan<kBlock>(t < T && kept(tris, remap, t, o) ? 1 : 0, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) rewrite_emit_kernel(const int* __restrict__ tris, int T, const int* __restrict__ remap,
                                                              const long long* __restrict__ blk_off, int* __restrict__ out) {
  __shared__ int s_w[kBlock / 32];
  const int t = blockIdx.x * kBlock + threadIdx.x;
  int o[3];
  const bool f = t < T && kept(tris, remap, t, o);
  int total;
  const int r = block_scan<kBlock>(f ? 1 : 0, s_w, &total);
  if (!f) return;
  const long long p = blk_off[blockIdx.x] + r;
  for (int k = 0; k < 3; ++k) out[3 * p + k] = o[k];
}

__global__ void __launch_bounds__(kBlock) vflag_kernel(const int* __restrict__ tris, int T, unsigned char* vflag) {
  const int t = blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  for (int k = 0; k < 3; ++k) vflag[__ldg(tris + 3 * (size_t)t + k)] = 1;   // every writer stores 1
}

__global__ void __launch_bounds__(kBlock) vcount_kernel(const unsigned char* __restrict__ vflag, int V, int* __restrict__ blk_cnt) {
  __shared__ int s_w[kBlock / 32];
  const int v = blockIdx.x * kBlock + threadIdx.x;
  int total;
  block_scan<kBlock>(v < V && vflag[v] ? 1 : 0, s_w, &total);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kBlock) vemit_kernel(const double* __restrict__ pos, int V, const unsigned char* __restrict__ vflag,
                                                       const long long* __restrict__ blk_off, int* __restrict__ remap,
                                                       float* __restrict__ out) {
  __shared__ int s_w[kBlock / 32];
  const int v = blockIdx.x * kBlock + threadIdx.x;
  const bool f = v < V && vflag[v];
  int total;
  const int r = block_scan<kBlock>(f ? 1 : 0, s_w, &total);
  if (!f) return;
  const long long p = blk_off[blockIdx.x] + r;
  remap[v] = int(p);
  for (int j = 0; j < 3; ++j) out[3 * p + j] = __double2float_rn(pos[3 * (size_t)v + j]);
}

__global__ void __launch_bounds__(kBlock) tremap_kernel(const int* __restrict__ tris, int T, const int* __restrict__ remap,
                                                        int* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i < 3LL * T) out[i] = remap[__ldg(tris + i)];
}

inline unsigned nblocks(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

}  // namespace

extern "C" {

int nero_simplify_check_tris(const int* tris, int T, int V, long long* err, void* stream) {
  if (!tris || !err || T < 1 || V < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  err_init_kernel<<<1, 32, 0, s>>>(err);
  check_tris_kernel<<<nblocks(T), kBlock, 0, s>>>(tris, T, V, err);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_check_edges(const long long* hkey, const long long* hidx, long long n, int* twin, long long* err, void* stream) {
  if (!hkey || !hidx || !twin || !err || n < 3 || n > 0x7fffffffLL) return NERO_ERR_ARG;
  check_edges_kernel<<<nblocks(n), kBlock, 0, (cudaStream_t)stream>>>(hkey, hidx, n, twin, err);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_prepare(const float* verts, int V, const int* tris, int T, const int* vt_ptr, const int* vt_tri, const int* twin,
                          double* tri_q, double* pos, double* Q, unsigned char* locked, void* stream) {
  if (!verts || !tris || !vt_ptr || !vt_tri || !twin || !tri_q || !pos || !Q || !locked || V < 1 || T < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  tri_quadric_kernel<<<nblocks(T), kBlock, 0, s>>>(verts, tris, T, tri_q);
  vertex_kernel<<<nblocks(V), kBlock, 0, s>>>(verts, V, tris, vt_ptr, vt_tri, twin, tri_q, pos, Q, locked);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_edges(const double* pos, const double* Q, const unsigned char* locked, int V, const int* tris, int T,
                        const int* adj_ptr, const int* adj, const int* vt_ptr, const int* vt_tri, const int* ea, const int* eb, int E,
                        double* x, double* cost, long long* key, void* stream) {
  if (!pos || !Q || !locked || !tris || !adj_ptr || !adj || !vt_ptr || !vt_tri || !ea || !eb || !x || !cost || !key || V < 1 || T < 1 ||
      E < 1)
    return NERO_ERR_ARG;
  edge_kernel<<<nblocks(E), kBlock, 0, (cudaStream_t)stream>>>(pos, Q, locked, tris, adj_ptr, adj, vt_ptr, vt_tri, ea, eb, E, x, cost, key);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_select(const int* ea, const int* eb, int E, const long long* key, const int* adj_ptr, const int* adj, int V,
                         long long* vmin, long long* rmin, unsigned char* selected, void* stream) {
  if (!ea || !eb || !key || !adj_ptr || !adj || !vmin || !rmin || !selected || E < 1 || V < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  fill_key_kernel<<<nblocks(V), kBlock, 0, s>>>(vmin, V);
  vmin_kernel<<<nblocks(E), kBlock, 0, s>>>(ea, eb, E, key, vmin);
  rmin_kernel<<<nblocks(V), kBlock, 0, s>>>(adj_ptr, adj, V, vmin, rmin);
  selected_kernel<<<nblocks(E), kBlock, 0, s>>>(ea, eb, E, key, rmin, selected);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_collapse(const int* ea, const int* eb, int E, const long long* key, const unsigned char* selected, const long long* thr,
                           const double* x, int V, double* pos, double* Q, int* remap, unsigned char* flag, void* stream) {
  if (!ea || !eb || !key || !selected || !thr || !x || !pos || !Q || !remap || !flag || E < 1 || V < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  identity_kernel<<<nblocks(V), kBlock, 0, s>>>(remap, V);
  collapse_kernel<<<nblocks(E), kBlock, 0, s>>>(ea, eb, E, key, selected, thr, x, pos, Q, remap, flag);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_rewrite_count(const int* tris, int T, const int* remap, int* blk_cnt, long long* blk_off, long long* total,
                                void* stream) {
  if (!tris || !remap || !blk_cnt || !blk_off || !total || T < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  rewrite_count_kernel<<<nblocks(T), kBlock, 0, s>>>(tris, T, remap, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nblocks(T), s);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_rewrite_emit(const int* tris, int T, const int* remap, const long long* blk_off, long long nt, int* out, void* stream) {
  if (!tris || !remap || !blk_off || T < 1 || nt < 0 || nt > T || (nt > 0 && !out)) return NERO_ERR_ARG;
  if (nt > 0) rewrite_emit_kernel<<<nblocks(T), kBlock, 0, (cudaStream_t)stream>>>(tris, T, remap, blk_off, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_output_count(const int* tris, int T, int V, unsigned char* vflag, int* blk_cnt, long long* blk_off, long long* total,
                               void* stream) {
  if (!tris || !vflag || !blk_cnt || !blk_off || !total || T < 1 || V < 1) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  NERO_CUDA_TRY(cudaMemsetAsync(vflag, 0, (size_t)V, s));
  vflag_kernel<<<nblocks(T), kBlock, 0, s>>>(tris, T, vflag);
  vcount_kernel<<<nblocks(V), kBlock, 0, s>>>(vflag, V, blk_cnt);
  block_offsets<1>(blk_cnt, blk_off, total, nblocks(V), s);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_simplify_output_emit(const double* pos, int V, const int* tris, int T, const unsigned char* vflag, const long long* blk_off,
                              long long nv, int* remap, float* verts_out, int* tris_out, void* stream) {
  if (!pos || !tris || !vflag || !blk_off || !remap || !verts_out || !tris_out || V < 1 || T < 1 || nv < 1 || nv > V) return NERO_ERR_ARG;
  const cudaStream_t s = (cudaStream_t)stream;
  vemit_kernel<<<nblocks(V), kBlock, 0, s>>>(pos, V, vflag, blk_off, remap, verts_out);
  tremap_kernel<<<nblocks(3LL * T), kBlock, 0, s>>>(tris, T, remap, tris_out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
