// Screened Poisson reconstruction kernels: cell keys of the samples, the gather splats of the normal field and the density,
// the right-hand side G^T v, the operator A = L + ws S^T S, red-black Gauss-Seidel, residual, restriction and prolongation
// of the multigrid preconditioner, fp64 dot partials, the CG vector updates, interpolation and the trim test.
// include/nero_poisson.h states every operation; oracle/nero_oracle_poisson.py repeats them in numpy bit for bit.
//
// Every splat is a gather: a lattice point reads its support cells in a fixed order and each cell's samples in sorted order,
// so no floating-point atomics are needed and two runs give the same bits.
#include <cmath>

#include "common.cuh"
#include "../../include/nero_poisson.h"

namespace nero {
namespace {

constexpr int kBlock = NERO_POISSON_BLOCK;
constexpr int kWarps = kBlock / 32;
static_assert(kBlock == 256, "the pairwise tree of include/nero_align.h sums 256 values per block");

__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fs(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }

// h(d) = 1 - |d|
__device__ __forceinline__ float hat(float q, float c) { return fs(1.0f, fabsf(fs(q, c))); }

inline bool grid_ok(int N) { return N >= 3 && N <= NERO_POISSON_MAX_N; }
inline unsigned blocks_of(long long n) { return unsigned((n + kBlock - 1) / kBlock); }

__device__ __forceinline__ void node_of(long long idx, int N, int& i, int& j, int& k) {
  k = int(idx % N);
  const long long t = idx / N;
  j = int(t % N);
  i = int(t / N);
}

__global__ void keys_kernel(const double* __restrict__ p, long long n, double ox, double oy, double oz, double h, int N,
                            float* __restrict__ q, int* __restrict__ keys) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  const double o[3] = {ox, oy, oz};
  const float top = float(N - 1);
  int c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    float v = __double2float_rn(__ddiv_rn(__dsub_rn(p[3 * i + a], o[a]), h));
    v = fminf(fmaxf(v, 0.0f), top);
    q[3 * i + a] = v;
    c[a] = min(int(floorf(v)), N - 2);
  }
  keys[i] = (c[0] * (N - 1) + c[1]) * (N - 1) + c[2];
}

__global__ void cell_starts_kernel(const int* __restrict__ keys, long long n, int cells, int* __restrict__ start) {
  const long long c = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (c > cells) return;
  long long lo = 0, hi = n;                // first index with keys[i] >= c
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(keys + mid) < c) lo = mid + 1; else hi = mid;
  }
  start[c] = int(lo);
}

// the x, y or z edge lattice: one thread per edge
template <int A>
__global__ void edge_splat_kernel(const float* __restrict__ q, const float* __restrict__ nrm, const int* __restrict__ start, int N,
                                  float sigma, float* __restrict__ v) {
  const int D0 = A == 0 ? N - 1 : N, D1 = A == 1 ? N - 1 : N, D2 = A == 2 ? N - 1 : N;
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)D0 * D1 * D2) return;
  const int e2 = int(idx % D2);
  const long long t = idx / D2;
  const int e1 = int(t % D1), e0 = int(t / D1);
  const int e[3] = {e0, e1, e2};
  float c[3];
  int lo[3], hi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    if (a == A) {
      c[a] = float(e[a]) + 0.5f;
      lo[a] = max(e[a] - 1, 0);
      hi[a] = min(e[a] + 1, N - 2);
    } else {
      c[a] = float(e[a]);
      lo[a] = max(e[a] - 1, 0);
      hi[a] = min(e[a], N - 2);
    }
  }
  const int M = N - 1;
  float acc = 0.0f;
  for (int x = lo[0]; x <= hi[0]; ++x)
    for (int y = lo[1]; y <= hi[1]; ++y)
      for (int z = lo[2]; z <= hi[2]; ++z) {
        const int key = (x * M + y) * M + z;
        const int s0 = __ldg(start + key), s1 = __ldg(start + key + 1);
        for (int s = s0; s < s1; ++s) {
          const float wx = hat(__ldg(q + 3 * s), c[0]), wy = hat(__ldg(q + 3 * s + 1), c[1]), wz = hat(__ldg(q + 3 * s + 2), c[2]);
          if (wx <= 0.0f || wy <= 0.0f || wz <= 0.0f) continue;
          acc = fa(acc, fm(fm(fm(wx, wy), wz), __ldg(nrm + 3 * s + A)));
        }
      }
  v[idx] = __fdiv_rn(acc, sigma);
}

// the node gather of the 2 x 2 x 2 cells around node (i, j, k): acc0 of w and acc1 of w val (val = NULL: w w)
template <bool kSquare>
__device__ __forceinline__ void node_gather(const float* __restrict__ q, const float* __restrict__ val, const int* __restrict__ start,
                                            int N, int i, int j, int k, float& acc0, float& acc1) {
  const int M = N - 1;
  const float ci = float(i), cj = float(j), ck = float(k);
  acc0 = 0.0f;
  acc1 = 0.0f;
  for (int x = max(i - 1, 0); x <= min(i, N - 2); ++x)
    for (int y = max(j - 1, 0); y <= min(j, N - 2); ++y)
      for (int z = max(k - 1, 0); z <= min(k, N - 2); ++z) {
        const int key = (x * M + y) * M + z;
        const int s0 = __ldg(start + key), s1 = __ldg(start + key + 1);
        for (int s = s0; s < s1; ++s) {
          const float wx = hat(__ldg(q + 3 * s), ci), wy = hat(__ldg(q + 3 * s + 1), cj), wz = hat(__ldg(q + 3 * s + 2), ck);
          if (wx <= 0.0f || wy <= 0.0f || wz <= 0.0f) continue;
          const float w = fm(fm(wx, wy), wz);
          acc0 = fa(acc0, w);
          acc1 = fa(acc1, fm(w, kSquare ? w : __ldg(val + s)));
        }
      }
}

__global__ void node_splat_kernel(const float* __restrict__ q, const int* __restrict__ start, int N, float* __restrict__ density,
                                  float* __restrict__ diag) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)N * N * N) return;
  int i, j, k;
  node_of(idx, N, i, j, k);
  float a0, a1;
  node_gather<true>(q, nullptr, start, N, i, j, k, a0, a1);
  density[idx] = a0;
  diag[idx] = a1;
}

__global__ void rhs_kernel(const float* __restrict__ vx, const float* __restrict__ vy, const float* __restrict__ vz, int N,
                           float* __restrict__ b) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)N * N * N) return;
  int i, j, k;
  node_of(idx, N, i, j, k);
  const long long M = N - 1;
  float acc = 0.0f;
  // x edges: (N - 1) x N x N, edge (i, j, k) starts at node (i, j, k)
  if (i > 0) acc = fa(acc, vx[((i - 1) * (long long)N + j) * N + k]);
  if (i < N - 1) acc = fs(acc, vx[((long long)i * N + j) * N + k]);
  if (j > 0) acc = fa(acc, vy[((long long)i * M + (j - 1)) * N + k]);
  if (j < N - 1) acc = fs(acc, vy[((long long)i * M + j) * N + k]);
  if (k > 0) acc = fa(acc, vz[((long long)i * N + j) * M + (k - 1)]);
  if (k < N - 1) acc = fs(acc, vz[((long long)i * N + j) * M + k]);
  b[idx] = acc;
}

__device__ __forceinline__ float interp_at(const float* __restrict__ g, int N, float qx, float qy, float qz) {
  const int cx = min(max(int(floorf(qx)), 0), N - 2), cy = min(max(int(floorf(qy)), 0), N - 2), cz = min(max(int(floorf(qz)), 0), N - 2);
  float acc = 0.0f;
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 2; ++b)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float wx = hat(qx, float(cx + a)), wy = hat(qy, float(cy + b)), wz = hat(qz, float(cz + c));
        if (wx <= 0.0f || wy <= 0.0f || wz <= 0.0f) continue;
        acc = fa(acc, fm(fm(fm(wx, wy), wz), __ldg(g + ((long long)(cx + a) * N + (cy + b)) * N + (cz + c))));
      }
  return acc;
}

__global__ void interp_kernel(const float* __restrict__ g, int N, const float* __restrict__ q, long long m, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= m) return;
  out[i] = interp_at(g, N, q[3 * i], q[3 * i + 1], q[3 * i + 2]);
}

// m = sum of the neighbours' x in stencil order (from 0), deg = their number; lap = sum of (x_n - x_m) in the same order
struct Stencil { float m, lap; int deg; };

__device__ __forceinline__ Stencil stencil(const float* __restrict__ x, int N, long long idx, int i, int j, int k) {
  const float xn = x[idx];
  const long long sx = (long long)N * N, sy = N;
  Stencil s{0.0f, 0.0f, 0};
  auto add = [&](long long o) {
    const float xm = x[idx + o];
    s.m = fa(s.m, xm);
    s.lap = fa(s.lap, fs(xn, xm));
    ++s.deg;
  };
  if (i > 0) add(-sx);
  if (i < N - 1) add(sx);
  if (j > 0) add(-sy);
  if (j < N - 1) add(sy);
  if (k > 0) add(-1);
  if (k < N - 1) add(1);
  return s;
}

__global__ void matvec_kernel(const float* __restrict__ x, int N, const float* __restrict__ q, const int* __restrict__ start, float ws,
                              const float* __restrict__ sx, float* __restrict__ y) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)N * N * N) return;
  int i, j, k;
  node_of(idx, N, i, j, k);
  float a0, t;
  node_gather<false>(q, sx, start, N, i, j, k, a0, t);
  y[idx] = fa(stencil(x, N, idx, i, j, k).lap, fm(ws, t));
}

__global__ void smooth_kernel(float* x, const float* __restrict__ b, const float* __restrict__ d, int N, float s, int colour) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)N * N * N) return;
  int i, j, k;
  node_of(idx, N, i, j, k);
  if (((i + j + k) & 1) != colour) return;
  const Stencil st = stencil(x, N, idx, i, j, k);   // reads only the other colour
  x[idx] = __fdiv_rn(fa(b[idx], fm(s, st.m)), fa(fm(s, float(st.deg)), d[idx]));
}

__global__ void residual_kernel(const float* __restrict__ x, const float* __restrict__ b, const float* __restrict__ d, int N, float s,
                                float* __restrict__ r) {
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)N * N * N) return;
  int i, j, k;
  node_of(idx, N, i, j, k);
  r[idx] = fs(b[idx], fa(fm(s, stencil(x, N, idx, i, j, k).lap), fm(d[idx], x[idx])));
}

__global__ void restrict_kernel(const float* __restrict__ f, int Nf, float* __restrict__ c) {
  const int Nc = (Nf - 1) / 2 + 1;
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)Nc * Nc * Nc) return;
  int I, J, K;
  node_of(idx, Nc, I, J, K);
  float acc = 0.0f;
  for (int dx = -1; dx <= 1; ++dx) {
    const int x = 2 * I + dx;
    if (x < 0 || x >= Nf) continue;
    const float wx = dx ? 0.5f : 1.0f;
    for (int dy = -1; dy <= 1; ++dy) {
      const int y = 2 * J + dy;
      if (y < 0 || y >= Nf) continue;
      const float wy = dy ? 0.5f : 1.0f;
      for (int dz = -1; dz <= 1; ++dz) {
        const int z = 2 * K + dz;
        if (z < 0 || z >= Nf) continue;
        const float wz = dz ? 0.5f : 1.0f;
        acc = fa(acc, fm(fm(fm(wx, wy), wz), f[((long long)x * Nf + y) * Nf + z]));
      }
    }
  }
  c[idx] = acc;
}

__global__ void prolong_kernel(const float* __restrict__ c, int Nc, float* __restrict__ f) {
  const int Nf = 2 * (Nc - 1) + 1;
  const long long idx = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (idx >= (long long)Nf * Nf * Nf) return;
  int i, j, k;
  node_of(idx, Nf, i, j, k);
  const int nx = 1 + (i & 1), ny = 1 + (j & 1), nz = 1 + (k & 1);
  const float wx = (i & 1) ? 0.5f : 1.0f, wy = (j & 1) ? 0.5f : 1.0f, wz = (k & 1) ? 0.5f : 1.0f;
  const float w = fm(fm(wx, wy), wz);
  float acc = 0.0f;
  for (int a = 0; a < nx; ++a)
    for (int b = 0; b < ny; ++b)
      for (int e = 0; e < nz; ++e)
        acc = fa(acc, fm(w, c[((long long)(i / 2 + a) * Nc + (j / 2 + b)) * Nc + (k / 2 + e)]));
  f[idx] = fa(f[idx], acc);
}

__device__ __forceinline__ double warp_tree(double v) {
#pragma unroll
  for (int h = 1; h < 32; h <<= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, h));
  return v;
}

__global__ void __launch_bounds__(kBlock) dot_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n,
                                                     double* __restrict__ partial) {
  __shared__ double s[kWarps];
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  double v = 0.0;
  if (i < n) v = b ? __dmul_rn((double)a[i], (double)b[i]) : (double)a[i];   // exact: two fp32 significands fit fp64
  v = warp_tree(v);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0)
    partial[blockIdx.x] = __dadd_rn(__dadd_rn(__dadd_rn(s[0], s[1]), __dadd_rn(s[2], s[3])), __dadd_rn(__dadd_rn(s[4], s[5]), __dadd_rn(s[6], s[7])));
}

__global__ void update_kernel(float* __restrict__ x, float* __restrict__ r, const float* __restrict__ p, const float* __restrict__ ap,
                              float alpha, long long n) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  x[i] = fa(x[i], fm(alpha, p[i]));
  r[i] = fs(r[i], fm(alpha, ap[i]));
}

__global__ void direction_kernel(float* __restrict__ p, const float* __restrict__ z, float beta, long long n) {
  const long long i = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (i >= n) return;
  p[i] = fa(z[i], fm(beta, p[i]));
}

__global__ void trim_kernel(const float* __restrict__ dens, const int* __restrict__ tris, int T, float thr, unsigned char* __restrict__ keep) {
  const long long t = (long long)blockIdx.x * kBlock + threadIdx.x;
  if (t >= T) return;
  keep[t] = (dens[tris[3 * t]] >= thr && dens[tris[3 * t + 1]] >= thr && dens[tris[3 * t + 2]] >= thr) ? 1 : 0;
}

inline long long nodes(int N) { return (long long)N * N * N; }

}  // namespace

extern "C" int nero_poisson_keys(const double* points, long long n, double ox, double oy, double oz, double h, int N, float* q, int* keys,
                                 void* stream) {
  if (n < 1 || !grid_ok(N) || !(h > 0.0) || !points || !q || !keys) return NERO_ERR_ARG;
  keys_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(points, n, ox, oy, oz, h, N, q, keys);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_cell_starts(const int* keys, long long n, int cells, int* start, void* stream) {
  if (n < 1 || n > 0x7fffffffLL || cells < 1 || !keys || !start) return NERO_ERR_ARG;
  cell_starts_kernel<<<blocks_of((long long)cells + 1), kBlock, 0, (cudaStream_t)stream>>>(keys, n, cells, start);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_edge_splat(const float* q, const float* nrm, long long n, const int* start, int N, float sigma, float* vx,
                                       float* vy, float* vz, void* stream) {
  if (n < 1 || !grid_ok(N) || !(sigma > 0.0f) || !q || !nrm || !start || !vx || !vy || !vz) return NERO_ERR_ARG;
  const long long e = (long long)(N - 1) * N * N;
  edge_splat_kernel<0><<<blocks_of(e), kBlock, 0, (cudaStream_t)stream>>>(q, nrm, start, N, sigma, vx);
  edge_splat_kernel<1><<<blocks_of(e), kBlock, 0, (cudaStream_t)stream>>>(q, nrm, start, N, sigma, vy);
  edge_splat_kernel<2><<<blocks_of(e), kBlock, 0, (cudaStream_t)stream>>>(q, nrm, start, N, sigma, vz);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_node_splat(const float* q, long long n, const int* start, int N, float* density, float* diag, void* stream) {
  if (n < 1 || !grid_ok(N) || !q || !start || !density || !diag) return NERO_ERR_ARG;
  node_splat_kernel<<<blocks_of(nodes(N)), kBlock, 0, (cudaStream_t)stream>>>(q, start, N, density, diag);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_rhs(const float* vx, const float* vy, const float* vz, int N, float* b, void* stream) {
  if (!grid_ok(N) || !vx || !vy || !vz || !b) return NERO_ERR_ARG;
  rhs_kernel<<<blocks_of(nodes(N)), kBlock, 0, (cudaStream_t)stream>>>(vx, vy, vz, N, b);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_interp(const float* grid, int N, const float* q, long long m, float* out, void* stream) {
  if (m < 1 || !grid_ok(N) || !grid || !q || !out) return NERO_ERR_ARG;
  interp_kernel<<<blocks_of(m), kBlock, 0, (cudaStream_t)stream>>>(grid, N, q, m, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_matvec(const float* x, int N, const float* q, long long n, const int* start, float ws, float* sx, float* y,
                                   void* stream) {
  if (n < 1 || !grid_ok(N) || !x || !q || !start || !sx || !y) return NERO_ERR_ARG;
  interp_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(x, N, q, n, sx);
  matvec_kernel<<<blocks_of(nodes(N)), kBlock, 0, (cudaStream_t)stream>>>(x, N, q, start, ws, sx, y);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_smooth(float* x, const float* b, const float* d, int N, float s, int colour, void* stream) {
  if (!grid_ok(N) || (colour != 0 && colour != 1) || !(s > 0.0f) || !x || !b || !d) return NERO_ERR_ARG;
  smooth_kernel<<<blocks_of(nodes(N)), kBlock, 0, (cudaStream_t)stream>>>(x, b, d, N, s, colour);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_residual(const float* x, const float* b, const float* d, int N, float s, float* r, void* stream) {
  if (!grid_ok(N) || !(s > 0.0f) || !x || !b || !d || !r) return NERO_ERR_ARG;
  residual_kernel<<<blocks_of(nodes(N)), kBlock, 0, (cudaStream_t)stream>>>(x, b, d, N, s, r);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_restrict(const float* fine, int Nf, float* coarse, void* stream) {
  if (!grid_ok(Nf) || !(Nf & 1) || !fine || !coarse) return NERO_ERR_ARG;
  restrict_kernel<<<blocks_of(nodes((Nf - 1) / 2 + 1)), kBlock, 0, (cudaStream_t)stream>>>(fine, Nf, coarse);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_prolong(const float* coarse, int Nc, float* fine, void* stream) {
  if (Nc < 2 || 2 * (Nc - 1) + 1 > NERO_POISSON_MAX_N || !coarse || !fine) return NERO_ERR_ARG;
  prolong_kernel<<<blocks_of(nodes(2 * (Nc - 1) + 1)), kBlock, 0, (cudaStream_t)stream>>>(coarse, Nc, fine);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_dot(const float* a, const float* b, long long n, double* partial, void* stream) {
  if (n < 1 || !a || !partial) return NERO_ERR_ARG;
  dot_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(a, b, n, partial);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_update(float* x, float* r, const float* p, const float* ap, float alpha, long long n, void* stream) {
  if (n < 1 || !x || !r || !p || !ap) return NERO_ERR_ARG;
  update_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(x, r, p, ap, alpha, n);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_direction(float* p, const float* z, float beta, long long n, void* stream) {
  if (n < 1 || !p || !z) return NERO_ERR_ARG;
  direction_kernel<<<blocks_of(n), kBlock, 0, (cudaStream_t)stream>>>(p, z, beta, n);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_poisson_trim(const float* dens, int V, const int* tris, int T, float threshold, unsigned char* keep, void* stream) {
  if (T < 1 || V < 1 || !dens || !tris || !keep) return NERO_ERR_ARG;
  trim_kernel<<<blocks_of(T), kBlock, 0, (cudaStream_t)stream>>>(dens, tris, T, threshold, keep);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
