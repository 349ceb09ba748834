// Environment-light export: the outer light of either stage sampled on an equirectangular map.  The protocol is stated once
// in nero_b200/envmap.py, the map convention in include/nero_envmap.h.
//
//   rows     one thread per (texel, sub-sample) row: the direction in fp64 (no contraction, so it is the numpy expression
//            of nero_oracle_relight.env_dir), rotated by the optional frame and rounded to fp32 once; then IDE(d, kappa_inv)
//            [+ IDE of the sphere point] in the reference's fp32 arithmetic, staged per warp and stored as whole rows
//            (tile_io.cuh), padding columns zeroed.  The outer-light MLP itself is the existing fused chain.
//   resolve  one thread per texel: the cos(elevation)-weighted mean of its sub-samples, summed in fp64 in sub-sample order.
//
// Nothing is accumulated across threads, so the map is bit-identical from run to run and for any split into launches.
#include "common.cuh"
#include "math_enc.cuh"
#include "math_shade.cuh"
#include "math_mc.cuh"
#include "tile_io.cuh"
#include "../../include/nero_envmap.h"

namespace nero {

__constant__ IdeTable c_ide_env;

int set_ide_table_env(const float* mat17x36_host) {
  IdeTable t;
  int i = 0;
  for (int e = 0; e < 5; ++e) {
    const int l = 1 << e;
    for (int m = 0; m <= l; ++m) { t.m[i] = m; t.l[i] = l; ++i; }
  }
  for (int k = 0; k < 17; ++k)
    for (int j = 0; j < 36; ++j) { t.mat[k][j] = double(mat17x36_host[k * 36 + j]); t.matf[k][j] = mat17x36_host[k * 36 + j]; }
  NERO_CUDA_TRY(cudaMemcpyToSymbol(c_ide_env, &t, sizeof(IdeTable)));
  return NERO_OK;
}

namespace {

constexpr double kPiD = 3.141592653589793;     // numpy.pi
constexpr int kEnvBlock = 128;
constexpr int kEnvTileLd = 73;
constexpr int kMaxSsaa = 16;

// elevation of sub-sample row b of map row j (counted from the bottom): v = (j + (b + 1/2) / s) / H, el = (v - 1/2) pi
__device__ __forceinline__ double env_elevation(long long j, int b, int s, int H) {
  const double v = __ddiv_rn(__dadd_rn(double(j), __ddiv_rn(__dadd_rn(double(b), 0.5), double(s))), double(H));
  return __dmul_rn(__dadd_rn(v, -0.5), kPiD);
}

__device__ __forceinline__ void env_direction(long long r, int W, int H, int s, const double* __restrict__ F, float* d) {
  const int s2 = s * s;
  const long long t = r / s2;
  const int k = int(r - t * s2), a = k % s, b = k / s;
  const long long y = t / W;
  const int x = int(t - y * W);
  const double u = __ddiv_rn(__dadd_rn(double(x), __ddiv_rn(__dadd_rn(double(a), 0.5), double(s))), double(W));
  const double phi = __dmul_rn(__dmul_rn(__dadd_rn(0.5, -u), 2.0), kPiD);
  const double el = env_elevation(H - 1 - y, b, s, H);
  const double ce = cos(el);
  const double e[3] = {__dmul_rn(ce, cos(phi)), __dmul_rn(ce, sin(phi)), sin(el)};
  if (F == nullptr) {
    for (int c = 0; c < 3; ++c) d[c] = float(e[c]);
    return;
  }
  for (int c = 0; c < 3; ++c)
    d[c] = float(__dadd_rn(__dadd_rn(__dmul_rn(F[3 * c], e[0]), __dmul_rn(F[3 * c + 1], e[1])), __dmul_rn(F[3 * c + 2], e[2])));
}

__global__ void __launch_bounds__(kEnvBlock) env_rows_kernel(long long row0, long long n, int W, int H, int s,
                                                             const double* __restrict__ F, float kinv, int sphere, float3 center,
                                                             float* __restrict__ A, int lda, float* __restrict__ dirs) {
  __shared__ float s_tile[kEnvBlock / 32][32][kEnvTileLd];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const long long i = (long long)blockIdx.x * kEnvBlock + threadIdx.x;
  const long long w0 = i - lane;                              // first row of the warp
  if (w0 >= n) return;                                        // whole warps only: the stores below are warp-collective
  const int rows = int(n - w0 < 32 ? n - w0 : 32);
  float (*tile)[kEnvTileLd] = s_tile[wid];
  const bool valid = i < n;
  float d[3] = {0.f, 0.f, 1.f};
  if (valid) {
    env_direction(row0 + i, W, H, s, F, d);
    if (dirs) for (int c = 0; c < 3; ++c) dirs[i * 3 + c] = d[c];
    ide_forward(c_ide_env, d, kinv, tile[lane]);
  }
  float* a = A + size_t(w0) * lda;
  warp_rows_store4<kEnvTileLd, 18>(tile, a, lda, rows, lane);
  int k = 72;
  if (sphere) {
    if (valid) {
      const float c[3] = {center.x, center.y, center.z};
      float sp[3];
      if (sphere == 1) {
        sphere_dir_fwd(c, d, sp);
        ide_forward(c_ide_env, sp, kinv, tile[lane]);
      } else {
        float pu[3];
        mc_sphere_point(c, d, sp, pu);
        ide_forward(c_ide_env, sp, 0.f, tile[lane]);
      }
    }
    warp_rows_store4<kEnvTileLd, 18>(tile, a + 72, lda, rows, lane);
    k = 144;
  }
  for (int r = 0; r < rows; ++r)
    for (int c = k + lane; c < lda; c += 32) a[size_t(r) * lda + c] = 0.f;
}

__global__ void __launch_bounds__(kEnvBlock) env_resolve_kernel(const float* __restrict__ rad, int ld, long long tex0, long long ntex,
                                                                int W, int H, int s, float* __restrict__ env) {
  const long long i = (long long)blockIdx.x * kEnvBlock + threadIdx.x;
  if (i >= ntex) return;
  const long long t = tex0 + i, y = t / W;
  const int s2 = s * s;
  double sw = 0.0, acc[3] = {0.0, 0.0, 0.0};
  for (int k = 0; k < s2; ++k) {
    const double w = cos(env_elevation(H - 1 - y, k / s, s, H));
    const float* L = rad + size_t(i * s2 + k) * ld;
    sw = __dadd_rn(sw, w);
    for (int c = 0; c < 3; ++c) acc[c] = __dadd_rn(acc[c], __dmul_rn(w, double(L[c])));
  }
  for (int c = 0; c < 3; ++c) env[t * 3 + c] = float(__ddiv_rn(acc[c], sw));
}

bool env_grid(int W, int H, int s, long long& n_rows) {
  if (W < 1 || H < 1 || s < 1 || s > kMaxSsaa) return false;
  n_rows = (long long)W * H * s * s;
  return true;
}

}  // namespace

extern "C" {

int nero_env_rows(long long row0, long long n, int width, int height, int ssaa, const double* frame, float kappa_inv, int sphere,
                  float cx, float cy, float cz, float* A, int lda, float* dirs, void* stream) {
  long long total;
  if (!env_grid(width, height, ssaa, total) || row0 < 0 || n < 0 || row0 + n > total || !A) return NERO_ERR_ARG;
  if (sphere < 0 || sphere > 2 || lda % 4 != 0 || lda < (sphere ? 144 : 72)) return NERO_ERR_ARG;
  if (n == 0) return NERO_OK;
  const long long nblk = (n + kEnvBlock - 1) / kEnvBlock;
  if (nblk > 0x7fffffffLL) return NERO_ERR_ARG;
  env_rows_kernel<<<unsigned(nblk), kEnvBlock, 0, (cudaStream_t)stream>>>(row0, n, width, height, ssaa, frame, kappa_inv, sphere,
                                                                          make_float3(cx, cy, cz), A, lda, dirs);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

int nero_env_resolve(const float* rad, int ld, long long texel0, long long ntex, int width, int height, int ssaa, float* env,
                     void* stream) {
  long long total;
  if (!env_grid(width, height, ssaa, total) || !rad || !env || ld < 3 || texel0 < 0 || ntex < 0 ||
      texel0 + ntex > (long long)width * height)
    return NERO_ERR_ARG;
  if (ntex == 0) return NERO_OK;
  env_resolve_kernel<<<unsigned((ntex + kEnvBlock - 1) / kEnvBlock), kEnvBlock, 0, (cudaStream_t)stream>>>(rad, ld, texel0, ntex, width,
                                                                                                        height, ssaa, env);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // extern "C"

}  // namespace nero
