// Weight preparation (once per optimizer step) and weight-gradient finishing.
//
// nero_prep_weight: folds torch weight_norm (W = g * v / ||v||_row, network/field.py:118-119, 324-331) and
// writes, for rows [row0, row0+nrows) of the layer,
//   * img_f : the forward tensor-core operand image  (tile rows = output features, K = input layout columns)
//   * img_t : the transposed image for input-gradient GEMMs (tile rows = input layout columns, K = output features)
// both as split-bf16 (hi plane, lo plane) per 32-wide K chunk in the K-major SWIZZLE_64B shared-memory layout,
// so the GEMM kernels fetch a chunk (or two adjacent ones) with one bulk copy.  32-wide chunks let the fused chain stream
// its weights in 16 KB stages of 128 rows (k_gemm_chain.cu).  `kmap` places reference input column k at column
// kmap[k] of the (padded / re-ordered) activation layout the kernels actually use; `in_scale` folds constant
// input scalings.  Images must be zero-initialised once (padding stays zero).
//
// nero_wgrad_finish: reduces the split-K partials of k_gemm_wgrad.cu, maps layout columns back through kmap and
// accumulates into .grad of (weight_g, weight_v, bias) via the weight-norm chain rule, or (weight, bias).
#include "common.cuh"

namespace nero {

__device__ __forceinline__ float block_sum(float v, float* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int w = tid >> 5, l = tid & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float t = 0.0f;
  for (int i = 0; i < ((blockDim.x * blockDim.y) >> 5); ++i) t += sh[i];
  return t;
}

__device__ __forceinline__ void img_store(uint8_t* img, int rows_pad, int r, int kcol, float w) {
  const int c = kcol >> 5, kk = kcol & 31;
  uint8_t* base = img + size_t(c) * 2 * rows_pad * 64;
  __nv_bfloat16 hi, lo;
  split_bf16(w, hi, lo);
  const uint32_t off = sw64_offset(r, kk);
  *reinterpret_cast<__nv_bfloat16*>(base + off) = hi;
  *reinterpret_cast<__nv_bfloat16*>(base + size_t(rows_pad) * 64 + off) = lo;
}

__device__ __forceinline__ void prep_weight_row(int r, const float* __restrict__ v, const float* __restrict__ g, int K, int row0,
                                   const int* __restrict__ kmap, float in_scale, uint8_t* img_f, int rows_pad_f,
                                   uint8_t* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff, int ld_weff) {
  __shared__ float sh[32];
  const int n = row0 + r;         // layer row
  const float* vr = v + size_t(n) * K;
  float scale = 1.0f;
  if (g) {
    float ss = 0.0f;
    for (int k = threadIdx.x; k < K; k += blockDim.x) ss += vr[k] * vr[k];
    ss = block_sum(ss, sh);
    scale = g[n] / sqrtf(ss);
  }
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float w = vr[k] * scale;            // same op order as torch._weight_norm: v * (g / ||v||)
    if (w_eff) w_eff[size_t(n) * ld_weff + k] = w;
    const int kc = kmap ? kmap[k] : k;
    const float ws = w * in_scale;
    if (img_f) img_store(img_f, rows_pad_f, r, kc, ws);
    if (img_t && kc >= t_c0 && kc < t_c0 + t_ncols) img_store(img_t, rows_pad_t, kc - t_c0, r, ws);
  }
}

__global__ void prep_weight_kernel(const float* __restrict__ v, const float* __restrict__ g, int K, int row0,
                                   const int* __restrict__ kmap, float in_scale, uint8_t* img_f, int rows_pad_f,
                                   uint8_t* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff, int ld_weff) {
  prep_weight_row(blockIdx.x, v, g, K, row0, kmap, in_scale, img_f, rows_pad_f, img_t, rows_pad_t, t_c0, t_ncols, w_eff, ld_weff);
}
// all layers of a network in one launch: blockIdx.y selects the job
__global__ void prep_weight_batch_kernel(const nero_prep_job* __restrict__ jobs) {
  const nero_prep_job j = jobs[blockIdx.y];
  if (int(blockIdx.x) >= j.nrows) return;
  prep_weight_row(blockIdx.x, j.v, j.g, j.K, j.row0, j.kmap, j.in_scale, static_cast<uint8_t*>(j.img_f), j.rows_pad_f,
                  static_cast<uint8_t*>(j.img_t), j.rows_pad_t, j.t_c0, j.t_ncols, j.w_eff, j.ld_weff);
}
extern "C" int nero_prep_weight_batch(const void* jobs_dev, int n_jobs, int max_rows, void* stream) {
  if (n_jobs <= 0 || max_rows <= 0) return NERO_OK;
  if (!jobs_dev) return NERO_ERR_ARG;
  prep_weight_batch_kernel<<<dim3(max_rows, n_jobs), 128, 0, (cudaStream_t)stream>>>(static_cast<const nero_prep_job*>(jobs_dev));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_prep_weight(const float* v, const float* g, int K, int row0, int nrows, const int* kmap, float in_scale,
                                void* img_f, int rows_pad_f, void* img_t, int rows_pad_t, int t_c0, int t_ncols, float* w_eff,
                                int ld_weff, void* stream) {
  if (nrows <= 0) return NERO_OK;
  prep_weight_kernel<<<nrows, 128, 0, (cudaStream_t)stream>>>(v, g, K, row0, kmap, in_scale, static_cast<uint8_t*>(img_f), rows_pad_f,
                                                              static_cast<uint8_t*>(img_t), rows_pad_t, t_c0, t_ncols, w_eff, ld_weff);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

// one block per layer row n = row0 + blockIdx.x; blockDim = (kcols, ny): the P split-K partials are summed by ny thread
// groups in parallel (the per-row reads are latency bound), then reduced through shared memory ([ny][K] floats).
__device__ __forceinline__ void wgrad_finish_row(int r, const float* __restrict__ partial, int P, int rows_partial, int ld_partial,
                                    const float* __restrict__ bias_partial, int K, int row0,
                                    const int* __restrict__ kmap, float in_scale, const float* __restrict__ v,
                                    const float* __restrict__ g, float* grad_w, float* grad_g, float* grad_b,
                                    const float* __restrict__ extra_row, float extra_scale) {
  __shared__ float sh[32];
  extern __shared__ float s_dw[];  // [ny][K] partial sums, then [K] in slot 0
  const int ny = blockDim.y;
  const int n = row0 + r;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthreads = blockDim.x * blockDim.y;
  const size_t pstride = size_t(rows_partial) * ld_partial;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const int kc = kmap ? kmap[k] : k;
    const float* pp = partial + size_t(r) * ld_partial + kc;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int pidx = threadIdx.y;
    for (; pidx + 3 * ny < P; pidx += 4 * ny) {
      a0 += pp[size_t(pidx) * pstride]; a1 += pp[size_t(pidx + ny) * pstride];
      a2 += pp[size_t(pidx + 2 * ny) * pstride]; a3 += pp[size_t(pidx + 3 * ny) * pstride];
    }
    for (; pidx < P; pidx += ny) a0 += pp[size_t(pidx) * pstride];
    s_dw[threadIdx.y * K + k] = (a0 + a1) + (a2 + a3);
  }
  __syncthreads();
  for (int k = tid; k < K; k += nthreads) {
    const int kc = kmap ? kmap[k] : k;
    float acc = s_dw[k];
    for (int y = 1; y < ny; ++y) acc += s_dw[y * K + k];
    acc *= in_scale;
    if (extra_row && r == 0) acc += extra_scale * extra_row[kc];
    s_dw[k] = acc;   // slot 0 (each k is read and written by the same thread)
  }
  __syncthreads();
  if (grad_b && bias_partial && tid == 0) {
    float b = 0.0f;
    for (int pidx = 0; pidx < P; ++pidx) b += bias_partial[size_t(pidx) * rows_partial + r];
    grad_b[n] += b;
  }
  if (g) {
    const float* vr = v + size_t(n) * K;
    float ss = 0.0f, dot = 0.0f;
    for (int k = tid; k < K; k += nthreads) { ss += vr[k] * vr[k]; dot += s_dw[k] * vr[k]; }
    ss = block_sum(ss, sh);
    dot = block_sum(dot, sh);
    const float inv_norm = rsqrtf(ss);
    const float dg = dot * inv_norm;                 // dL/dg = dW . v_hat
    const float c = g[n] * inv_norm;
    for (int k = tid; k < K; k += nthreads)
      grad_w[size_t(n) * K + k] += c * (s_dw[k] - dg * vr[k] * inv_norm);
    if (tid == 0) grad_g[n] += dg;
  } else {
    for (int k = tid; k < K; k += nthreads) grad_w[size_t(n) * K + k] += s_dw[k];
  }
}

__global__ void wgrad_finish_kernel(const float* __restrict__ partial, int P, int rows_partial, int ld_partial,
                                    const float* __restrict__ bias_partial, int K, int row0,
                                    const int* __restrict__ kmap, float in_scale, const float* __restrict__ v,
                                    const float* __restrict__ g, float* grad_w, float* grad_g, float* grad_b,
                                    const float* __restrict__ extra_row, float extra_scale) {
  wgrad_finish_row(blockIdx.x, partial, P, rows_partial, ld_partial, bias_partial, K, row0, kmap, in_scale, v, g, grad_w, grad_g, grad_b,
                   extra_row, extra_scale);
}
// many layers in one launch: blockIdx.y selects the job (jobs must not share destination rows)
__global__ void wgrad_finish_batch_kernel(const nero_finish_job* __restrict__ jobs) {
  const nero_finish_job j = jobs[blockIdx.y];
  if (int(blockIdx.x) >= j.nrows) return;
  wgrad_finish_row(blockIdx.x, j.partial, j.P, j.rows_partial, j.ld_partial, j.bias_partial, j.K, j.row0, j.kmap, j.in_scale, j.v, j.g,
                   j.grad_w, j.grad_g, j.grad_b, j.extra_row, j.extra_scale);
}
extern "C" int nero_wgrad_finish_batch(const void* jobs_dev, int n_jobs, int max_rows, int max_k, void* stream) {
  if (n_jobs <= 0 || max_rows <= 0) return NERO_OK;
  if (!jobs_dev || max_k <= 0 || max_k > 1024) return NERO_ERR_ARG;
  // (256, 4) blocks: four groups of partial slices are summed in parallel (the per-row reads are latency bound)
  wgrad_finish_batch_kernel<<<dim3(max_rows, n_jobs), dim3(256, 4), 4 * max_k * sizeof(float), (cudaStream_t)stream>>>(
      static_cast<const nero_finish_job*>(jobs_dev));
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

extern "C" int nero_wgrad_finish(const float* partial, int P, int rows_partial, int ld_partial, const float* bias_partial, int K,
                                 int row0, int nrows, const int* kmap, float in_scale, const float* v, const float* g, float* grad_w,
                                 float* grad_g, float* grad_b, const float* extra_row, float extra_scale, void* stream) {
  if (nrows <= 0) return NERO_OK;
  int bx = 32;
  while (bx < K && bx < 256) bx <<= 1;
  wgrad_finish_kernel<<<nrows, dim3(bx, 4), 4 * K * sizeof(float), (cudaStream_t)stream>>>(partial, P, rows_partial, ld_partial, bias_partial,
                                                                                          K, row0, kmap, in_scale, v, g, grad_w, grad_g,
                                                                                          grad_b, extra_row, extra_scale);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

// column sums: out[j] (+)= sum_m w[m] * X[m, j]   (w may be null = ones).  Used for the sdf row of lin8:
// dW8[0,:] = sum_m dsdf[m] * h8[m,:] + sum_m ubar8[m,:]   and for its bias.
// Block row y writes its partial sums to colsum_partials[y]; a second kernel adds them up in a fixed order, so the result
// is the same every run (no floating-point atomics).
constexpr int kColsumMaxCols = 1024;
__device__ float colsum_partials[kNumSMs * kColsumMaxCols];

__global__ void colsum_kernel(const float* __restrict__ X, int ldx, int ncol, const float* __restrict__ w, int ldw,
                              const int* __restrict__ m_ptr, int m_cap) {
  int M = m_ptr ? *m_ptr : m_cap;
  if (M > m_cap) M = m_cap;
  // 256 threads = 8 row lanes x 32 column lanes of 4 adjacent columns each (one float4 per row and thread)
  const int lane = threadIdx.x & 31, rlane = threadIdx.x >> 5;
  const int col = (blockIdx.x * 32 + lane) * 4;
  const int rows_per_block = (M + gridDim.y - 1) / gridDim.y;
  const int r0 = blockIdx.y * rows_per_block, r1 = min(M, r0 + rows_per_block);
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  const bool vec = (ldx & 3) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 && col + 3 < ncol;
  if (vec) {
    int r = r0 + rlane;
    for (; r + 24 < r1; r += 32) {          // four independent row loads in flight
      float4 x[4]; float s[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        x[u] = *reinterpret_cast<const float4*>(X + size_t(r + 8 * u) * ldx + col);
        s[u] = w ? w[size_t(r + 8 * u) * ldw] : 1.0f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) { acc[0] += s[u] * x[u].x; acc[1] += s[u] * x[u].y; acc[2] += s[u] * x[u].z; acc[3] += s[u] * x[u].w; }
    }
    for (; r < r1; r += 8) {
      const float4 x = *reinterpret_cast<const float4*>(X + size_t(r) * ldx + col);
      const float s = w ? w[size_t(r) * ldw] : 1.0f;
      acc[0] += s * x.x; acc[1] += s * x.y; acc[2] += s * x.z; acc[3] += s * x.w;
    }
  } else {
    for (int r = r0 + rlane; r < r1; r += 8) {
      const float s = w ? w[size_t(r) * ldw] : 1.0f;
      for (int c = 0; c < 4; ++c)
        if (col + c < ncol) acc[c] += s * X[size_t(r) * ldx + col + c];
    }
  }
  __shared__ float sh[8][32][5];
  for (int c = 0; c < 4; ++c) sh[rlane][lane][c] = acc[c];
  __syncthreads();
  if (rlane == 0) {
    for (int c = 0; c < 4; ++c) {
      if (col + c >= ncol) break;
      float t = 0.0f;
      for (int i = 0; i < 8; ++i) t += sh[i][lane][c];
      colsum_partials[blockIdx.y * kColsumMaxCols + col + c] = t;
    }
  }
}
__global__ void colsum_finish_kernel(int ncol, int nparts, float* out) {
  const int col = blockIdx.x * blockDim.x + threadIdx.x;
  if (col >= ncol) return;
  float t = 0.0f;
  for (int y = 0; y < nparts; ++y) t += colsum_partials[y * kColsumMaxCols + col];
  out[col] += t;
}

extern "C" int nero_colsum(const float* X, int ldx, int ncol, const float* w, int ldw, const int* m_ptr, int m_cap, float* out,
                           void* stream) {
  if (m_cap <= 0 || ncol <= 0) return NERO_OK;
  if (ncol > kColsumMaxCols) return NERO_ERR_ARG;
  const cudaStream_t st = (cudaStream_t)stream;
  dim3 grid((ncol + 127) / 128, kNumSMs);
  colsum_kernel<<<grid, 256, 0, st>>>(X, ldx, ncol, w, ldw, m_ptr, m_cap);
  colsum_finish_kernel<<<(ncol + 127) / 128, 128, 0, st>>>(ncol, kNumSMs, out);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}


// Adam over ONE flat fp32 parameter buffer (torch.optim.Adam semantics, amsgrad=False, maximize=False):
//   g += wd * p;  m = m + (g - m)(1 - b1);  v = b2 v + (1 - b2) g g;  p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
// bc1 = 1 - b1^t, bc2 = 1 - b2^t are computed on the host.  Replaces the multi-tensor optimizer launch over the ~140
// small parameter tensors of a NeRO stage (train/trainer.py:73-76, 160-166) with one pass over 2.2 M floats.
__global__ void adam_flat_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 long n, float lr_over_bc1, float b1, float b2, float eps, float inv_sqrt_bc2, float wd) {
  const long i4 = (long(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (i4 >= n) return;
  if (i4 + 3 < n) {
    float4 P = *reinterpret_cast<float4*>(p + i4), M = *reinterpret_cast<float4*>(m + i4), V = *reinterpret_cast<float4*>(v + i4);
    const float4 G = *reinterpret_cast<const float4*>(g + i4);
    float* pp = reinterpret_cast<float*>(&P); float* mm = reinterpret_cast<float*>(&M); float* vv = reinterpret_cast<float*>(&V);
    const float* gg = reinterpret_cast<const float*>(&G);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float gr = gg[j] + wd * pp[j];
      mm[j] = mm[j] + (gr - mm[j]) * (1.0f - b1);
      vv[j] = vv[j] * b2 + (1.0f - b2) * gr * gr;
      pp[j] -= lr_over_bc1 * (mm[j] / (sqrtf(vv[j]) * inv_sqrt_bc2 + eps));
    }
    *reinterpret_cast<float4*>(p + i4) = P; *reinterpret_cast<float4*>(m + i4) = M; *reinterpret_cast<float4*>(v + i4) = V;
  } else {
    for (long i = i4; i < n; ++i) {
      const float gr = g[i] + wd * p[i];
      m[i] = m[i] + (gr - m[i]) * (1.0f - b1);
      v[i] = v[i] * b2 + (1.0f - b2) * gr * gr;
      p[i] -= lr_over_bc1 * (m[i] / (sqrtf(v[i]) * inv_sqrt_bc2 + eps));
    }
  }
}
extern "C" int nero_adam_flat(float* p, const float* g, float* m, float* v, long long n, float lr_over_bc1, float b1, float b2, float eps,
                              float inv_sqrt_bc2, float weight_decay, void* stream) {
  if (!p || !g || !m || !v) return NERO_ERR_ARG;
  if (n <= 0) return NERO_OK;
  if ((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) | reinterpret_cast<uintptr_t>(v)) & 15)
    return NERO_ERR_ARG;
  const long n4 = (n + 3) / 4;
  adam_flat_kernel<<<int((n4 + 255) / 256), 256, 0, (cudaStream_t)stream>>>(p, g, m, v, long(n), lr_over_bc1, b1, b2, eps, inv_sqrt_bc2,
                                                                            weight_decay);
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
