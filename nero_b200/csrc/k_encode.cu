// Stand-alone encoding kernels (SURVEY.md section 8b "ide/pe standalone", 8d algorithmic bytes): the positional encoding
// of get_embedder (network/field.py:14-58) here, the integrated directional encoding of generate_ide_fn
// (utils/ref_utils.py:53-117) next to its coefficient table in k_shade.cu, as HBM-streaming kernels.  In the training path both are fused into their consumers
// (ray_fill, shade_prep, mc_fill); these entry points exist for export scripts / other callers and for the bandwidth
// evidence of the encoding math: one thread encodes one sample into shared memory, the block then writes the rows out
// with fully coalesced 128-byte segments.
#include "common.cuh"
#include "math_enc.cuh"

namespace nero {

constexpr int kEncBlock = 128;

// out[i, 0:d(1+2L)] = PE_L(x[i, 0:d]) * scale
template <int D>
__global__ void __launch_bounds__(kEncBlock) pe_kernel(const float* __restrict__ x, int ldx, int M, int L, float scale, float* __restrict__ out, int ldo) {
  extern __shared__ float s_rows[];
  const int ncol = D * (1 + 2 * L);
  const int pitch = ncol | 1;                                   // odd pitch: conflict-free row-per-thread writes
  const int i0 = blockIdx.x * kEncBlock;
  const int i = i0 + threadIdx.x;
  if (i < M) {
    float v[D];
#pragma unroll
    for (int c = 0; c < D; ++c) v[c] = x[size_t(i) * ldx + c];
    pe_encode<D>(v, L, s_rows + threadIdx.x * pitch, scale);
  }
  __syncthreads();
  const int rows = min(kEncBlock, M - i0);
  if (ldo == ncol) {                                            // dense output: one contiguous range per block
    float* dst = out + size_t(i0) * ncol;
    for (int e = threadIdx.x; e < rows * ncol; e += kEncBlock) dst[e] = s_rows[(e / ncol) * pitch + e % ncol];
  } else {
    for (int r = threadIdx.x >> 5; r < rows; r += kEncBlock / 32)
      for (int c = threadIdx.x & 31; c < ncol; c += 32) out[size_t(i0 + r) * ldo + c] = s_rows[r * pitch + c];
  }
}

extern "C" int nero_pe(const float* x, int d, int ldx, int M, int L, float scale, float* out, int ldo, void* stream) {
  if (!x || !out || (d != 3 && d != 4) || L < 0 || L > 16 || ldx < d || ldo < d * (1 + 2 * L)) return NERO_ERR_ARG;
  if (M <= 0) return NERO_OK;
  const int ncol = d * (1 + 2 * L);
  const size_t smem = size_t(kEncBlock) * (ncol | 1) * sizeof(float);
  const int grid = (M + kEncBlock - 1) / kEncBlock;
  const cudaStream_t st = (cudaStream_t)stream;
  if (d == 3) pe_kernel<3><<<grid, kEncBlock, smem, st>>>(x, ldx, M, L, scale, out, ldo);
  else {
    static bool attr = false;
    if (!attr) { cudaFuncSetAttribute(pe_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024); attr = true; }
    pe_kernel<4><<<grid, kEncBlock, smem, st>>>(x, ldx, M, L, scale, out, ldo);
  }
  NERO_LAUNCH_CHECK();
  return NERO_OK;
}

}  // namespace nero
