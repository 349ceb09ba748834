"""Denoising of relit frames on the GPU: a feature-guided edge-avoiding a-trous wavelet filter (Dammertz et al. 2010; the
spatial filter of SVGF, Schied et al. 2017) on albedo-demodulated radiance.

The path tracer's AOV instances (Relighter.render_sums) add per-pixel feature sums over the camera samples that hit the mesh:
the demodulated radiance D = L / (g + DEMOD_EPS) and the square of its luminance, and the first hit's guide albedo
g = (1 - m) albedo + 0.04 (1 - m) + m albedo (diffuse plus normal-incidence specular reflectance of NeRO's BRDF), face normal,
point and depth.  `denoise` then runs
  prep     per-pixel means over the hits, the luminance variance of the mean (fp64; VAR_NONE below two hits), unit normal,
           pixel footprint depth / focal, and coverage alpha = hits / spp;
  iterate  `iterations` passes at steps 1, 2, 4, ...: 5x5 B3-spline taps weighted by a luminance stop scaled by the
           3x3-prefiltered variance, a normal stop and a position stop sigma_x pixel footprints wide (times the step), each
           times the tap's coverage; the variance propagates as sum w^2 var / (sum w)^2;
  finish   remodulation by g + DEMOD_EPS and premultiplication by the pixel's own alpha: the [h,w,4] layout Relighter.render
           returns, so to_rgba8 / write_png_rgba apply unchanged and alpha passes through untouched.
Every formula and the buffer layouts are stated in include/nero_denoise.h; oracle/nero_oracle_denoise.py restates them in fp64.
One thread per output pixel, taps in a fixed order and no atomics: two runs give the same bits.
"""
from . import ops

AOV = 16               # NERO_DENOISE_AOV: floats per pixel of the feature sums
DEMOD_EPS = 1e-3       # NERO_DENOISE_DEMOD_EPS
VAR_NONE = 1e20        # NERO_DENOISE_VAR_NONE
MAX_ITERATIONS = 8     # NERO_DENOISE_MAX_LEVEL + 1
ITERATIONS = 5         # the defaults: NERO_DENOISE_ITERATIONS, _SIGMA_L, _SIGMA_N, _SIGMA_X (pixel footprints), _EPS
SIGMA_L = 4.0
SIGMA_N = 64.0
SIGMA_X = 1.4
EPS = 1e-3


def denoise(accum, aov, spp, focal, iterations=ITERATIONS, sigma_l=SIGMA_L, sigma_n=SIGMA_N, sigma_x=SIGMA_X, eps=EPS):
    """accum [h,w,4] (rgb and hit-count sums) and aov [h,w,16] feature sums of `spp` samples per pixel, CUDA float32 ->
    the denoised image, CUDA float32 [h,w,4] (linear RGB premultiplied by coverage, alpha = hits / spp).
    focal: the camera's focal length in pixels (K[0,0]), which sets the pixel footprint."""
    import torch
    if accum.dim() != 3 or accum.shape[2] != 4 or tuple(aov.shape) != tuple(accum.shape[:2]) + (AOV,):
        raise ValueError(f'accum {tuple(accum.shape)} and aov {tuple(aov.shape)}: expected [h,w,4] and [h,w,{AOV}]')
    if accum.dtype != torch.float32 or aov.dtype != torch.float32 or not accum.is_contiguous() or not aov.is_contiguous():
        raise ValueError('accum and aov must be contiguous float32 tensors')
    ops.require_cuda(accum.device, 'denoise')
    ops.require_cuda(aov.device, 'denoise')
    if not 1 <= iterations <= MAX_ITERATIONS:
        raise ValueError(f'iterations {iterations}: expected 1..{MAX_ITERATIONS}')
    if spp < 1 or not focal > 0 or not min(sigma_l, sigma_n, sigma_x, eps) > 0:
        raise ValueError('spp, focal, the sigmas and eps must be positive')
    h, w = accum.shape[:2]
    col = torch.empty(2, h, w, 4, device=accum.device)
    feat = torch.empty(h, w, 12, device=accum.device)
    out = torch.empty(h, w, 4, device=accum.device)
    ops.K('nero_denoise_prep', accum, aov, spp, w, h, focal, col[0], feat)
    for i in range(iterations):
        ops.K('nero_denoise_iterate', col[i % 2], feat, w, h, i, sigma_l, sigma_n, sigma_x, eps, col[(i + 1) % 2])
    ops.K('nero_denoise_finish', col[iterations % 2], feat, w, h, out)
    return out
