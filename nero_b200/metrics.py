"""Image metrics on the GPU: PSNR and SSIM of rendered images, and drop-ins for the reference's validation metrics.

Reference being replaced (paths relative to the reference repository):
  network/metrics.py:11-17      compute_psnr: float32 squared errors of [N,3] arrays, np.mean(., 0), then the mean
  network/metrics.py:39-104     ShapeRenderMetrics / MaterialRenderMetrics: PSNR, skimage SSIM and a montage .jpg per view
  network/metrics.py:104-115    name2metrics, psnr(results), name2key_metrics
  utils/base_utils.py:450-456   color_map_forward / color_map_backward
  utils/draw_utils.py:163-183   concat_images / concat_images_list

Definitions (k_metrics.cu, include/nero_metrics.h):
  * Quantisation is color_map_backward on fp32 input: v = x * 255 as one fp32 multiply rounded to nearest, clipped to
    [0, 255] and truncated to uint8; NaN becomes 0 (what numpy does on x86), +inf 255 and -inf 0.  Scores are always taken
    on uint8 images, as the reference does; ground truth takes the same route (color_map_forward then color_map_backward,
    the identity on 8-bit data).
  * PSNR of one image: sse_c is the exact int64 sum of squared uint8 differences in channel c, mse_c = sse_c / (H W) in
    fp64, mse the mean of the mse_c in channel order, psnr = 10 log10(65025 / mse), inf when mse == 0.  This is the exact
    value.  The reference sums in float32 (numpy's sequential column sums pass 2^24 at 800^2), which loses up to ~0.5 % of
    the squared error and reports a PSNR up to ~0.02 dB too high; it also returns float32 where this returns float64.
  * SSIM is skimage's structural_similarity(gt, pr, win_size=11, channel_axis=2, data_range=255) with its defaults (uniform
    window, sample covariance, K1 = 0.01, K2 = 0.03).  Per channel, in fp64: ux, uy, uxx, uyy, uxy are uniform_filter of X,
    Y, X X, Y Y, X Y over 11 x 11; vx = cov_norm (uxx - ux ux), vy and vxy likewise; A1 = (2 ux) uy + C1, A2 = 2 vxy + C2,
    B1 = ux ux + uy uy + C1, B2 = vx + vy + C2; S = (A1 A2) / (B1 B2).  A channel's score is the mean of S with a 5-pixel
    border cropped, the image's the mean over its channels.  cov_norm = 121 / 120, C1 = (0.01 255)^2, C2 = (0.03 255)^2.
    The filter is scipy.ndimage.uniform_filter ('reflect' boundary) restated as a running sum per line, axis 0 first: t is
    the sum of the 11 extended values in order, out[0] = t / 11, then t += (e[k + 10] - e[k - 1]), out[k] = t / 11.  Every
    operation is an uncontracted fp64 op, so the S map equals the numpy / scipy expression bit for bit.  The mean sums each
    cropped row left to right and the rows in order (numpy's pairwise mean differs in the last bits).  An image side below
    11 raises ValueError, as skimage does.
"""
import os

import numpy as np

from . import ops

WIN = 11
_NP = WIN * WIN
COV_NORM = _NP / (_NP - 1)
C1 = (0.01 * 255) ** 2
C2 = (0.03 * 255) ** 2
MAX_WORK = 1 << 28                # fp64 elements of SSIM workspace per launch (2 GiB); larger batches run in groups of images


def _torch():
    import torch
    return torch


def color_map_backward(x):
    """CUDA float32 tensor -> CUDA uint8 tensor of the same shape (the quantisation of the module docstring)."""
    torch = _torch()
    if not isinstance(x, torch.Tensor):
        raise TypeError(f'color_map_backward takes a CUDA tensor, got {type(x).__name__}')
    ops.require_cuda(x.device, 'color_map_backward')
    if x.dtype != torch.float32:
        raise ValueError(f'color_map_backward takes float32 input, got {x.dtype}')
    x = x.contiguous()
    out = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    ops.K('nero_metrics_quantize', x, x.numel(), out, launches=int(x.numel() > 0))
    return out


def _pair(gt, pr, what):
    """Checked uint8 CUDA [B, H, W, C] views of two [H, W, C] or [B, H, W, C] images; -> (gt, pr, batched)."""
    torch = _torch()
    for a in (gt, pr):
        if not isinstance(a, torch.Tensor):
            raise TypeError(f'{what} takes CUDA tensors, got {type(a).__name__}')
        ops.require_cuda(a.device, what)
        if a.dtype != torch.uint8:
            raise ValueError(f'{what} takes uint8 images, got {a.dtype}')
    if gt.shape != pr.shape:
        raise ValueError(f'{what}: images differ in shape: {tuple(gt.shape)} and {tuple(pr.shape)}')
    if gt.dim() not in (3, 4) or not 1 <= gt.shape[-1] <= 4 or gt.numel() == 0:
        raise ValueError(f'{what} takes non-empty [H, W, C] or [B, H, W, C] images with 1 to 4 channels, got {tuple(gt.shape)}')
    batched = gt.dim() == 4
    if not batched:
        gt, pr = gt[None], pr[None]
    return gt.contiguous(), pr.contiguous(), batched


def psnr(gt, pr):
    """Exact PSNR of uint8 CUDA images [H, W, C] -> float, or [B, H, W, C] -> float64 [B]; inf for identical images."""
    torch = _torch()
    gt, pr, batched = _pair(gt, pr, 'psnr')
    B, H, W, C = gt.shape
    sse = torch.empty(B, C, dtype=torch.int64, device=gt.device)
    ops.K('nero_metrics_sse', gt, pr, B, H, W, C, sse)
    out = []
    for s in sse.cpu().numpy():
        mse = np.mean(s.astype(np.float64) / (H * W))
        out.append(np.inf if mse == 0 else 10 * np.log10(65025.0 / mse))
    return np.asarray(out, np.float64) if batched else float(out[0])


def ssim(gt, pr, full=False):
    """SSIM of uint8 CUDA images [H, W, C] -> float, or [B, H, W, C] -> float64 [B].  full=True also returns the S map as a
    CUDA float64 tensor of the input's shape, as skimage's full=True does."""
    torch = _torch()
    gt, pr, batched = _pair(gt, pr, 'ssim')
    B, H, W, C = gt.shape
    if min(H, W) < WIN:
        raise ValueError(f'ssim: win_size {WIN} exceeds image extent ({H}, {W})')
    per_image = 5 * H * W * C + C * H
    group = max(1, MAX_WORK // per_image)
    work = torch.empty(min(B, group) * per_image, dtype=torch.float64, device=gt.device)
    chan = torch.empty(B, C, dtype=torch.float64, device=gt.device)
    smap = torch.empty(B, H, W, C, dtype=torch.float64, device=gt.device) if full else None
    for b0 in range(0, B, group):
        n = min(group, B - b0)
        ops.K('nero_metrics_ssim', gt[b0:b0 + n], pr[b0:b0 + n], n, H, W, C, WIN, COV_NORM, C1, C2, work,
              None if smap is None else smap[b0:b0 + n], chan[b0:b0 + n], launches=3)
    score = np.asarray([np.mean(c) for c in chan.cpu().numpy()], np.float64)
    score = score if batched else float(score[0])
    if not full:
        return score
    return score, smap if batched else smap[0]


# ------------------------------------------------------------------------------------------------ the drop-ins
def concat_images_list(*imgs, vert=False):
    """concat_images_list (utils/draw_utils.py:163-183) on uint8 CUDA [h, w, 3] tensors: side by side (or stacked with
    vert=True), each image at the top (left) of its slot and zero padding below (right) of it."""
    torch = _torch()
    if len(imgs) == 1:
        return imgs[0]
    ax = 0 if vert else 1
    other = 1 - ax
    n = max(int(i.shape[other]) for i in imgs)
    pads = []
    for i in imgs:
        if i.shape[other] < n:
            shape = list(i.shape)
            shape[other] = n - i.shape[other]
            i = torch.cat([i, i.new_zeros(shape)], other)
        pads.append(i)
    return torch.cat(pads, ax)


def _key_img(v, h, w):
    """process_key_img (network/metrics.py:19-23) on the GPU."""
    img = color_map_backward(v.detach()).reshape(h, w, -1)
    return img.repeat(1, 1, 3) if img.shape[-1] == 1 else img


def write_montage(path, img):
    """Copy a uint8 CUDA [h, w, 3] RGB montage to the host once and write it with OpenCV (RGB -> BGR)."""
    import cv2
    if not cv2.imwrite(path, np.ascontiguousarray(img.cpu().numpy()[..., ::-1])):
        raise OSError(f'could not write {path}')


def _montage_path(kwargs, step):
    out = os.path.join('data', 'train_vis', str(kwargs['model_name']))
    os.makedirs(out, exist_ok=True)
    return os.path.join(out, f'{step}-index-{kwargs["data_index"]}.jpg')


class ShapeRenderMetrics:
    """network/metrics.py:39-72: PSNR / SSIM of `ray_rgb` against `gt_rgb` and the validation montage
    (data/train_vis/{model_name}/{step}-index-{data_index}.jpg), computed on the GPU."""
    MATERIAL_KEYS = ('diffuse_albedo', 'diffuse_light', 'diffuse_color', 'specular_albedo', 'specular_light', 'specular_color',
                     'specular_ref', 'metallic', 'roughness', 'occ_prob', 'indirect_light')

    def __init__(self, cfg):
        pass

    def __call__(self, data_pr, data_gt, step, **kwargs):
        rgb_gt = color_map_backward(data_pr['gt_rgb'].detach())
        rgb_pr = color_map_backward(data_pr['ray_rgb'].detach())
        outputs = {'psnr': np.asarray([psnr(rgb_gt, rgb_pr)]), 'ssim': np.asarray([ssim(rgb_gt, rgb_pr)])}
        h, w, _ = rgb_pr.shape
        imgs = [rgb_gt, rgb_pr, color_map_backward(data_pr['normal'].detach()).reshape(h, w, 3)]
        if 'human_light' in data_pr:
            imgs.append(_key_img(data_pr['human_light'], h, w))
        rows = [concat_images_list(*imgs)]
        mats = [_key_img(data_pr[k], h, w) for k in self.MATERIAL_KEYS if k in data_pr]
        rows += [concat_images_list(*mats[0:3]), concat_images_list(*mats[3:7]), concat_images_list(*mats[7:])]
        write_montage(_montage_path(kwargs, step), concat_images_list(*rows, vert=True))
        return outputs


class MaterialRenderMetrics:
    """network/metrics.py:74-102: PSNR / SSIM of `rgb_pr` against `rgb_gt` and the validation montage, on the GPU."""
    EXTRA_KEYS = ('albedo', 'metallic', 'roughness', 'specular_light', 'specular_color', 'diffuse_light', 'diffuse_color')

    def __init__(self, cfg):
        pass

    def __call__(self, data_pr, data_gt, step, *args, **kwargs):
        rgb_gt = color_map_backward(data_pr['rgb_gt'].detach())
        rgb_pr = color_map_backward(data_pr['rgb_pr'].detach())
        outputs = {'psnr': np.asarray([psnr(rgb_gt, rgb_pr)]), 'ssim': np.asarray([ssim(rgb_gt, rgb_pr)])}
        imgs = [rgb_gt, rgb_pr]
        for k in self.EXTRA_KEYS:
            img = color_map_backward(data_pr[k].detach())
            imgs.append(img.repeat(1, 1, 3) if img.shape[-1] == 1 else img)
        montage = concat_images_list(concat_images_list(*imgs[:5]), concat_images_list(*imgs[5:]), vert=True)
        write_montage(_montage_path(kwargs, step), montage)
        return outputs


name2metrics = {
    'shape_render': ShapeRenderMetrics,
    'mat_render': MaterialRenderMetrics,
}


def key_psnr(results):
    """The reference's key metric psnr(results) (network/metrics.py:109-110): the mean of the validation PSNRs."""
    return np.mean(results['psnr'])


name2key_metrics = {
    'psnr': key_psnr,
}
