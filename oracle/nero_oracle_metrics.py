"""numpy / scipy oracle of the image metrics (nero_b200/metrics.py, k_metrics.cu).

Restates, independently of the kernels:
  * color_map_backward: utils/base_utils.py:453-456 on fp32 input (one fp32 multiply, clip, truncate; NaN -> 0).
  * psnr_exact: int64 squared-error sums per channel, fp64 means, 10 log10(255^2 / mse); inf when mse == 0.
  * psnr_reference: network/metrics.py:11-17 as written, numpy's float32 per-channel sums included.
  * uniform_filter_explicit: scipy.ndimage.uniform_filter(., size) ('reflect') as a running sum per line, axis 0 then axis 1.
  * ssim / ssim_map: skimage.metrics.structural_similarity(gt, pr, win_size=11, channel_axis=2, data_range=255) with its
    defaults (uniform window, sample covariance, K1 = 0.01, K2 = 0.03), on the explicit filter.
  * concat_images_list: utils/draw_utils.py:163-183 with np.pad in place of cv2.copyMakeBorder, and the two montages of
    network/metrics.py:39-104.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np

WIN = 11
K1, K2 = 0.01, 0.03


def color_map_backward(x):
    """fp32 [...] -> uint8: v = x * 255 in fp32, clipped to [0, 255] and truncated; NaN -> 0."""
    v = np.asarray(x, np.float32) * np.float32(255)
    v = np.where(np.isnan(v), np.float32(0), np.clip(v, 0, 255))
    return v.astype(np.uint8)


def sse(gt, pr):
    """Exact int64 [C] sums of squared differences of two uint8 [H, W, C] images."""
    d = gt.astype(np.int64) - pr.astype(np.int64)
    return (d * d).reshape(-1, gt.shape[-1]).sum(0)


def psnr_exact(gt, pr):
    h, w = gt.shape[:2]
    mse = np.mean(sse(gt, pr).astype(np.float64) / (h * w))
    return np.inf if mse == 0 else 10 * np.log10(65025.0 / mse)


def psnr_reference(gt, pr):
    """compute_psnr (network/metrics.py:11-17) as written: float32 throughout, numpy's sequential float32 column sums."""
    gt = gt.reshape([-1, 3]).astype(np.float32)
    pr = pr.reshape([-1, 3]).astype(np.float32)
    mse = np.mean((gt - pr) ** 2, 0)
    mse = np.mean(mse)
    return 10 * np.log10(255 * 255 / mse)


def _reflect_index(n, r):
    """Indices of a line of length n extended by r on each side with half-sample reflection (d c b a | a b c d | d c b a)."""
    i = np.arange(-r, n + r)
    i = np.where(i < 0, -i - 1, i)
    return np.where(i >= n, 2 * n - 1 - i, i)


def uniform_filter1d_explicit(a, size, axis):
    """Running-sum restatement of scipy.ndimage.uniform_filter1d(a, size, axis, mode='reflect') on fp64 data."""
    a = np.moveaxis(np.asarray(a, np.float64), axis, 0)
    n, r = a.shape[0], size // 2
    e = a[_reflect_index(n, r)]
    out = np.empty_like(a)
    t = e[0].copy()
    for j in range(1, size):
        t = t + e[j]
    out[0] = t / size
    for k in range(1, n):
        t = t + (e[k + size - 1] - e[k - 1])
        out[k] = t / size
    return np.moveaxis(out, 0, axis)


def uniform_filter_explicit(a, size=WIN):
    """scipy.ndimage.uniform_filter(a, size) of a 2-D plane: axis 0, then axis 1 on the fp64 result."""
    return uniform_filter1d_explicit(uniform_filter1d_explicit(a, size, 0), size, 1)


def _check(gt, pr, win_size):
    if gt.shape != pr.shape:
        raise ValueError(f'images differ in shape: {gt.shape} and {pr.shape}')
    if win_size % 2 != 1:
        raise ValueError('Window size must be odd.')
    if min(gt.shape[:2]) < win_size:
        raise ValueError(f'win_size {win_size} exceeds image extent {gt.shape[:2]}')


def ssim_plane(x, y, win_size=WIN, data_range=255.0):
    """(S map, mean of S over the map with a (win_size - 1) / 2 border cropped) of two 2-D planes, in fp64."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    f = lambda a: uniform_filter_explicit(a, win_size)
    np_ = win_size ** 2
    cov_norm = np_ / (np_ - 1)
    ux, uy, uxx, uyy, uxy = f(x), f(y), f(x * x), f(y * y), f(x * y)
    vx = cov_norm * (uxx - ux * ux)
    vy = cov_norm * (uyy - uy * uy)
    vxy = cov_norm * (uxy - ux * uy)
    C1, C2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    A1, A2 = 2 * ux * uy + C1, 2 * vxy + C2
    B1, B2 = ux * ux + uy * uy + C1, vx + vy + C2
    S = (A1 * A2) / (B1 * B2)
    p = (win_size - 1) // 2
    return S, S[p:S.shape[0] - p, p:S.shape[1] - p].mean(dtype=np.float64)


def ssim_map(gt, pr, win_size=WIN):
    """(S [H, W, C] fp64, per-channel means [C]) of two [H, W, C] images."""
    _check(gt, pr, win_size)
    res = [ssim_plane(gt[..., c], pr[..., c], win_size) for c in range(gt.shape[-1])]
    return np.stack([r[0] for r in res], -1), np.asarray([r[1] for r in res])


def ssim(gt, pr, win_size=WIN):
    """structural_similarity(gt, pr, win_size, channel_axis=2, data_range=255): the mean over channels."""
    return float(np.mean(ssim_map(gt, pr, win_size)[1]))


# ------------------------------------------------------------------------------------------------ montage
def concat_images(img0, img1, vert=False):
    if not vert:
        h0, h1 = img0.shape[0], img1.shape[0]
        if h0 < h1: img0 = np.pad(img0, ((0, h1 - h0), (0, 0), (0, 0)))
        if h1 < h0: img1 = np.pad(img1, ((0, h0 - h1), (0, 0), (0, 0)))
        return np.concatenate([img0, img1], axis=1)
    w0, w1 = img0.shape[1], img1.shape[1]
    if w0 < w1: img0 = np.pad(img0, ((0, 0), (0, w1 - w0), (0, 0)))
    if w1 < w0: img1 = np.pad(img1, ((0, 0), (0, w0 - w1), (0, 0)))
    return np.concatenate([img0, img1], axis=0)


def concat_images_list(*args, vert=False):
    out = args[0]
    for img in args[1:]:
        out = concat_images(out, img, vert)
    return out


def _key_img(v, h, w):
    img = color_map_backward(v).reshape([h, w, -1])
    return np.repeat(img, 3, axis=-1) if img.shape[-1] == 1 else img


SHAPE_MATERIAL_KEYS = ['diffuse_albedo', 'diffuse_light', 'diffuse_color', 'specular_albedo', 'specular_light', 'specular_color',
                       'specular_ref', 'metallic', 'roughness', 'occ_prob', 'indirect_light']
MATERIAL_EXTRA_KEYS = ['albedo', 'metallic', 'roughness', 'specular_light', 'specular_color', 'diffuse_light', 'diffuse_color']


def shape_montage(data_pr):
    """ShapeRenderMetrics' image (network/metrics.py:43-71) from numpy fp32 outputs."""
    gt, pr = color_map_backward(data_pr['gt_rgb']), color_map_backward(data_pr['ray_rgb'])
    h, w, _ = pr.shape
    imgs = [gt, pr, color_map_backward(data_pr['normal']).reshape([h, w, 3])]
    if 'human_light' in data_pr:
        imgs.append(_key_img(data_pr['human_light'], h, w))
    rows = [concat_images_list(*imgs)]
    mats = [_key_img(data_pr[k], h, w) for k in SHAPE_MATERIAL_KEYS if k in data_pr]
    rows += [concat_images_list(*mats[0:3]), concat_images_list(*mats[3:7]), concat_images_list(*mats[7:])]
    return concat_images_list(*rows, vert=True)


def material_montage(data_pr):
    """MaterialRenderMetrics' image (network/metrics.py:78-101) from numpy fp32 outputs."""
    imgs = [color_map_backward(data_pr['rgb_gt']), color_map_backward(data_pr['rgb_pr'])]
    for k in MATERIAL_EXTRA_KEYS:
        img = color_map_backward(data_pr[k])
        imgs.append(np.repeat(img, 3, axis=-1) if img.shape[-1] == 1 else img)
    return concat_images_list(concat_images_list(*imgs[:5]), concat_images_list(*imgs[5:]), vert=True)
