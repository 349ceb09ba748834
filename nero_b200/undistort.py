"""Lens undistortion on the GPU: a COLMAP model with SIMPLE_RADIAL cameras and its images resampled to a pinhole project,
without COLMAP's image_undistorter.

Reference being replaced (paths relative to the reference repository):
  run_colmap.py:65-70   colmap image_undistorter --image_path <images> --input_path <root>/sparse/0 --output_path <dense>
CustomDatabase._parse_colmap (dataset/database.py) and objprep._intrinsics read a SIMPLE_RADIAL camera and drop its k, so
images with lens distortion would be trained, matched and cropped as if they were pinhole images.  After this step every
camera is SIMPLE_PINHOLE and the images agree with it.  The rule below is this project's own; it is not pinned to
COLMAP's undistorter, which picks its output camera and interpolation differently (DESIGN.md section 2).

The convention (k_undistort.cu, include/nero_undistort.h, oracle/nero_oracle_undistort.py):
  * Model.  SIMPLE_RADIAL (f, cx, cy, k): Y = R X + t, x = Y_x / Y_z, y = Y_y / Y_z, r2 = x^2 + y^2,
    u = (f x)(1 + k r2) + cx, v = (f y)(1 + k r2) + cy.  Pixel (i, j) has its centre at (i + 1/2, j + 1/2), the convention
    of the keypoints (features.py).
  * Inverse.  xd = (u - cx) / f, yd = (v - cy) / f, rd = |(xd, yd)|; NEWTON fixed steps of Newton's method on
    r (1 + k r^2) = rd from r = rd, in fp64; x = xd (r / rd) (xd itself when rd = 0).  A point is invalid when it leaves
    the monotone branch (1 + 3 k r^2 <= 0) or its residual exceeds TOL; invalid points are never used.
  * Undistorted camera (host, fp64).  The boundary points (0, j + 1/2), (w, j + 1/2) of every row and (i + 1/2, 0),
    (i + 1/2, h) of every column are inverted; x0 = max over the left edge, x1 = min over the right edge, y0 = max over
    the top edge, y1 = min over the bottom edge: the largest axis-aligned rectangle inside them.  The output camera is
    SIMPLE_PINHOLE with the same f, W' = floor(f (x1 - x0) + 1/2), H' = floor(f (y1 - y0) + 1/2) and
    cx' = cx + f ((0 - cx) / f - x0) (= -f x0, written so that k = 0 gives back cx exactly), cy' likewise.  A camera is
    refused, by name, when a boundary point is invalid or W' / w or H' / h leaves [0.5, 2].  With k = 0 the rule returns
    (w, h, cx, cy) and the warp returns the input bytes.
  * Warp.  Output pixel (i, j): x = (i + 1/2 - cx') / f, y = (j + 1/2 - cy') / f, distorted into the input at (u, v),
    sampled bilinearly at texel point (u - 1/2, v - 1/2) with the taps clamped to the image, each channel rounded half up
    to uint8.  All fp64, uncontracted, so the oracle reproduces the bytes.
  * Project.  Pinhole cameras (SIMPLE_PINHOLE, PINHOLE) pass through and their images are copied byte for byte.  Every
    SIMPLE_RADIAL camera becomes the SIMPLE_PINHOLE camera above and its images are warped: PNG through relight.write_png,
    JPEG through OpenCV at quality 100 (lossy, as COLMAP's output is).  Image ids, names, poses and points3D are unchanged;
    POINTS2D are inverted and mapped to f x + cx', f y + cy'.  A keypoint whose inverse is invalid refuses the project
    before any output file is written (its POINTS2D index is referenced by points3D, so it cannot be dropped silently).
    Any other camera model is refused before any GPU work.
"""
import os
import shutil

import numpy as np

NEWTON = 50          # NERO_UNDISTORT_NEWTON (include/nero_undistort.h)
TOL = 1e-12          # NERO_UNDISTORT_TOL
PINHOLE_MODELS = ('SIMPLE_PINHOLE', 'PINHOLE')
RADIAL_MODELS = ('SIMPLE_RADIAL',)


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ host fp64
def undistort_host(u, v, f, cx, cy, k):
    """(x, y, valid) of image points (u, v) of camera (f, cx, cy, k), on the host: the kernel's inverse, operation for
    operation."""
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    xd, yd = (u - cx) / f, (v - cy) / f
    rd = np.sqrt(xd * xd + yd * yd)
    r = rd.copy()
    with np.errstate(all='ignore'):
        for _ in range(NEWTON):
            t = k * (r * r)
            r = r - (r * (1.0 + t) - rd) / (1.0 + 3.0 * t)
        t = k * (r * r)
        e = r * (1.0 + t) - rd
        valid = (1.0 + 3.0 * t > 0.0) & (np.abs(e) <= TOL) & (r >= 0.0)
        s = r / np.where(rd > 0.0, rd, 1.0)
    return np.where(rd > 0.0, xd * s, xd), np.where(rd > 0.0, yd * s, yd), valid


def camera(w, h, f, cx, cy, k, name='camera'):
    """(W', H', cx', cy') of the undistorted SIMPLE_PINHOLE camera of SIMPLE_RADIAL (f, cx, cy, k) at w x h.  ValueError,
    naming the camera, when the rule refuses it."""
    w, h, f, cx, cy, k = int(w), int(h), float(f), float(cx), float(cy), float(k)
    if w < 1 or h < 1 or not f > 0 or not all(np.isfinite([f, cx, cy, k])):
        raise ValueError(f'{name}: needs w, h >= 1, f > 0 and finite parameters, got {w} x {h}, {(f, cx, cy, k)}')
    rows, cols = np.arange(h) + 0.5, np.arange(w) + 0.5
    lx, _, lv = undistort_host(np.zeros(h), rows, f, cx, cy, k)
    rx, _, rv = undistort_host(np.full(h, float(w)), rows, f, cx, cy, k)
    _, ty, tv = undistort_host(cols, np.zeros(w), f, cx, cy, k)
    _, by, bv = undistort_host(cols, np.full(w, float(h)), f, cx, cy, k)
    bad = int((~lv).sum() + (~rv).sum() + (~tv).sum() + (~bv).sum())
    if bad:
        raise ValueError(f'{name}: k = {k:g} is outside the invertible range at {bad} image border points')
    x0, x1, y0, y1 = lx.max(), rx.min(), ty.max(), by.min()
    W, H = int(np.floor(f * (x1 - x0) + 0.5)), int(np.floor(f * (y1 - y0) + 0.5))
    if not (0.5 <= W / w <= 2.0 and 0.5 <= H / h <= 2.0):
        raise ValueError(f'{name}: k = {k:g} gives an undistorted image of {W} x {H} from {w} x {h} (the ratio must lie in '
                         '[0.5, 2])')
    return W, H, cx + f * ((0.0 - cx) / f - x0), cy + f * ((0.0 - cy) / f - y0)


# ------------------------------------------------------------------------------------------------ GPU
def points(xy, f, cx, cy, k):
    """Undistorted normalised coordinates of image points xy [n, 2] (numpy or tensor) of camera (f, cx, cy, k) ->
    (xn CUDA fp64 [n, 2], valid CUDA bool [n])."""
    torch = _torch()
    x = xy if torch.is_tensor(xy) else torch.from_numpy(np.asarray(xy, np.float64))
    x = x.to('cuda', torch.float64).reshape(-1, 2).contiguous()
    n = x.shape[0]
    xn = torch.empty(n, 2, dtype=torch.float64, device=x.device)
    valid = torch.empty(n, dtype=torch.int32, device=x.device)
    _ops().K('nero_undistort_points', x, n, float(f), float(cx), float(cy), float(k), xn, valid)
    return xn, valid.bool()


def image(rgb, f, cx, cy, k, W, H, cx2, cy2):
    """uint8 RGB [h, w, 3] (numpy or tensor) of camera (f, cx, cy, k) resampled to the pinhole camera (f, cx2, cy2) of
    size W x H -> CUDA uint8 [H, W, 3]."""
    torch = _torch()
    x = rgb if torch.is_tensor(rgb) else torch.from_numpy(np.ascontiguousarray(rgb, np.uint8))
    if x.dtype != torch.uint8 or x.dim() != 3 or x.shape[2] != 3:
        raise ValueError(f'undistort.image needs uint8 RGB [h,w,3], got {x.dtype} {tuple(x.shape)}')
    x = x.cuda().contiguous()
    h, w = x.shape[:2]
    out = torch.empty(int(H), int(W), 3, dtype=torch.uint8, device=x.device)
    _ops().K('nero_undistort_image', x, w, h, float(f), float(cx), float(cy), float(k), out, int(W), int(H), float(cx2), float(cy2))
    return out


# ------------------------------------------------------------------------------------------------ project
def plan(sparse):
    """Read the model in `sparse` and work out every camera's output without touching the GPU ->
    (cameras, images, points, new_cameras), new_cameras = {id: (model, W, H, params)}.  ValueError for a camera model
    other than SIMPLE_PINHOLE, PINHOLE and SIMPLE_RADIAL, or a camera the rule refuses."""
    from . import objprep
    cams, images, pts = objprep.read_colmap_records(sparse)
    new = {}
    for cid, (model, w, h, par) in cams.items():
        if model in PINHOLE_MODELS:
            new[cid] = (model, w, h, list(par))
        elif model in RADIAL_MODELS:
            f, cx, cy, k = par
            W, H, cx2, cy2 = camera(w, h, f, cx, cy, k, name=f'camera {cid}')
            new[cid] = ('SIMPLE_PINHOLE', W, H, [f, cx2, cy2])
        else:
            raise ValueError(f'camera {cid} is {model}: the undistorter takes SIMPLE_RADIAL, SIMPLE_PINHOLE and PINHOLE cameras '
                             'only (other distortion models are not supported)')
    for iid, (_, _, cid, name, _, _) in images.items():
        if cid not in cams:
            raise ValueError(f'{sparse}: image {iid} ({name}) uses camera {cid}, which the model does not define')
    return cams, images, pts, new


def _write_image(path, rgb):
    if os.path.splitext(path)[1].lower() == '.png':
        from .relight import write_png
        write_png(path, rgb)
        return
    import cv2
    if not cv2.imwrite(path, np.ascontiguousarray(rgb[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, 100]):
        raise OSError(f'{path}: cannot write the image')


def project(sparse, image_dir, output, log=None):
    """The whole tool: <output>/images/<name> and <output>/sparse/0 from the model in `sparse` and its images.  The
    caller checks that `output` may be written.  -> summary dict."""
    from . import mvs, objprep
    cams, images, pts, new = plan(sparse)
    for iid, (_, _, cid, name, _, _) in images.items():          # missing files and formats, before any output file
        if not os.path.isfile(os.path.join(image_dir, name)):
            raise FileNotFoundError(f'image {iid}: {os.path.join(image_dir, name)} does not exist')
        if cams[cid][0] in RADIAL_MODELS and os.path.splitext(name)[1].lower() not in ('.png', '.jpg', '.jpeg'):
            raise ValueError(f'image {iid} ({name}): the undistorter writes .png and .jpg / .jpeg images only')
    out_images = {}
    for iid, (q, t, cid, name, xys, p3d) in images.items():      # keypoints first: an invalid one writes nothing
        model, _, _, par = cams[cid]
        if model in PINHOLE_MODELS:
            out_images[iid] = (q, t, cid, name, xys, p3d)
            continue
        f, cx, cy, k = par
        _, _, _, (_, cx2, cy2) = new[cid]
        xn, ok = points(xys, f, cx, cy, k)
        xn, ok = xn.cpu().numpy(), ok.cpu().numpy()
        if not ok.all():
            raise ValueError(f'image {iid} ({name}): {int((~ok).sum())} keypoints lie outside the invertible range of camera {cid}')
        out_images[iid] = (q, t, cid, name, np.stack([f * xn[:, 0] + cx2, f * xn[:, 1] + cy2], 1), p3d)
    warped = copied = 0
    for iid, (q, t, cid, name, xys, p3d) in images.items():
        model, w, h, par = cams[cid]
        src, dst = os.path.join(image_dir, name), os.path.join(output, 'images', name)
        os.makedirs(os.path.dirname(dst), exist_ok=True)
        if model in PINHOLE_MODELS:
            shutil.copyfile(src, dst)
            copied += 1
            continue
        f, cx, cy, k = par
        _, W, H, (_, cx2, cy2) = new[cid]
        rgb = mvs.read_rgb(src)
        if rgb.shape[:2] != (h, w):
            raise ValueError(f'{src} is {rgb.shape[1]} x {rgb.shape[0]}, but its camera {cid} is {w} x {h}')
        _write_image(dst, image(rgb, f, cx, cy, k, W, H, cx2, cy2).cpu().numpy())
        warped += 1
        if log:
            log(f'{name}: {w} x {h} -> {W} x {H}')
    objprep.write_colmap_model(os.path.join(output, 'sparse', '0'), new, out_images, pts)
    return dict(cameras=new, warped=warped, copied=copied, points=len(pts))
