"""numpy fp64 restatement of include/nero_undistort.h and nero_b200/undistort.py: the SIMPLE_RADIAL model, its inverse, the
rule that picks the undistorted pinhole camera and the image warp, operation for operation, so the kernels' outputs are
compared bit for bit.  numpy evaluates every float64 operation correctly rounded and never contracts a * b + c."""
import numpy as np

NEWTON = 50          # NERO_UNDISTORT_NEWTON
TOL = 1e-12          # NERO_UNDISTORT_TOL


def distort(x, y, f, cx, cy, k):
    """Image point (u, v) of normalised coordinates (x, y)."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    d = 1.0 + k * (x * x + y * y)
    return (f * x) * d + cx, (f * y) * d + cy


def undistort(u, v, f, cx, cy, k):
    """(x, y, valid) of image points (u, v): the fixed-step Newton inverse of the header."""
    u, v = np.asarray(u, np.float64), np.asarray(v, np.float64)
    xd, yd = (u - cx) / f, (v - cy) / f
    rd = np.sqrt(xd * xd + yd * yd)
    r = rd.copy()
    with np.errstate(all='ignore'):
        for _ in range(NEWTON):
            t = k * (r * r)
            e = r * (1.0 + t) - rd
            r = r - e / (1.0 + 3.0 * t)
        t = k * (r * r)
        e = r * (1.0 + t) - rd
        valid = (1.0 + 3.0 * t > 0.0) & (np.abs(e) <= TOL) & (r >= 0.0)
        s = np.where(rd > 0.0, r / np.where(rd > 0.0, rd, 1.0), 1.0)
    return np.where(rd > 0.0, xd * s, xd), np.where(rd > 0.0, yd * s, yd), valid


def camera(w, h, f, cx, cy, k):
    """(W', H', cx', cy') of the undistorted pinhole camera, or None when the rule refuses the camera."""
    rows, cols = np.arange(h) + 0.5, np.arange(w) + 0.5
    lx, _, lv = undistort(np.zeros(h), rows, f, cx, cy, k)
    rx, _, rv = undistort(np.full(h, float(w)), rows, f, cx, cy, k)
    _, ty, tv = undistort(cols, np.zeros(w), f, cx, cy, k)
    _, by, bv = undistort(cols, np.full(w, float(h)), f, cx, cy, k)
    if not (lv.all() and rv.all() and tv.all() and bv.all()):
        return None
    x0, x1, y0, y1 = lx.max(), rx.min(), ty.max(), by.min()
    W, H = int(np.floor(f * (x1 - x0) + 0.5)), int(np.floor(f * (y1 - y0) + 0.5))
    if not (0.5 <= W / w <= 2.0 and 0.5 <= H / h <= 2.0):
        return None
    return W, H, cx + f * ((0.0 - cx) / f - x0), cy + f * ((0.0 - cy) / f - y0)


def _axis(t, n):
    f0 = np.floor(t)
    a = t - f0
    c = np.fmin(np.fmax(f0, -1.0), float(n)).astype(np.int64)
    return np.clip(c, 0, n - 1), np.clip(c + 1, 0, n - 1), a


def warp(src, f, cx, cy, k, W, H, cx2, cy2):
    """uint8 [H, W, 3] of the input src [h, w, 3] of camera (f, cx, cy, k) resampled to the pinhole camera (f, cx2, cy2)."""
    src = np.asarray(src, np.uint8)
    h, w = src.shape[:2]
    j, i = np.mgrid[0:H, 0:W]
    x, y = ((i + 0.5) - cx2) / f, ((j + 0.5) - cy2) / f
    u, v = distort(x, y, f, cx, cy, k)
    x0, x1, a = _axis(u - 0.5, w)
    y0, y1, b = _axis(v - 0.5, h)
    a, b = a[..., None], b[..., None]
    p = src.astype(np.float64)
    a0, b0 = 1.0 - a, 1.0 - b
    top = a0 * p[y0, x0] + a * p[y0, x1]
    bot = a0 * p[y1, x0] + a * p[y1, x1]
    val = np.floor((b0 * top + b * bot) + 0.5)
    return np.fmin(np.fmax(val, 0.0), 255.0).astype(np.uint8)


def pattern(x, y):
    """A smooth RGB test image as a function of normalised coordinates, in [0, 255]: its distorted and undistorted
    renderings are exact (each pixel evaluates it at its own ray), so resampling is measured against the truth."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    return np.stack([127.5 + 100 * np.sin(9 * x + 1) * np.cos(7 * y),
                     127.5 + 100 * np.cos(6 * x - 5 * y),
                     127.5 + 100 * np.sin(4 * x * y + 8 * y)], -1)


def render_pattern(w, h, f, cx, cy, k):
    """uint8 [h, w, 3]: pattern() at the ray of every pixel centre of camera (f, cx, cy, k), through the inverse."""
    j, i = np.mgrid[0:h, 0:w]
    x, y, ok = undistort(i + 0.5, j + 0.5, f, cx, cy, k)
    assert ok.all()
    return np.clip(np.floor(pattern(x, y) + 0.5), 0, 255).astype(np.uint8)
