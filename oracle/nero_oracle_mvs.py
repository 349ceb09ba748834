"""numpy restatement of the dense multi-view stereo kernels of k_mvs.cu (include/nero_mvs.h) in the GPU's arithmetic order,
so the kernels must match it bit for bit; plus a synthetic project (images, sparse model with tracks, true depth) of the
table / box / sphere scene of nero_oracle_objprep.scene for the tests and the benchmark.

There is no reference code to pin the kernels against: the reference workflow runs COLMAP's CUDA patch_match_stereo.  This
file states what the kernels compute instead (the protocol of nero_b200/mvs.py).  Elementwise numpy float32 arithmetic
rounds every operation to nearest, as the kernels' __f*_rn intrinsics, IEEE division and square root do; fp64 likewise.
"""
import os

import numpy as np

import nero_oracle_objprep as OOp

f32 = np.float32
MIN_VAR = f32(1e-5)
NO_COST = f32(2.0)
BEST = 3


# ------------------------------------------------------------------------------------------------ kernels
def grey(rgb, s):
    """fp32 [h // s, w // s] of uint8 RGB [h,w,3]."""
    rgb = np.asarray(rgb, np.int64)
    h, w = rgb.shape[0] // s, rgb.shape[1] // s
    y = (299 * rgb[..., 0] + 587 * rgb[..., 1] + 114 * rgb[..., 2])[:h * s, :w * s]
    acc = y.reshape(h, s, w, s).sum((1, 3))
    return acc.astype(f32) / f32(255000 * s * s)


def _offsets(radius, step):
    return list(range(-radius, radius + 1, step))


def ref_stats(g, radius, step):
    """fp32 [h,w,2]: mean, variance of every pixel's reference window."""
    h, w = g.shape
    ys, xs = np.mgrid[0:h, 0:w]
    s = np.zeros((h, w), f32)
    s2 = np.zeros((h, w), f32)
    n = 0
    for l in _offsets(radius, step):
        for k in _offsets(radius, step):
            r = g[np.clip(ys + l, 0, h - 1), np.clip(xs + k, 0, w - 1)]
            s = s + r
            s2 = s2 + r * r
            n += 1
    m = s / f32(n)
    return np.stack([m, s2 / f32(n) - m * m], -1)


def _mix(x):
    return OOp._mix(x)


def stream_key(seed, view, stage, pixel):
    with np.errstate(over='ignore'):
        h = _mix(np.uint32(np.uint32(seed) * np.uint32(0x9e3779b9) + np.uint32(0x7f4a7c15)))
        h = _mix(h ^ np.uint32(view))
        h = _mix(h ^ np.uint32(stage))
        return _mix(np.asarray(pixel, np.uint32) ^ h)


def uniform(key, dim):
    with np.errstate(over='ignore'):
        return (_mix(key ^ np.uint32(dim)) >> np.uint32(8)).astype(f32) * f32(2.0 ** -24)


def bilinear(img, X, Y):
    h, w = img.shape
    X = np.fmin(np.fmax(X, f32(-1)), f32(w) + f32(1))
    Y = np.fmin(np.fmax(Y, f32(-1)), f32(h) + f32(1))
    fx, fy = X - f32(0.5), Y - f32(0.5)
    x0, y0 = np.floor(fx), np.floor(fy)
    a, b = fx - x0, fy - y0
    ix, iy = x0.astype(np.int64), y0.astype(np.int64)
    xa, xb = np.clip(ix, 0, w - 1), np.clip(ix + 1, 0, w - 1)
    ya, yb = np.clip(iy, 0, h - 1), np.clip(iy + 1, 0, h - 1)
    a1 = f32(1) - a
    top = a1 * img[ya, xa] + a * img[ya, xb]
    bot = a1 * img[yb, xa] + a * img[yb, xb]
    return (f32(1) - b) * top + b * bot


class View:
    """One reference view as the kernels see it: grey, kinv (ifx, ify, ocx, ocy), stats, sources (grey images), src_geo
    [S,12] fp32, dmin, dmax (fp32), radius, step, seed, view."""

    def __init__(self, g, kinv, stats, src_greys, src_geo, dmin, dmax, radius, step, seed, view):
        self.g, self.stats, self.src, self.geo = g, stats, src_greys, np.asarray(src_geo, f32)
        self.ifx, self.ify, self.ocx, self.ocy = (f32(v) for v in kinv)
        self.dmin, self.dmax = f32(dmin), f32(dmax)
        self.radius, self.step, self.seed, self.view = radius, step, seed, view
        self.h, self.w = g.shape

    def ray(self, xs, ys):
        return ((xs.astype(f32) + f32(0.5)) * self.ifx + self.ocx, (ys.astype(f32) + f32(0.5)) * self.ify + self.ocy)


def source_cost(v, j, H, xs, ys, mr, vr):
    src = v.src[j]
    hs, ws = src.shape
    u, w = xs.astype(f32) + f32(0.5), ys.astype(f32) + f32(0.5)
    with np.errstate(all='ignore'):
        c2 = (H[6] * u + H[7] * w) + H[8]
        cx = ((H[0] * u + H[1] * w) + H[2]) / c2
        cy = ((H[3] * u + H[4] * w) + H[5]) / c2
        ok = (c2 > 0) & (cx >= 0) & (cx < f32(ws)) & (cy >= 0) & (cy < f32(hs))
        s = np.zeros(xs.shape, f32)
        s2 = np.zeros(xs.shape, f32)
        cr = np.zeros(xs.shape, f32)
        n = 0
        for l in _offsets(v.radius, v.step):
            pv = w + f32(l)
            for k in _offsets(v.radius, v.step):
                pu = u + f32(k)
                h2 = (H[6] * pu + H[7] * pv) + H[8]
                X = ((H[0] * pu + H[1] * pv) + H[2]) / h2
                Y = ((H[3] * pu + H[4] * pv) + H[5]) / h2
                val = bilinear(src, X, Y)
                ref = v.g[np.clip(ys + l, 0, v.h - 1), np.clip(xs + k, 0, v.w - 1)]
                s = s + val
                s2 = s2 + val * val
                cr = cr + ref * val
                n += 1
        fn = f32(n)
        ms = s / fn
        vs = s2 / fn - ms * ms
        ok &= vs >= MIN_VAR
        cov = cr / fn - mr * ms
        c = np.fmin(np.fmax(f32(1) - cov / np.sqrt(vr * vs), f32(0)), NO_COST)
    return np.where(ok, c, NO_COST).astype(f32)


def plane_cost(v, xs, ys, d, n0, n1, n2):
    """Aggregate cost of the planes (d, n) at the pixels (xs, ys) (arrays)."""
    rx, ry = v.ray(xs, ys)
    st = v.stats[ys, xs]
    mr, vr = st[..., 0], st[..., 1]
    with np.errstate(all='ignore'):
        q = d * ((n0 * rx + n1 * ry) + n2)
        m = ((n0 * v.ifx) / q, (n1 * v.ify) / q, ((n0 * v.ocx + n1 * v.ocy) + n2) / q)
        b0 = np.full(xs.shape, NO_COST)
        b1, b2 = b0.copy(), b0.copy()
        for j in range(len(v.src)):
            A, b = v.geo[j, :9], v.geo[j, 9:]
            H = [A[3 * r + c] + b[r] * m[c] for r in range(3) for c in range(3)]
            c = source_cost(v, j, H, xs, ys, mr, vr)
            l0, l1, l2 = c < b0, c < b1, c < b2
            nb2 = np.where(l0 | l1, b1, np.where(l2, c, b2))
            nb1 = np.where(l0, b0, np.where(l1, c, b1))
            b0, b1, b2 = np.where(l0, c, b0), nb1, nb2
        out = ((b0 + b1) + b2) / f32(3) if len(v.src) >= BEST else (b0 + b1) / f32(2)
    return np.where(vr >= MIN_VAR, out, NO_COST).astype(f32)


def random_plane(v, key, dim0, rx, ry):
    lo, hi = f32(1) / v.dmax, f32(1) / v.dmin
    d = f32(1) / (lo + uniform(key, dim0) * (hi - lo))
    a, b, c = (f32(2) * uniform(key, dim0 + k) - f32(1) for k in (1, 2, 3))
    nn = (a * a + b * b) + c * c
    zero = ~(nn > 0)
    with np.errstate(all='ignore'):
        l = np.sqrt(nn)
        a, b, c = np.where(zero, f32(0), a / l), np.where(zero, f32(0), b / l), np.where(zero, f32(-1), c / l)
    den = (a * rx + b * ry) + c
    flip, bad = den > 0, ~(den > 0) & ~(den < 0)
    a = np.where(flip, -a, np.where(bad, f32(0), a))
    b = np.where(flip, -b, np.where(bad, f32(0), b))
    c = np.where(flip, -c, np.where(bad, f32(-1), c))
    return np.stack([d, a, b, c], -1).astype(f32)


def init(v):
    """(planes [h,w,4], cost [h,w]) of nero_mvs_init."""
    ys, xs = np.mgrid[0:v.h, 0:v.w]
    rx, ry = v.ray(xs, ys)
    p = random_plane(v, stream_key(v.seed, v.view, 0, ys * v.w + xs), 0, rx, ry)
    return p, plane_cost(v, xs, ys, p[..., 0], p[..., 1], p[..., 2], p[..., 3])


def pass_(v, planes, cost, it, colour):
    """nero_mvs_pass on copies of (planes, cost)."""
    planes, cost = planes.copy(), cost.copy()
    ys, xs = np.nonzero(((np.arange(v.h)[:, None] + np.arange(v.w)[None, :]) & 1) == colour)
    rx, ry = v.ray(xs, ys)
    cur = planes[ys, xs]
    best, best_c = cur.copy(), cost[ys, xs].copy()

    def consider(ok, p):
        nonlocal best, best_c
        safe = np.where(ok[:, None], p, cur)
        c = plane_cost(v, xs, ys, safe[:, 0], safe[:, 1], safe[:, 2], safe[:, 3])
        upd = ok & (c < best_c)
        best = np.where(upd[:, None], safe, best)
        best_c = np.where(upd, c, best_c)

    for k in range(8):
        dist = 1 if k < 4 else 5
        sgn = dist if k & 1 else -dist
        xn, yn = (xs, ys + sgn) if k & 2 else (xs + sgn, ys)
        inb = (xn >= 0) & (xn < v.w) & (yn >= 0) & (yn < v.h)
        pn = planes[np.clip(yn, 0, v.h - 1), np.clip(xn, 0, v.w - 1)]
        rxn, ryn = v.ray(xn, yn)
        with np.errstate(all='ignore'):
            qn = pn[:, 0] * ((pn[:, 1] * rxn + pn[:, 2] * ryn) + pn[:, 3])
            den = (pn[:, 1] * rx + pn[:, 2] * ry) + pn[:, 3]
            d = qn / den
        ok = inb & (den < 0) & (d >= v.dmin) & (d <= v.dmax)
        consider(ok, np.stack([d, pn[:, 1], pn[:, 2], pn[:, 3]], -1).astype(f32))
    key = stream_key(v.seed, v.view, 1 + 2 * it + colour, ys * v.w + xs)
    lo, hi = f32(1) / v.dmax, f32(1) / v.dmin
    with np.errstate(all='ignore'):
        idp = f32(1) / cur[:, 0] + (f32(2) * uniform(key, 0) - f32(1)) * ((hi - lo) * f32(2.0 ** -(it + 2)))
        d = f32(1) / idp
    consider((d >= v.dmin) & (d <= v.dmax), np.stack([d, cur[:, 1], cur[:, 2], cur[:, 3]], -1).astype(f32))
    sc = f32(2.0 ** -(it + 1))
    a, b, c = (cur[:, k] + (f32(2) * uniform(key, k) - f32(1)) * sc for k in (1, 2, 3))
    nn = (a * a + b * b) + c * c
    with np.errstate(all='ignore'):
        l = np.sqrt(nn)
        a, b, c = a / l, b / l, c / l
        ok = (nn > 0) & (((a * rx + b * ry) + c) < 0)
    consider(ok, np.stack([cur[:, 0], a, b, c], -1).astype(f32))
    consider(np.ones(xs.shape, bool), random_plane(v, key, 4, rx, ry))
    planes[ys, xs] = best
    cost[ys, xs] = best_c
    return planes, cost


def patchmatch(v, iterations):
    """[(planes, cost)] after the initialisation and after every pass."""
    out = [init(v)]
    for it in range(iterations):
        for colour in (0, 1):
            out.append(pass_(v, *out[-1], it, colour))
    return out


def geometric_filter(K, planes, cost, src, geo, max_cost, reproj2, rel_depth, cos_max, min_consistent):
    """(depth fp32 [h,w], count int32 [h,w]) of nero_mvs_filter; src: [(planes_j, cost_j)], geo [S,28] fp64."""
    h, w = cost.shape
    fx, fy, cx, cy = (float(K[0][0]), float(K[1][1]), float(K[0][2]), float(K[1][2]))
    ys, xs = np.mgrid[0:h, 0:w]
    d = planes[..., 0].astype(np.float64)
    n = planes[..., 1:].astype(np.float64)
    u, vv = xs + 0.5, ys + 0.5
    X = [d * ((u - cx) / fx), d * ((vv - cy) / fy), d]
    test = cost.astype(np.float64) <= max_cost
    agree = np.zeros((h, w), np.int32)

    def rigid(g, x):
        return [((g[3 * r] * x[0] + g[3 * r + 1] * x[1]) + g[3 * r + 2] * x[2]) + g[9 + r] for r in range(3)]

    with np.errstate(all='ignore'):
        for j, (pj, cj) in enumerate(src):
            g = geo[j]
            hj, wj = cj.shape
            Y = rigid(g, X)
            pu = g[24] * (Y[0] / Y[2]) + g[26]
            pv = g[25] * (Y[1] / Y[2]) + g[27]
            ok = test & (Y[2] > 0) & (pu >= 0) & (pu < wj) & (pv >= 0) & (pv < hj)
            px = np.where(ok, np.floor(pu), 0).astype(np.int64)
            py = np.where(ok, np.floor(pv), 0).astype(np.int64)
            ok &= cj[py, px].astype(np.float64) <= max_cost
            q = pj[py, px].astype(np.float64)
            dj = q[..., 0]
            Z = [dj * ((px + 0.5 - g[26]) / g[24]), dj * ((py + 0.5 - g[27]) / g[25]), dj]
            W = rigid(g[12:], Z)
            ok &= W[2] > 0
            eu = (fx * (W[0] / W[2]) + cx) - u
            ev = (fy * (W[1] / W[2]) + cy) - vv
            m = [(g[12 + 3 * r] * q[..., 1] + g[13 + 3 * r] * q[..., 2]) + g[14 + 3 * r] * q[..., 3] for r in range(3)]
            cosv = (n[..., 0] * m[0] + n[..., 1] * m[1]) + n[..., 2] * m[2]
            ok &= (eu * eu + ev * ev <= reproj2) & (np.abs(W[2] - d) <= rel_depth * d) & (cosv >= cos_max)
            agree += ok.astype(np.int32)
    return np.where(agree >= min_consistent, planes[..., 0], f32(0)).astype(f32), agree


def unproject(depth, K, pose):
    """World points of the pixels with depth > 0 at their centres, row-major, fp64 (what depth_to_points_cuda computes
    from the centred K, before its fp32 output)."""
    ys, xs = np.nonzero(depth > 0)
    K = np.asarray(K, np.float64)
    d = depth[ys, xs].astype(np.float64)
    Xc = np.stack([(xs + 0.5 - K[0, 2]) / K[0, 0] * d, (ys + 0.5 - K[1, 2]) / K[1, 1] * d, d], -1)
    P = np.asarray(pose, np.float64)
    return (Xc - P[:, 3]) @ P[:, :3]


# ------------------------------------------------------------------------------------------------ synthetic project
BOX_HALF, BOX_H = 0.15, 1.0
SPHERE_H, SPHERE_R = 1.3, 0.3
TABLE_R = 1.8
TINTS = np.asarray([[1.0, 0.85, 0.7], [0.7, 0.9, 1.0], [0.9, 1.0, 0.8]])


def frame():
    """(up, e1, e2, o) of nero_oracle_objprep.scene: the table's normal, two axes in it and the point under the object."""
    up = np.asarray([0.21, -0.33, 0.92])
    up /= np.linalg.norm(up)
    e1 = np.cross(up, [1.0, 0.0, 0.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(up, e1)
    return up, e1, e2, np.asarray([1.3, -0.7, 2.1])


def _lattice(i, j, k):
    with np.errstate(over='ignore'):
        h = _mix(i.astype(np.int64).astype(np.uint32) * np.uint32(0x8da6b343))
        h = _mix(h ^ (j.astype(np.int64).astype(np.uint32) * np.uint32(0xd8163841)))
        h = _mix(h ^ (k.astype(np.int64).astype(np.uint32) * np.uint32(0xcb1ab31f)))
    return (h >> np.uint32(8)).astype(np.float64) / 2.0 ** 24


def value_noise(p, cell):
    """Trilinear value noise with smoothstep weights on a lattice of spacing cell, in [0, 1)."""
    q = p / cell
    f = np.floor(q)
    t = q - f
    t = t * t * (3 - 2 * t)
    i = f.astype(np.int64)
    out = 0.0
    for dx in (0, 1):
        for dy in (0, 1):
            for dz in (0, 1):
                wgt = (t[:, 0] if dx else 1 - t[:, 0]) * (t[:, 1] if dy else 1 - t[:, 1]) * (t[:, 2] if dz else 1 - t[:, 2])
                out = out + wgt * _lattice(i[:, 0] + dx, i[:, 1] + dy, i[:, 2] + dz)
    return out


def albedo(p, surface, cell):
    a = 0.1 + 0.85 * (0.65 * value_noise(p, cell) + 0.35 * value_noise(p + 17.0, cell / 2))
    return a[:, None] * TINTS[np.maximum(surface, 0)]


def render(pose, K, w, h, cell=0.03):
    """Ray cast of the scene through the pixel centres -> dict(rgb uint8 [h,w,3], depth fp64 [h,w] (z-depth, 0 on a miss),
    normal fp64 [h,w,3] (world), surface int [h,w] (-1 none, 0 table, 1 box, 2 sphere)).  No shading: the images are
    photo-consistent."""
    up, e1, e2, o = frame()
    P = np.asarray(pose, np.float64)
    R, t = P[:, :3], P[:, 3]
    C = -R.T @ t
    ys, xs = np.mgrid[0:h, 0:w]
    pc = np.stack([xs + 0.5, ys + 0.5, np.ones_like(xs, dtype=np.float64)], -1).reshape(-1, 3)
    dc = pc @ np.linalg.inv(np.asarray(K, np.float64)).T
    dw = dc @ R                                   # R^T d per ray; its camera z is 1, so the ray parameter is the z-depth
    n = dw.shape[0]
    best = np.full(n, np.inf)
    surf = np.full(n, -1)
    nrm = np.zeros((n, 3))
    with np.errstate(all='ignore'):
        den = dw @ up
        tt = ((o - C) @ up) / den
        hit = C + tt[:, None] * dw - o
        rad = np.linalg.norm(hit - (hit @ up)[:, None] * up, axis=1)
        ok = (tt > 0) & (rad <= TABLE_R)
        upd = ok & (tt < best)
        best[upd], surf[upd], nrm[upd] = tt[upd], 0, up
        B = np.stack([e1, e2, up])
        cl, dl = B @ (C - o), dw @ B.T
        lo, hi = np.asarray([-BOX_HALF, -BOX_HALF, 0.0]), np.asarray([BOX_HALF, BOX_HALF, BOX_H])
        t1, t2 = (lo - cl) / dl, (hi - cl) / dl
        tmin, tmax = np.minimum(t1, t2), np.maximum(t1, t2)
        tn, tf = tmin.max(1), tmax.min(1)
        ax = tmin.argmax(1)
        ok = (tn <= tf) & (tn > 0)
        upd = ok & (tn < best)
        sgn = -np.sign(dl[np.arange(n), ax])
        best[upd], surf[upd] = tn[upd], 1
        nrm[upd] = sgn[upd, None] * B[ax[upd]]
        sc = o + SPHERE_H * up
        oc = C - sc
        a = (dw * dw).sum(1)
        b = dw @ oc
        disc = b * b - a * (oc @ oc - SPHERE_R ** 2)
        ts = (-b - np.sqrt(disc)) / a
        ok = (disc >= 0) & (ts > 0)
        upd = ok & (ts < best)
        best[upd], surf[upd] = ts[upd], 2
        nrm[upd] = (C + ts[upd, None] * dw[upd] - sc) / SPHERE_R
    hitp = C + np.where(np.isfinite(best), best, 0)[:, None] * dw
    rgb = np.zeros((n, 3))
    m = surf >= 0
    rgb[m] = albedo(hitp[m], surf[m], cell)
    return dict(rgb=np.clip(np.round(rgb * 255), 0, 255).astype(np.uint8).reshape(h, w, 3),
                depth=np.where(m, best, 0.0).reshape(h, w), normal=nrm.reshape(h, w, 3), surface=surf.reshape(h, w))


def surface_distance(p):
    """Unsigned distance of points [n,3] to the scene's surfaces (table disc, box, sphere)."""
    up, e1, e2, o = frame()
    q = (np.asarray(p, np.float64) - o) @ np.stack([e1, e2, up]).T
    rad = np.linalg.norm(q[:, :2], axis=1)
    table = np.sqrt(np.maximum(rad - TABLE_R, 0) ** 2 + q[:, 2] ** 2)
    c = np.abs(q - [0.0, 0.0, BOX_H / 2]) - [BOX_HALF, BOX_HALF, BOX_H / 2]
    box = np.linalg.norm(np.maximum(c, 0), axis=1) + np.abs(np.minimum(c.max(1), 0))
    sphere = np.abs(np.linalg.norm(q - [0.0, 0.0, SPHERE_H], axis=1) - SPHERE_R)
    return np.minimum(np.minimum(table, box), sphere)


def object_bbox():
    """World axis-aligned bounding box (lo [3], hi [3]) of the box and the sphere."""
    up, e1, e2, o = frame()
    corners = [o + a * e1 + b * e2 + hh * up for a in (-BOX_HALF, BOX_HALF) for b in (-BOX_HALF, BOX_HALF) for hh in (0.0, BOX_H)]
    sc = o + SPHERE_H * up
    pts = np.asarray(corners + [sc - SPHERE_R, sc + SPHERE_R])
    return pts.min(0), pts.max(0)


def _render_job(a):
    return render(*a)


def project(root, n_views, w, h, seed=0, fmt='bin', per_view=60, cell=0.03, focal=0.9, workers=1):
    """Write a synthetic project: <root>/images/img_XXX.png and the COLMAP model <root>/sparse/0 (PINHOLE f = focal w,
    tracks of sparse points sampled on the visible surfaces).  -> dict(names, poses [n,3,4] (fp64), K, truth (render()
    dicts in name order), up, center).  workers > 1 renders the views in that many processes."""
    import cv2
    sc = OOp.scene(n_table=10, n_obj=10, outlier_frac=0.0, n_cams=n_views, seed=seed)
    poses = sc['poses']
    K = np.asarray([[focal * w, 0, w / 2], [0, focal * w, h / 2], [0, 0, 1]], np.float64)
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    names = [f'img_{i:03d}.png' for i in range(n_views)]
    jobs = [(P, K, w, h, cell) for P in poses]
    if workers > 1:
        import multiprocessing
        with multiprocessing.get_context('fork').Pool(workers) as pool:
            truth = pool.map(_render_job, jobs)
    else:
        truth = [render(*a) for a in jobs]
    for name, tr in zip(names, truth):
        cv2.imwrite(os.path.join(root, 'images', name), np.ascontiguousarray(tr['rgb'][..., ::-1]))
    rng = np.random.RandomState(seed + 1)
    pts = []
    for P, tr in zip(poses, truth):
        ys, xs = np.nonzero(tr['depth'] > 0)
        sel = rng.choice(ys.shape[0], min(per_view, ys.shape[0]), replace=False)
        d = tr['depth'][ys[sel], xs[sel]]
        Xc = np.stack([(xs[sel] + 0.5 - K[0, 2]) / K[0, 0] * d, (ys[sel] + 0.5 - K[1, 2]) / K[1, 1] * d, d], -1)
        pts.append((Xc - P[:, 3]) @ P[:, :3])
    pts = np.concatenate(pts, 0)
    obs = {i: [] for i in range(n_views)}
    points = {}
    for pid, X in enumerate(pts):
        track = []
        for i, (P, tr) in enumerate(zip(poses, truth)):
            x = K @ (P[:, :3] @ X + P[:, 3])
            if x[2] <= 0:
                continue
            u, v = x[0] / x[2], x[1] / x[2]
            if not (0 <= u < w and 0 <= v < h):
                continue
            dt = tr['depth'][int(v), int(u)]
            if dt > 0 and abs(dt - x[2]) <= 0.01 * x[2]:
                track.append((i, len(obs[i])))
                obs[i].append(((u, v), pid + 1))
        if len(track) >= 2:
            points[pid + 1] = (X, [128, 128, 128], 0.5, [1 + i for i, _ in track], [k for _, k in track])
    images = {}
    for i, (P, name) in enumerate(zip(poses, names)):
        xys = np.asarray([o[0] for o in obs[i]]).reshape(-1, 2)
        p3d = np.asarray([o[1] if o[1] in points else -1 for o in obs[i]], np.int64)
        images[1 + i] = (OOp.rotmat2qvec(P[:, :3]), P[:, 3], 1, name, xys, p3d)
    cams = {1: ('PINHOLE', w, h, [K[0, 0], K[1, 1], K[0, 2], K[1, 2]])}
    OOp.write_colmap_model(os.path.join(root, 'sparse', '0'), cams, images, points, fmt)
    return dict(names=names, poses=poses, K=K, truth=truth, up=sc['up'], center=sc['center'])
