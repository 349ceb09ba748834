"""CPU oracle of relighting from UV textures (nero_relight_render_textured in nero_b200/csrc/k_relight.cu) in numpy float64.

TEST INFRASTRUCTURE ONLY.  The path tracer is nero_oracle_relight's: the same random numbers, environment sampler, BRDF,
shading step and exhaustive ray casts.  Only the materials at a hit differ: the uv is interpolated barycentrically and the
texture is looked up bilinearly with wrapping (texture_lookup), and alpha is the filtered roughness itself, not its square.
"""
import numpy as np

import nero_oracle_relight as OR


def texture_lookup(tex, uv):
    """Bilinear, wrapping lookup of tex [H,W,C] (row 0 at the top of the image) at uv [...,2] with v = 0 at the bottom row:
    s = u W - 1/2, t = (1 - v) H - 1/2, taps floor(s), floor(s) + 1 (likewise t) taken modulo the size, and the lerp form
    a + f (b - a) along x, then along y."""
    tex = np.asarray(tex, np.float64)
    H, W = tex.shape[:2]
    uv = np.asarray(uv, np.float64)
    s, t = uv[..., 0] * W - 0.5, (1 - uv[..., 1]) * H - 0.5
    x0, y0 = np.floor(s), np.floor(t)
    fx, fy = (s - x0)[..., None], (t - y0)[..., None]
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    g = lambda y, x: tex[np.mod(y, H), np.mod(x, W)]
    lerp = lambda a, b, f: a + f * (b - a)
    return lerp(lerp(g(y0, x0), g(y0, x0 + 1), fx), lerp(g(y0 + 1, x0), g(y0 + 1, x0 + 1), fx), fy)


def surface(verts, tris, uv_materials, tri, t, u, v, o, d):
    """nero_oracle_relight.surface with materials from UV textures: uv_materials = (vt [N,2], ft [T,3], tex [H,W,8]).
    -> (hit point, two-sided outward face normal, albedo, metallic, alpha = filtered roughness)."""
    vt, ft, tex = uv_materials
    V, T = np.asarray(verts, np.float64), np.asarray(tris, np.int64)[tri]
    e1, e2 = V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    n = OR.normalize(-np.cross(e1, e2))
    n = np.where((OR.dot(n, d) > 0)[:, None], -n, n)
    w = np.stack([1 - u - v, u, v], -1)[..., None]
    uv = (np.asarray(vt, np.float64)[np.asarray(ft, np.int64)[tri]] * w).sum(1)
    m = texture_lookup(tex, uv)
    return o + t[:, None] * d, n, m[:, :3], m[:, 3], m[:, 4]


def render(verts, tris, uv_materials, tables, pose, K, h, w, spp, max_bounces=4, seed=0, ggx_smith=0, spp0=0):
    """The textured kernel's image [h,w,4] (linear premultiplied RGB, alpha) from samples [spp0, spp0 + spp); the loop of
    nero_oracle_relight.render with this module's surface()."""
    pose, K = np.asarray(pose, np.float64), np.asarray(K, np.float64)
    R, t = pose[:, :3], pose[:, 3]
    pix = np.arange(h * w)
    x, y = pix % w, pix // w
    acc = np.zeros((h * w, 4))
    for s in range(spp0, spp0 + spp):
        c = np.stack([(x + OR.uniform(seed, pix, s, 0, 0) - K[0, 2]) / K[0, 0], (y + OR.uniform(seed, pix, s, 0, 1) - K[1, 2]) / K[1, 1],
                      np.ones(h * w)], -1)
        d = OR.normalize(c @ R)
        o = np.broadcast_to(-R.T @ t, d.shape).copy()
        tri, tt, uu, vv = OR.trace(verts, tris, o, d)
        alive = tri >= 0
        acc[:, 3] += alive
        idx = np.nonzero(alive)[0]
        thr = np.ones((idx.size, 3))
        o, d, tri, tt, uu, vv = o[idx], d[idx], tri[idx], tt[idx], uu[idx], vv[idx]
        for b in range(max_bounces):
            if idx.size == 0:
                break
            p, n, alb, met, alpha = surface(verts, tris, uv_materials, tri, tt, uu, vv, o, d)
            po = p + OR.EPS * n
            rnd = lambda dim: OR.uniform(seed, idx, s, b, dim)

            def occluded(mask, l):
                out = np.zeros(mask.shape, bool)
                k = np.nonzero(mask)[0]
                out[k] = OR.trace(verts, tris, po[k], l[k])[0] >= 0
                return out
            nxt = {}

            def trace_next(mask, l):
                res = OR.trace(verts, tris, po, l)
                nxt['res'] = res
                return mask & (res[0] >= 0), None
            Lb, f_thr, l, cont, _ = OR.shade(n, -d, alb, met, alpha, tables, ggx_smith, rnd, occluded, trace_next)
            acc[idx, :3] += thr * Lb
            thr = thr * f_thr
            if b + 1 >= max_bounces:
                break
            k = np.nonzero(cont)[0]
            tri, tt, uu, vv = (a[k] for a in nxt['res'])
            idx, thr, o, d = idx[k], thr[k], po[k], l[k]
    return (acc / spp).reshape(h, w, 4)
