"""CPU oracle of the relighting path tracer (nero_b200/csrc/k_relight.cu, math_relight.cuh) in numpy float64.

TEST INFRASTRUCTURE ONLY.  The same random numbers (the integer hash restated bit for bit), the same float32 environment
tables and binary search, lobe rule, power-heuristic MIS and ray offset as the kernel; closest and any hit by exhaustive
Moeller-Trumbore with barycentrics (the arithmetic of nero_oracle_mat.trace_bruteforce).  Differences from the kernel come
from fp32 versus fp64 arithmetic only.
"""
import numpy as np

EPS = 1e-4              # kRelightEps
MIN_ALPHA = 1e-3        # kRelightMinAlpha
M32 = 0xffffffff
PI = np.pi


# ------------------------------------------------------------------------------------------------ random numbers
def _mix(x):
    x = x ^ (x >> np.uint64(16))
    x = (x * np.uint64(0x85ebca6b)) & np.uint64(M32)
    x = x ^ (x >> np.uint64(13))
    x = (x * np.uint64(0xc2b2ae35)) & np.uint64(M32)
    return x ^ (x >> np.uint64(16))


def uniform(seed, pixel, sample, bounce, dim):
    """rl_uniform: every argument may be an integer array; returns float64 values that are exactly the kernel's float32s."""
    u64 = lambda a: np.asarray(a, np.int64).astype(np.uint64) & np.uint64(M32)
    h = _mix((u64(seed) * np.uint64(0x9e3779b9) + np.uint64(0x7f4a7c15)) & np.uint64(M32))
    h = _mix(h ^ u64(pixel))
    h = _mix(h ^ u64(sample))
    h = _mix(h ^ ((u64(bounce) << np.uint64(8)) | u64(dim)))
    return (h >> np.uint64(8)).astype(np.float64) * (1.0 / 16777216.0)


# ------------------------------------------------------------------------------------------------ environment
def search(cdf, u):
    """rl_search: the j with cdf[j] <= u < cdf[j+1] on the float32 table."""
    cdf = np.asarray(cdf, np.float32).astype(np.float64)
    return np.clip(np.searchsorted(cdf, u, side='right') - 1, 0, cdf.shape[-1] - 2)


def env_dir(u, v):
    u, v = np.broadcast_arrays(np.asarray(u, np.float64), np.asarray(v, np.float64))
    phi, el = (0.5 - u) * 2 * PI, (v - 0.5) * PI
    ce = np.cos(el)
    return np.stack([ce * np.cos(phi), ce * np.sin(phi), np.sin(el)], -1), ce


def env_uv(d):
    return 0.5 - np.arctan2(d[..., 1], d[..., 0]) / (2 * PI), 0.5 + np.arctan2(d[..., 2], np.hypot(d[..., 0], d[..., 1])) / PI


def texel(u, v, W, H):
    i = np.clip((u * W).astype(np.int64), 0, W - 1)
    j = np.clip((v * H).astype(np.int64), 0, H - 1)
    return j * W + i


def env_pdf(p_texel, W, H, ce):
    return p_texel * W * H / (2 * PI * PI * np.maximum(ce, 1e-12))


def sample_env(tables, r):
    """r [...,4] uniforms -> (direction, texel index, solid-angle pdf)."""
    H, W = tables['p'].shape
    j = search(tables['cdf_rows'], r[..., 0])
    rows = np.asarray(tables['cdf_cols'], np.float32).astype(np.float64)[j]
    i = (rows <= r[..., 1:2]).sum(-1) - 1
    i = np.clip(i, 0, W - 1)
    d, ce = env_dir((i + r[..., 2]) / W, (j + r[..., 3]) / H)
    tx = j * W + i
    return d, tx, env_pdf(tables['p'].reshape(-1).astype(np.float64)[tx], W, H, ce)


def env_lookup_pdf(tables, d):
    H, W = tables['p'].shape
    u, v = env_uv(d)
    tx = texel(u, v, W, H)
    return tx, env_pdf(tables['p'].reshape(-1).astype(np.float64)[tx], W, H, np.hypot(d[..., 0], d[..., 1]))


# ------------------------------------------------------------------------------------------------ BRDF and its sampler
def dot(a, b):
    return (a * b).sum(-1)


def normalize(a):
    return a / np.maximum(np.linalg.norm(a, axis=-1, keepdims=True), 1e-12)


def frame(z):
    """mc_frame (math_mc.cuh; get_orthogonal_directions, field.py:755-772)."""
    zero = np.zeros_like(z[..., 0])
    o0 = np.stack([z[..., 1], -z[..., 0], zero], -1)
    o1 = np.stack([-z[..., 2], zero, z[..., 0]], -1)
    n0, n1 = np.linalg.norm(o0, axis=-1), np.linalg.norm(o1, axis=-1)
    pick = (n0 > n1)[..., None]
    x = np.where(pick, o0, o1) / np.maximum(np.where(pick[..., 0], n0, n1), 1e-12)[..., None]
    return x, np.cross(z, x)


def luminance(c):
    return 0.2126 * c[..., 0] + 0.7152 * c[..., 1] + 0.0722 * c[..., 2]


def spec_prob(albedo, metallic):
    m1 = 1.0 - metallic
    f0 = 0.04 * m1[..., None] + metallic[..., None] * albedo
    kd, ks = luminance(albedo) * m1, luminance(f0)
    return np.where(kd > 0, np.maximum(ks / np.where(kd > 0, kd + ks, 1.0), 0.25), 1.0)


def sample_diffuse(n, r1, r2):
    x, y = frame(n)
    phi, st, ct = 2 * PI * r1, np.sqrt(r2), np.sqrt(1 - r2)
    return (np.cos(phi) * st)[..., None] * x + (np.sin(phi) * st)[..., None] * y + ct[..., None] * n


def sample_ggx(n, v, alpha, r1, r2):
    a = np.maximum(alpha, MIN_ALPHA)
    x, y = frame(n)
    phi = 2 * PI * r1
    ct = np.sqrt((1 - r2) / (1 + (a * a - 1) * r2))
    st = np.sqrt(np.maximum(1 - ct * ct, 0))
    h = (np.cos(phi) * st)[..., None] * x + (np.sin(phi) * st)[..., None] * y + ct[..., None] * n
    return 2 * dot(v, h)[..., None] * h - v


def bsdf_pdf(n, v, l, alpha, ps):
    NoL = dot(n, l)
    h = normalize(v + l)
    NoH, VoH = np.clip(dot(n, h), 0, 1), np.maximum(dot(v, h), 1e-12)
    a2 = np.maximum(alpha, MIN_ALPHA) ** 2
    D = a2 / (PI * (NoH * NoH * (a2 - 1) + 1) ** 2)
    return np.where(NoL > 0, (1 - ps) * NoL / PI + ps * D * NoH / (4 * VoH), 0.0)


def geometry(NoV, NoL, a, ggx_smith):
    """geometry_term (field.py:869-894, 923-930)."""
    if not ggx_smith:
        k = a / 2
        return NoV / (NoV * (1 - k) + k + 1e-5) * NoL / (NoL * (1 - k) + k + 1e-5)
    a2 = a * a
    lv = 0.5 * np.sqrt(1 + a2 * ((1 - NoV * NoV) / (NoV * NoV + 1e-7))) - 0.5
    ll = 0.5 * np.sqrt(1 + a2 * ((1 - NoL * NoL) / (NoL * NoL + 1e-7))) - 0.5
    return 1 / (1 + lv + ll)


def brdf(n, v, l, albedo, metallic, alpha, ggx_smith):
    """NeRO's stage-II BRDF: albedo (1-m)/pi + F D G / (4 NoV NoL) with distribution_ggx's +1e-4 (field.py:916-921)."""
    NoV, NoL = dot(n, v), dot(n, l)
    h = normalize(v + l)
    NoH, VoH = np.clip(dot(n, h), 0, 1), np.clip(dot(v, h), 0, 1)
    nov, nol = np.minimum(NoV, 1), np.minimum(NoL, 1)
    a2 = alpha * alpha
    D = a2 / (PI * (NoH * NoH * (a2 - 1) + 1) ** 2 + 1e-4)
    with np.errstate(divide='ignore', invalid='ignore'):
        spec = D * geometry(nov, nol, alpha, ggx_smith) / (4 * nov * nol)
    f5 = (1 - VoH) ** 5
    m1 = (1 - metallic)[..., None]
    f0 = 0.04 * m1 + metallic[..., None] * albedo
    f = albedo * m1 / PI + (f0 + (1 - f0) * f5[..., None]) * spec[..., None]
    return np.where(((NoV > 0) & (NoL > 0))[..., None], f, 0.0)


def mis(a, b):
    return a * a / (a * a + b * b)


# ------------------------------------------------------------------------------------------------ geometry
def trace(verts, tris, o, d, t_max=1e30, chunk=2048):
    """Closest hit by exhaustive Moeller-Trumbore -> (triangle index or -1, t, u, v)."""
    V = np.asarray(verts, np.float64)
    T = np.asarray(tris, np.int64)
    v0, e1, e2 = V[T[:, 0]], V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    n = o.shape[0]
    tri, tt, uu, vv = np.full(n, -1), np.full(n, t_max), np.zeros(n), np.zeros(n)
    for c0 in range(0, n, chunk):
        oc, dc = o[c0:c0 + chunk, None], d[c0:c0 + chunk, None]
        pv = np.cross(dc, e2[None])
        det = dot(e1[None], pv)
        ok = np.abs(det) > 1e-12
        inv = 1.0 / np.where(ok, det, 1.0)
        tv = oc - v0[None]
        u = dot(tv, pv) * inv
        qv = np.cross(tv, e1[None])
        v = dot(dc, qv) * inv
        t = dot(e2[None], qv) * inv
        ok = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 0) & (t < t_max)
        t = np.where(ok, t, np.inf)
        k = t.argmin(1)
        r = np.arange(k.shape[0])
        hit = np.isfinite(t[r, k])
        tri[c0:c0 + chunk] = np.where(hit, k, -1)
        tt[c0:c0 + chunk] = np.where(hit, t[r, k], t_max)
        uu[c0:c0 + chunk], vv[c0:c0 + chunk] = np.where(hit, u[r, k], 0), np.where(hit, v[r, k], 0)
    return tri, tt, uu, vv


def surface(verts, tris, vmat, tri, t, u, v, o, d):
    """Hit point, two-sided outward face normal and the barycentrically interpolated materials (albedo, metallic, alpha)."""
    V, T = np.asarray(verts, np.float64), np.asarray(tris, np.int64)[tri]
    e1, e2 = V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    n = normalize(-np.cross(e1, e2))
    n = np.where((dot(n, d) > 0)[:, None], -n, n)
    w = np.stack([1 - u - v, u, v], -1)[..., None]
    m = (np.asarray(vmat, np.float64)[T] * w).sum(1)
    return o + t[:, None] * d, n, m[:, :3], m[:, 3], m[:, 4] ** 2


# ------------------------------------------------------------------------------------------------ estimator
def shade(n, v, albedo, metallic, alpha, tables, ggx_smith, rnd, occluded, trace_next):
    """One interaction of the path tracer at points with side normals n and view directions v.

    rnd(dim) -> uniforms of this bounce; occluded(o, l) -> bool (shadow ray); trace_next(o, l) -> (hit mask, state) for the
    continuation ray.  Returns (NEE + escaping-BSDF radiance per unit throughput, throughput factor, continuation ray, hit
    mask of the continuation, state)."""
    ps = spec_prob(albedo, metallic)
    env = tables['env'].reshape(-1, 4).astype(np.float64)[:, :3]
    L = np.zeros_like(n)
    # next-event estimation
    l, tx, pl = sample_env(tables, np.stack([rnd(2), rnd(3), rnd(4), rnd(5)], -1))
    NoL = dot(n, l)
    ok = (NoL > 0) & (pl > 0)
    f = brdf(n, v, l, albedo, metallic, alpha, ggx_smith)
    vis = ok & ~occluded(ok, l)
    pb = bsdf_pdf(n, v, l, alpha, ps)
    w = np.where(vis, mis(pl, pb) * NoL / np.where(vis, pl, 1.0), 0.0)
    L += f * env[tx] * w[:, None]
    # BRDF sample
    r1, r2 = rnd(7), rnd(8)
    l = np.where((rnd(6) < ps)[:, None], sample_ggx(n, v, alpha, r1, r2), sample_diffuse(n, r1, r2))
    l = normalize(l)
    pb = bsdf_pdf(n, v, l, alpha, ps)
    go = pb > 0
    f = brdf(n, v, l, albedo, metallic, alpha, ggx_smith)
    thr = np.where(go[:, None], f * dot(n, l)[:, None] / np.where(go, pb, 1.0)[:, None], 0.0)
    hit, state = trace_next(go, l)
    esc = go & ~hit
    tx, pl = env_lookup_pdf(tables, l)
    L += thr * env[tx] * np.where(esc, mis(pb, pl), 0.0)[:, None]
    return L, thr, l, go & hit, state


def render(verts, tris, vmat, tables, pose, K, h, w, spp, max_bounces=4, seed=0, ggx_smith=0, spp0=0):
    """The kernel's image [h,w,4] (linear premultiplied RGB, alpha) from samples [spp0, spp0 + spp)."""
    pose, K = np.asarray(pose, np.float64), np.asarray(K, np.float64)
    R, t = pose[:, :3], pose[:, 3]
    pix = np.arange(h * w)
    x, y = pix % w, pix // w
    acc = np.zeros((h * w, 4))
    for s in range(spp0, spp0 + spp):
        c = np.stack([(x + uniform(seed, pix, s, 0, 0) - K[0, 2]) / K[0, 0], (y + uniform(seed, pix, s, 0, 1) - K[1, 2]) / K[1, 1],
                      np.ones(h * w)], -1)
        d = normalize(c @ R)
        o = np.broadcast_to(-R.T @ t, d.shape).copy()
        tri, tt, uu, vv = trace(verts, tris, o, d)
        alive = tri >= 0
        acc[:, 3] += alive
        idx = np.nonzero(alive)[0]
        thr = np.ones((idx.size, 3))
        o, d, tri, tt, uu, vv = o[idx], d[idx], tri[idx], tt[idx], uu[idx], vv[idx]
        for b in range(max_bounces):
            if idx.size == 0:
                break
            p, n, alb, met, alpha = surface(verts, tris, vmat, tri, tt, uu, vv, o, d)
            po = p + EPS * n
            rnd = lambda dim: uniform(seed, idx, s, b, dim)

            def occluded(mask, l):
                out = np.zeros(mask.shape, bool)
                k = np.nonzero(mask)[0]
                out[k] = trace(verts, tris, po[k], l[k])[0] >= 0
                return out
            nxt = {}

            def trace_next(mask, l):
                res = trace(verts, tris, po, l)
                nxt['res'] = res
                return mask & (res[0] >= 0), None
            Lb, f_thr, l, cont, _ = shade(n, -d, alb, met, alpha, tables, ggx_smith, rnd, occluded, trace_next)
            acc[idx, :3] += thr * Lb
            thr = thr * f_thr
            if b + 1 >= max_bounces:
                break
            k = np.nonzero(cont)[0]
            tri, tt, uu, vv = (a[k] for a in nxt['res'])
            idx, thr, o, d = idx[k], thr[k], po[k], l[k]
    return (acc / spp).reshape(h, w, 4)
