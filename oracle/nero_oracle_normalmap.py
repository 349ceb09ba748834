"""numpy restatement of the normal-map bake (nero_b200/normalmap.py, k_normalmap.cu) and of relighting with the map
(nero_relight_render_textured_nmap in k_relight.cu) for the tests.

  vertex_normals  per vertex, -cross(e1, e2) of its triangles summed in ascending triangle order in float32 (every operation
                  rounded on its own, as numpy rounds them), then s / sqrt((x x + y y) + z z); a zero sum gives 0.  Bit for
                  bit the kernel's.
  bake            nero_oracle_texmap's rasteriser and fp32 interpolation for the texel points, the cage direction in
                  float32, and the cage ray cast in float64 by exhaustive Moeller-Trumbore over the detail mesh (the
                  arithmetic of nero_oracle_relight.trace) with t in (0, 2 distance).  Texels whose ray is a near tie -- another
                  triangle within TIE_T of the closest t whose normal differs, or a hit within TIE_T of either end of the t
                  range or within TIE_UV of a triangle's edge at the mesh's hit/miss boundary -- are flagged: there the fp32
                  traversal may pick the other answer.
  surface / shade / render
                  nero_oracle_relight_tex's path tracer with the shading rule of include/nero_normalmap.h:
                    n_g = the flat outward normal flipped to face the ray; n_s = the filtered map normal normalised and
                    flipped by the same sign (n_g when its length is below 1e-6, or when dot(n_s, wo) <= 0);
                    the BRDF, its pdf and both lobe samplers use n_s; a light or continuation direction with
                    dot(n_g, l) <= 0 carries nothing and a continuation of that kind ends the path; offsets along n_g.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np

import nero_oracle_relight as OR
import nero_oracle_relight_tex as ORT
import nero_oracle_texmap as OT

TIE_T = 1e-5
TIE_UV = 1e-6
MIN_LEN = 1e-6


# ------------------------------------------------------------------------------------------------ encoding
def encode(n):
    n = np.asarray(n, np.float32)
    k = np.floor((n * np.float32(0.5) + np.float32(0.5)) * np.float32(255) + np.float32(0.5))
    return np.clip(k, 0, 255).astype(np.uint8)


def decode(k):
    return (2.0 * np.asarray(k, np.float64) / 255.0 - 1.0).astype(np.float32)


# ------------------------------------------------------------------------------------------------ vertex normals
def normalize32(s):
    """s / |s| in float32 with |s| = sqrt((x x + y y) + z z); zero rows stay zero."""
    s = np.asarray(s, np.float32)
    l2 = (s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2]
    ok = l2 > 0
    out = np.zeros_like(s)
    out[ok] = s[ok] / np.sqrt(l2[ok])[:, None]
    return out


def face_areas32(verts, tris):
    """-cross(v1 - v0, v2 - v0) per triangle in float32, component by component."""
    V = np.asarray(verts, np.float32)
    T = np.asarray(tris, np.int64)
    e1, e2 = V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    return np.stack([-(e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]), -(e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]),
                     -(e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0])], -1)


def vertex_normals(verts, tris):
    """-> float32 [V,3], the kernel's bits."""
    V = np.asarray(verts).shape[0]
    T = np.asarray(tris, np.int64)
    a = face_areas32(verts, T)
    flat = T.reshape(-1)
    order = np.argsort(flat, kind='stable')               # each vertex's corners in ascending triangle order
    vert, tri = flat[order], order // 3
    cnt = np.bincount(flat, minlength=V)
    start = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    rank = np.arange(flat.size) - start[vert]
    s = np.zeros((V, 3), np.float32)
    for k in range(int(cnt.max()) if cnt.size else 0):
        m = rank == k
        s[vert[m]] = s[vert[m]] + a[tri[m]]
    return normalize32(s)


# ------------------------------------------------------------------------------------------------ bake
def cast(dverts, dtris, o, d, t_max):
    """Closest hit in (0, t_max) by exhaustive Moeller-Trumbore in float64 -> (tri or -1, t, u, v, tie)."""
    V = np.asarray(dverts, np.float64)
    T = np.asarray(dtris, np.int64)
    chunk = max(1, (1 << 20) // T.shape[0])
    v0, e1, e2 = V[T[:, 0]], V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    dn = vertex_normals(dverts, dtris).astype(np.float64)
    n = o.shape[0]
    tri, tt, uu, vv, tie = np.full(n, -1), np.zeros(n), np.zeros(n), np.zeros(n), np.zeros(n, bool)
    for c0 in range(0, n, chunk):
        oc, dc = o[c0:c0 + chunk, None], d[c0:c0 + chunk, None]
        pv = np.cross(dc, e2[None])
        det = OR.dot(e1[None], pv)
        ok = np.abs(det) > 1e-12
        inv = 1.0 / np.where(ok, det, 1.0)
        tv = oc - v0[None]
        u = OR.dot(tv, pv) * inv
        qv = np.cross(tv, e1[None])
        v = OR.dot(dc, qv) * inv
        t = OR.dot(e2[None], qv) * inv
        strict = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 0) & (t < t_max)
        loose = ok & (u >= -TIE_UV) & (v >= -TIE_UV) & (u + v <= 1 + TIE_UV) & (t > -TIE_T) & (t < t_max + TIE_T)
        ts = np.where(strict, t, np.inf)
        k = ts.argmin(1)
        r = np.arange(k.shape[0])
        hit = np.isfinite(ts[r, k])
        tb = ts[r, k]
        # another candidate (edges loosened by TIE_UV, t by TIE_T) as close as the closest hit, with a different normal
        near = loose & (np.abs(t - tb[:, None]) < TIE_T)
        t_tie = np.zeros(k.shape[0], bool)
        for i in np.nonzero(near.sum(1) > 1)[0]:
            ks = np.nonzero(near[i])[0]
            wk = np.stack([1 - u[i, ks] - v[i, ks], u[i, ks], v[i, ks]], -1)[..., None]
            nk = OR.normalize((wk * dn[T[ks]]).sum(1))
            t_tie[i] = (np.linalg.norm(nk - nk[ks == k[i]], axis=-1) > 1e-4).any()
        end_tie = hit & ((tb < TIE_T) | (tb > t_max - TIE_T))
        edge_tie = (~hit & loose.any(1)) | (hit & (loose & ~strict & (t < tb[:, None] + TIE_T)).any(1))
        s = slice(c0, c0 + chunk)
        tri[s], tt[s] = np.where(hit, k, -1), np.where(hit, tb, 0.0)
        uu[s], vv[s] = np.where(hit, u[r, k], 0.0), np.where(hit, v[r, k], 0.0)
        tie[s] = t_tie | end_tie | edge_tie
    return tri, tt, uu, vv, tie


def bake_texels(verts, tris, vt, ft, dverts, dtris, width, height, distance=0.02):
    """Per covered texel in row-major order -> dict texel [n] (row-major index), point / cage [n,3] float32 (the kernel's
    bits), hit [n] bool, tie [n] bool, t [n] (the hit's ray parameter, 0 for a miss), normal [n,3] float64 (the cage direction where the ray misses), img [h,w,5] uint8
    (the bytes before inpainting)."""
    owner, _, bary = OT.rasterize(vt, ft, width, height)
    m = owner >= 0
    texel = np.nonzero(m.reshape(-1))[0]
    point = OT.interpolate(verts, tris, owner, bary)[m]
    ln = vertex_normals(verts, tris)
    cage = normalize32(OT.interpolate(ln, tris, owner, bary)[m])
    d32 = np.float32(distance)
    o = point + d32 * cage
    tri, t, u, v, tie = cast(dverts, dtris, o.astype(np.float64), -cage.astype(np.float64), 2.0 * float(d32))
    hit = tri >= 0
    dn = vertex_normals(dverts, dtris).astype(np.float64)
    T = np.asarray(dtris, np.int64)
    w = np.stack([1 - u - v, u, v], -1)[..., None]
    normal = np.where(hit[:, None], OR.normalize((w * dn[T[np.maximum(tri, 0)]]).sum(1)), cage.astype(np.float64))
    img = np.zeros((height * width, 5), np.uint8)
    img[texel, :3] = encode(normal)
    return dict(texel=texel, point=point, cage=cage, hit=hit, tie=tie, t=t, normal=normal, img=img.reshape(height, width, 5),
                owner=owner)


def bake(verts, tris, vt, ft, dverts, dtris, size, ssaa=2, distance=0.02):
    """normalmap.bake restated -> (img uint8 [h0,w0,3], stats, bake_texels' dict)."""
    h0, w0 = (size, size) if np.isscalar(size) else size
    b = bake_texels(verts, tris, vt, ft, dverts, dtris, w0 * ssaa, h0 * ssaa, distance)
    img, _ = OT.inpaint(b['img'], b['owner'] >= 0)
    if ssaa == 2:
        img = OT.downsample(img)
    n = b['texel'].size
    return img[..., :3], {'covered': n, 'hits': int(b['hit'].sum()), 'misses': n - int(b['hit'].sum())}, b


# ------------------------------------------------------------------------------------------------ relighting with the map
def surface(verts, tris, uv_materials, tri, t, u, v, o, d):
    """-> (hit point, n_g, n_s, albedo, metallic, alpha); uv_materials = (vt, ft, tex [H,W,8] with the map in 5-7)."""
    vt, ft, tex = uv_materials
    V, T = np.asarray(verts, np.float64), np.asarray(tris, np.int64)[tri]
    e1, e2 = V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]]
    n = OR.normalize(-np.cross(e1, e2))
    sign = np.where(OR.dot(n, d) > 0, -1.0, 1.0)[:, None]
    ng = sign * n
    w = np.stack([1 - u - v, u, v], -1)[..., None]
    uv = (np.asarray(vt, np.float64)[np.asarray(ft, np.int64)[tri]] * w).sum(1)
    m = ORT.texture_lookup(tex, uv)
    f = m[:, 5:8]
    ln = np.linalg.norm(f, axis=-1, keepdims=True)
    ns = sign * f / np.maximum(ln, MIN_LEN)
    use = (ln[:, 0] >= MIN_LEN) & (OR.dot(ns, -d) > 0)
    ns = np.where(use[:, None], ns, ng)
    return o + t[:, None] * d, ng, ns, m[:, :3], m[:, 3], m[:, 4]


def shade(ns, ng, v, albedo, metallic, alpha, tables, ggx_smith, rnd, occluded, trace_next):
    """nero_oracle_relight.shade with the BRDF on n_s and the flat-face tests on n_g."""
    ps = OR.spec_prob(albedo, metallic)
    env = tables['env'].reshape(-1, 4).astype(np.float64)[:, :3]
    L = np.zeros_like(ns)
    l, tx, pl = OR.sample_env(tables, np.stack([rnd(2), rnd(3), rnd(4), rnd(5)], -1))
    NoL = OR.dot(ns, l)
    ok = (NoL > 0) & (pl > 0) & (OR.dot(ng, l) > 0)
    f = OR.brdf(ns, v, l, albedo, metallic, alpha, ggx_smith)
    vis = ok & ~occluded(ok, l)
    pb = OR.bsdf_pdf(ns, v, l, alpha, ps)
    w = np.where(vis, OR.mis(pl, pb) * NoL / np.where(vis, pl, 1.0), 0.0)
    L += f * env[tx] * w[:, None]
    r1, r2 = rnd(7), rnd(8)
    l = np.where((rnd(6) < ps)[:, None], OR.sample_ggx(ns, v, alpha, r1, r2), OR.sample_diffuse(ns, r1, r2))
    l = OR.normalize(l)
    pb = OR.bsdf_pdf(ns, v, l, alpha, ps)
    go = (pb > 0) & (OR.dot(ng, l) > 0)
    f = OR.brdf(ns, v, l, albedo, metallic, alpha, ggx_smith)
    thr = np.where(go[:, None], f * OR.dot(ns, l)[:, None] / np.where(go, pb, 1.0)[:, None], 0.0)
    hit, state = trace_next(go, l)
    esc = go & ~hit
    tx, pl = OR.env_lookup_pdf(tables, l)
    L += thr * env[tx] * np.where(esc, OR.mis(pb, pl), 0.0)[:, None]
    return L, thr, l, go & hit, state


def render(verts, tris, uv_materials, tables, pose, K, h, w, spp, max_bounces=4, seed=0, ggx_smith=0, spp0=0):
    """The normal-mapped kernel's image [h,w,4]: nero_oracle_relight_tex.render with this module's surface and shade."""
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
            p, ng, ns, alb, met, alpha = surface(verts, tris, uv_materials, tri, tt, uu, vv, o, d)
            po = p + OR.EPS * ng
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
            Lb, f_thr, l, cont, _ = shade(ns, ng, -d, alb, met, alpha, tables, ggx_smith, rnd, occluded, trace_next)
            acc[idx, :3] += thr * Lb
            thr = thr * f_thr
            if b + 1 >= max_bounces:
                break
            k = np.nonzero(cont)[0]
            tri, tt, uu, vv = (a[k] for a in nxt['res'])
            idx, thr, o, d = idx[k], thr[k], po[k], l[k]
    return (acc / spp).reshape(h, w, 4)
