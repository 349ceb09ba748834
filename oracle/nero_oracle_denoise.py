"""CPU oracle of the relit-frame denoiser (include/nero_denoise.h, nero_b200/csrc/k_denoise.cu and the AOV instances of
k_relight.cu) in numpy float64.

TEST INFRASTRUCTURE ONLY.  The feature sums trace the camera rays with nero_oracle_relight's own random numbers, trace()
and surface() (nero_oracle_relight_tex.surface for textured materials) and take each sample's radiance from that module's
render(spp=1, spp0=s), which is exact per sample.  prep / iterate / finish restate the filter; they take the sums as given, so
the GPU's own fp32 sums can be fed to them.
"""
import numpy as np

import nero_oracle_relight as OR

AOV = 16
DEMOD_EPS = 1e-3
VAR_NONE = 1e20


def features(verts, tris, materials, tables, pose, K, h, w, spp, max_bounces=4, seed=0, ggx_smith=0, spp0=0, textured=False):
    """Samples [spp0, spp0 + spp) -> (accum [h,w,4], aov [h,w,16]) sums in fp64, the layout of include/nero_denoise.h.
    materials: the [V,8] table (per-vertex) or (vt, ft, tex) with textured=True."""
    if textured:
        import nero_oracle_relight_tex as M
    else:
        M = OR
    pose, K = np.asarray(pose, np.float64), np.asarray(K, np.float64)
    R, t = pose[:, :3], pose[:, 3]
    pix = np.arange(h * w)
    x, y = pix % w, pix // w
    acc, aov = np.zeros((h * w, 4)), np.zeros((h * w, AOV))
    for s in range(spp0, spp0 + spp):
        c = np.stack([(x + OR.uniform(seed, pix, s, 0, 0) - K[0, 2]) / K[0, 0], (y + OR.uniform(seed, pix, s, 0, 1) - K[1, 2]) / K[1, 1],
                      np.ones(h * w)], -1)
        d = OR.normalize(c @ R)
        o = np.broadcast_to(-R.T @ t, d.shape).copy()
        tri, tt, uu, vv = OR.trace(verts, tris, o, d)
        k = np.nonzero(tri >= 0)[0]
        p, n, alb, met, _ = M.surface(verts, tris, materials, tri[k], tt[k], uu[k], vv[k], o[k], d[k])
        L = M.render(verts, tris, materials, tables, pose, K, h, w, 1, max_bounces, seed, ggx_smith, spp0=s).reshape(-1, 4)
        assert np.array_equal(L[:, 3] > 0, tri >= 0)
        L = L[k, :3]
        m1 = (1 - met)[:, None]
        g = m1 * alb + 0.04 * m1 + met[:, None] * alb
        D = L / (g + DEMOD_EPS)
        acc[k, :3] += L
        acc[k, 3] += 1
        aov[k, 0:3] += D
        aov[k, 3] += OR.luminance(D) ** 2
        aov[k, 4:7] += g
        aov[k, 8:11] += n
        aov[k, 12:15] += p
        aov[k, 15] += tt[k] * (d[k] @ R[2])
    return acc.reshape(h, w, 4), aov.reshape(h, w, AOV)


def prep(accum, aov, spp, focal):
    """-> col [h,w,4] (demodulated mean, luminance variance of the mean), feat [h,w,12] (albedo, alpha, unit normal, 0,
    point, footprint)."""
    accum, aov = np.asarray(accum, np.float64), np.asarray(aov, np.float64)
    hits = accum[..., 3]
    inv = np.where(hits > 0, 1.0 / np.where(hits > 0, hits, 1.0), 0.0)[..., None]
    c = aov[..., 0:3] * inv
    l = OR.luminance(c)
    var = np.where(hits >= 2, np.maximum(aov[..., 3] * inv[..., 0] - l * l, 0.0) / np.maximum(hits - 1, 1.0), VAR_NONE)
    nl = np.linalg.norm(aov[..., 8:11], axis=-1, keepdims=True)
    n = np.where(nl > 0, aov[..., 8:11] / np.where(nl > 0, nl, 1.0), 0.0)
    fp = aov[..., 15:16] * inv / focal
    col = np.concatenate([c, var[..., None]], -1)
    feat = np.concatenate([aov[..., 4:7] * inv, (hits / spp)[..., None], n, np.zeros_like(fp), aov[..., 12:15] * inv, fp], -1)
    return col, feat


def _shift(a, dy, dx):
    """(b, valid): b[y, x] = a[y + dy, x + dx] where that pixel exists."""
    H, W = a.shape[:2]
    yy, xx = np.arange(H) + dy, np.arange(W) + dx
    vy, vx = (yy >= 0) & (yy < H), (xx >= 0) & (xx < W)
    return a[np.clip(yy, 0, H - 1)][:, np.clip(xx, 0, W - 1)], vy[:, None] & vx[None, :]


def iterate(col, feat, level, sigma_l, sigma_n, sigma_x, eps):
    """One a-trous iteration at step 2^level."""
    col, feat = np.asarray(col, np.float64), np.asarray(feat, np.float64)
    step = 1 << level
    alpha, nrm, pos, fp = feat[..., 3], feat[..., 4:7], feat[..., 8:11], feat[..., 11]
    g3 = (0.25, 0.5, 0.25)
    vs, vw = np.zeros(alpha.shape), np.zeros(alpha.shape)
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            vq, ok = _shift(col[..., 3], dy, dx)
            k = g3[dx + 1] * g3[dy + 1] * (_shift(alpha, dy, dx)[0] if dy or dx else 1.0)
            vs += np.where(ok, k * vq, 0.0)
            vw += np.where(ok, k, 0.0)
    lp = OR.luminance(col[..., :3])
    h5 = np.asarray([1, 4, 6, 4, 1]) / 16.0
    s, sv, sw = np.zeros(col.shape[:2] + (3,)), np.zeros(alpha.shape), np.zeros(alpha.shape)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        l_scale = 1.0 / (sigma_l * np.sqrt(vs / vw) + eps)
        x_scale = 1.0 / (sigma_x * fp * step) ** 2
        for j in range(-2, 3):
            for i in range(-2, 3):
                cq, ok = _shift(col, j * step, i * step)
                wt = np.full(alpha.shape, h5[i + 2] * h5[j + 2])
                if i or j:
                    aq = _shift(alpha, j * step, i * step)[0]
                    nq = _shift(nrm, j * step, i * step)[0]
                    xq = _shift(pos, j * step, i * step)[0]
                    dl = np.abs(lp - OR.luminance(cq[..., :3]))
                    d2 = ((pos - xq) ** 2).sum(-1)
                    nd = np.maximum((nrm * nq).sum(-1), 0.0)
                    wt = wt * aq * nd ** sigma_n * np.exp(-dl * l_scale - d2 * x_scale)
                    ok = ok & (aq > 0)
                wt = np.where(ok, wt, 0.0)
                s += wt[..., None] * cq[..., :3]
                sv += wt * wt * cq[..., 3]
                sw += wt
        out = np.concatenate([s / sw[..., None], (sv / (sw * sw))[..., None]], -1)
    return np.where((alpha > 0)[..., None], out, col)


def finish(col, feat):
    """-> [h,w,4]: remodulated, premultiplied by the pixel's own alpha, alpha."""
    col, feat = np.asarray(col, np.float64), np.asarray(feat, np.float64)
    a = feat[..., 3:4]
    return np.concatenate([col[..., :3] * (feat[..., 0:3] + DEMOD_EPS) * a, a], -1)


def denoise(accum, aov, spp, focal, iterations=5, sigma_l=4.0, sigma_n=64.0, sigma_x=1.4, eps=1e-3):
    col, feat = prep(accum, aov, spp, focal)
    for i in range(iterations):
        col = iterate(col, feat, i, sigma_l, sigma_n, sigma_x, eps)
    return finish(col, feat)
