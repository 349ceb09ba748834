"""numpy restatement of the glTF export's kernels (include/nero_gltf.h, k_gltf.cu) for the tests.

  weld           exact integers: each vertex's corners in the corner walk's order are its corners in ascending 3 t + s, so
                 the distinct (position, uv) pairs ranked by their first corner in that order are the kernel's welded vertices.
  frames         the tangent frames in float64 from the same float32 inputs, the kernel's skips, weights and fallbacks.
  tangent_space  the conversion in float32 with the kernel's operation order (every numpy float32 operation is rounded on its
                 own, as the kernel's _rn intrinsics are), on nero_oracle_texmap's raster and barycentrics.
  viewer_decode  the glTF 2.0 sample viewer's per-fragment decode of the converted bytes in float64:
                 normalize(T x0 + B x1 + N x2) with x = 2k/255 - 1 and the frame interpolated as the conversion does.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np

import nero_oracle_texmap as OT

F32 = np.float32


def encode(n):
    n = np.asarray(n, F32)
    k = np.floor((n * F32(0.5) + F32(0.5)) * F32(255) + F32(0.5))
    return np.clip(k, 0, 255).astype(np.uint8)


def material_tables():
    """(lut_m, lut_r) of include/nero_gltf.h, from the sRGB decoding of utils/raw_utils.py in float64."""
    s = np.arange(256, dtype=np.float64) / 255.0
    lin = np.where(s <= 0.04045, 25 / 323 * s, np.maximum((200 * s + 11) / 211, np.finfo(np.float32).eps) ** (12 / 5))
    return np.rint(255.0 * lin).astype(np.uint8), np.rint(255.0 * np.sqrt(lin)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ weld
def weld(tris, ft, V):
    """-> (wv [W], wt [W], wf [T,3]) int32."""
    tris = np.asarray(tris, np.int64)
    ft = np.asarray(ft, np.int64)
    flat, uv = tris.reshape(-1), ft.reshape(-1)
    order = np.argsort(flat, kind='stable')                       # corners by vertex, then by 3 t + s
    key = flat[order] * (int(uv.max(initial=0)) + 1) + uv[order]
    _, first, inv = np.unique(key, return_index=True, return_inverse=True)
    rank = np.empty(first.size, np.int64)
    rank[np.argsort(first, kind='stable')] = np.arange(first.size)  # pairs in order of their first corner
    wf = np.empty(flat.size, np.int64)
    wf[order] = rank[inv.reshape(-1)]
    pair_corner = order[np.sort(first)]
    return flat[pair_corner].astype(np.int32), uv[pair_corner].astype(np.int32), wf.reshape(-1, 3).astype(np.int32)


# ------------------------------------------------------------------------------------------------ tangent frames
def _norm(a):
    return np.sqrt((a * a).sum(-1))


def frames(verts, tris, vt, ft, normals, wv, wt, wf):
    """-> (wnormal [W,3], wtangent [W,4]) float64.  normals: the position vertices' float32 normals; vt: the file's uv."""
    P = np.asarray(verts, F32).astype(np.float64)
    UV = np.asarray(vt, F32).astype(np.float64)
    tris, ft = np.asarray(tris, np.int64), np.asarray(ft, np.int64)
    wv, wf = np.asarray(wv, np.int64), np.asarray(wf, np.int64).reshape(-1)
    W = wv.size
    n = np.asarray(normals, F32).astype(np.float64)[wv]
    zero = (n * n).sum(1) == 0
    n[zero] = (0.0, 0.0, 1.0)
    T = tris.shape[0]
    t, s = np.divmod(np.arange(3 * T), 3)
    c = [tris[t, (s + j) % 3] for j in range(3)]
    u = [ft[t, (s + j) % 3] for j in range(3)]
    e1, e2 = P[c[1]] - P[c[0]], P[c[2]] - P[c[0]]
    d1, d2 = UV[u[1]] - UV[u[0]], UV[u[2]] - UV[u[0]]
    det = d1[:, 0] * d2[:, 1] - d2[:, 0] * d1[:, 1]
    sdet = np.where(det == 0, 1.0, det)[:, None]
    tf = (d2[:, 1:2] * e1 - d1[:, 1:2] * e2) / sdet
    bf = (d1[:, 0:1] * e2 - d2[:, 0:1] * e1) / sdet
    nc = n[wf]
    tp = tf - nc * (nc * tf).sum(1, keepdims=True)
    l1, l2, lp = _norm(e1), _norm(e2), _norm(tp)
    ok = (det != 0) & (l1 > 0) & (l2 > 0) & (lp > 0) & ~zero[wf]
    safe = lambda x: np.where(x > 0, x, 1.0)[:, None]
    a = np.arccos(np.clip(((e1 / safe(l1)) * (e2 / safe(l2))).sum(1), -1, 1))
    sign = np.where((np.cross(nc, tf) * bf).sum(1) < 0, -1.0, 1.0)
    S, h, used = np.zeros((W, 3)), np.zeros(W), np.zeros(W, bool)
    np.add.at(S, wf[ok], a[ok, None] * tp[ok] / lp[ok, None])
    np.add.at(h, wf[ok], sign[ok] * a[ok])
    used[wf[ok]] = True
    S = S - n * (n * S).sum(1, keepdims=True)
    lS = _norm(S)
    good = used & (lS > 0)
    tan = np.zeros((W, 4))
    tan[good, :3] = S[good] / lS[good, None]
    tan[:, 3] = np.where(good & (h < 0), -1.0, 1.0)
    ax = np.argmin(np.abs(n), 1)                                  # the first smallest component
    fb = np.cross(np.eye(3)[ax], n)
    fb = fb / np.where(_norm(fb) > 0, _norm(fb), 1.0)[:, None]
    tan[~good, :3] = fb[~good]
    tan[zero, :3] = (1.0, 0.0, 0.0)
    return n, tan


# ------------------------------------------------------------------------------------------------ tangent-space conversion
def _dot32(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def _cross32(a, b):
    return np.stack([a[..., 1] * b[..., 2] - a[..., 2] * b[..., 1], a[..., 2] * b[..., 0] - a[..., 0] * b[..., 2],
                     a[..., 0] * b[..., 1] - a[..., 1] * b[..., 0]], -1)


def _normalize32(s):
    l2 = _dot32(s, s)
    ok = l2 > 0
    out = s.copy()
    out[ok] = s[ok] / np.sqrt(l2[ok])[:, None]
    return out, ok


def _blend32(b, r):
    """((b0 r0 + b1 r1) + b2 r2): b [n,3], r [n,3,k]."""
    return (b[:, 0:1] * r[:, 0] + b[:, 1:2] * r[:, 1]) + b[:, 2:3] * r[:, 2]


def atlas(vt):
    """(u, 1 - v) of the file's vt in float32: glTF's TEXCOORD_0, the atlas the conversion rasterises."""
    vt = np.asarray(vt, F32)
    return np.stack([vt[:, 0], F32(1) - vt[:, 1]], -1)


def texel_frames(atlas, ft, wf, wnormal, wtangent, width, height, dtype=F32):
    """The raster of the atlas (glTF's uv) at width x height and the interpolated frames of its covered texels -> dict owner
    [h,w], texel [n] (row-major), bary [n,3] float32, N, T, B [n,3] in dtype (float32: the kernel's operations and
    normalisations; float64: the viewer's)."""
    owner, _, bary = OT.rasterize(atlas, ft, width, height)
    m = owner >= 0
    texel = np.nonzero(m.reshape(-1))[0]
    b = bary[m].astype(dtype)
    v = np.asarray(wf, np.int64)[owner[m]]
    n = np.asarray(wnormal, dtype)[v]
    t4 = np.asarray(wtangent, dtype)[v]
    c = _cross32(n, t4[..., :3]) * t4[..., 3:4]
    out = dict(owner=owner, texel=texel, bary=bary[m])
    for key, r in (('N', n), ('T', t4[..., :3]), ('B', c)):
        f = _blend32(b, r)
        if dtype == F32:
            out[key] = _normalize32(f)[0]
        else:
            out[key] = f / np.where(_norm(f) > 0, _norm(f), 1.0)[:, None]
    return out


def tangent_space(vt, ft, wf, wnormal, wtangent, omap):
    """The kernel's conversion -> (img [h,w,5] uint8 before inpainting, texel_frames' float32 dict).  omap uint8 [h,w,3]."""
    omap = np.asarray(omap, np.uint8)
    h, w = omap.shape[:2]
    fr = texel_frames(atlas(vt), ft, wf, np.asarray(wnormal, F32), np.asarray(wtangent, F32), w, h)
    N, T, B = fr['N'], fr['T'], fr['B']
    k = omap.reshape(-1, 3)[fr['texel']]
    m, mok = _normalize32(F32(2) * k.astype(F32) / F32(255) - F32(1))
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        bn, nt, tb = _cross32(B, N), _cross32(N, T), _cross32(T, B)
        det = _dot32(T, bn)
        y = np.stack([_dot32(m, bn) / det, _dot32(m, nt) / det, _dot32(m, tb) / det], -1).astype(F32)
        fin = np.isfinite(y).all(1)
        y[~fin] = 0
        y, yok = _normalize32(y)
    good = mok & (det != 0) & np.isfinite(det) & fin & yok & np.isfinite(y).all(1)
    x = np.where(good[:, None], y, np.array([0, 0, 1], F32))
    img = np.zeros((h * w, 5), np.uint8)
    img[fr['texel'], :3] = encode(x)
    return img.reshape(h, w, 5), fr


def viewer_decode(img, frames64):
    """normalize(T x0 + B x1 + N x2) in float64 per covered texel of texel_frames(..., np.float64), x = 2k/255 - 1 of the
    tangent-space bytes img [h,w,>=3]."""
    x = 2.0 * np.asarray(img)[..., :3].reshape(-1, 3)[frames64['texel']].astype(np.float64) / 255.0 - 1.0
    d = frames64['T'] * x[:, 0:1] + frames64['B'] * x[:, 1:2] + frames64['N'] * x[:, 2:3]
    return d / _norm(d)[:, None]


def angle_deg(a, b):
    a = a / _norm(a)[:, None]
    b = b / _norm(b)[:, None]
    return np.degrees(np.arccos(np.clip((a * b).sum(1), -1, 1)))
