"""numpy fp64 restatement of include/nero_meshdist.h: the closest point of a triangle (Ericson's Voronoi regions with the
degenerate rule), operation for operation, and the point-to-mesh distance over every triangle (query()) with the same tie rule, so the kernel's dist, tri and closest point are compared bit for bit.  numpy evaluates every float64 operation
correctly rounded and never contracts a * b + c."""
import numpy as np

CHUNK = 1 << 20      # triangles per vectorised pass


def _dot(u, v):
    return (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]


def _lerp(x, t, e):
    return x + t[:, None] * e


def _segment(x, y, e, xp):
    m, l = _dot(xp, e), _dot(e, e)
    with np.errstate(all='ignore'):
        t = m / l
    q = _lerp(x, t, e)
    q = np.where((m >= l)[:, None], y, q)
    return np.where((m <= 0.0)[:, None], x, q)


def _d2(p, q):
    d = p - q
    return _dot(d, d)


def _segments(p, a, b, c, ab, ac, bc, ap, bp):
    q = _segment(a, b, ab, ap)
    best = _d2(p, q)
    q1 = _segment(a, c, ac, ap)
    d1 = _d2(p, q1)
    take = d1 < best
    q = np.where(take[:, None], q1, q)
    best = np.where(take, d1, best)
    q2 = _segment(b, c, bc, bp)
    return np.where((_d2(p, q2) < best)[:, None], q2, q)


def closest_points(p, a, b, c):
    """Closest points q [m,3] of triangles (a, b, c) to points p, row by row (all [m,3] float64), and the region code of
    each row: 0 a, 1 b, 2 c, 3 edge ab, 4 edge ac, 5 edge bc, 6 face, 7 the three edge segments."""
    p, a, b, c = (np.asarray(x, np.float64).reshape(-1, 3) for x in (p, a, b, c))
    ab, ac, ap, bp, cp, bc = b - a, c - a, p - a, p - b, p - c, c - b
    nx = ab[:, 1] * ac[:, 2] - ab[:, 2] * ac[:, 1]
    ny = ab[:, 2] * ac[:, 0] - ab[:, 0] * ac[:, 2]
    nz = ab[:, 0] * ac[:, 1] - ab[:, 1] * ac[:, 0]
    d1, d2 = _dot(ab, ap), _dot(ac, ap)
    d3, d4 = _dot(ab, bp), _dot(ac, bp)
    vc = d1 * d4 - d3 * d2
    d5, d6 = _dot(ab, cp), _dot(ac, cp)
    vb = d5 * d2 - d1 * d6
    va = d3 * d6 - d5 * d4
    e, f = d4 - d3, d5 - d6
    s = (va + vb) + vc
    region = np.full(p.shape[0], -1, np.int8)
    todo = ~((nx == 0.0) & (ny == 0.0) & (nz == 0.0))
    region[~todo] = 7

    def take(mask, code):
        nonlocal todo
        mask = todo & mask
        region[mask] = code
        todo = todo & ~mask

    take((d1 <= 0.0) & (d2 <= 0.0), 0)
    take((d3 >= 0.0) & (d4 <= d3), 1)
    den_ab = d1 - d3
    take((vc <= 0.0) & (d1 >= 0.0) & (d3 <= 0.0) & (den_ab > 0.0), 3)
    take((vc <= 0.0) & (d1 >= 0.0) & (d3 <= 0.0), 7)
    take((d6 >= 0.0) & (d5 <= d6), 2)
    den_ac = d2 - d6
    take((vb <= 0.0) & (d2 >= 0.0) & (d6 <= 0.0) & (den_ac > 0.0), 4)
    take((vb <= 0.0) & (d2 >= 0.0) & (d6 <= 0.0), 7)
    den_bc = e + f
    take((va <= 0.0) & (e >= 0.0) & (f >= 0.0) & (den_bc > 0.0), 5)
    take((va <= 0.0) & (e >= 0.0) & (f >= 0.0), 7)
    take((va >= 0.0) & (vb >= 0.0) & (vc >= 0.0) & (s > 0.0), 6)
    take(np.ones_like(todo), 7)
    with np.errstate(all='ignore'):
        cands = [a, b, c, _lerp(a, d1 / den_ab, ab), _lerp(a, d2 / den_ac, ac), _lerp(b, e / den_bc, bc),
                 _lerp(_lerp(a, vb / s, ab), vc / s, ac)]
    q = np.empty_like(p)
    for code, cand in enumerate(cands):
        sel = region == code
        q[sel] = cand[sel]
    sel = region == 7
    if sel.any():
        q[sel] = _segments(*(x[sel] for x in (p, a, b, c, ab, ac, bc, ap, bp)))
    return q, region


def triangle_d2(p, a, b, c):
    """Squared distances d2 [m] of the header's routine, row by row."""
    p = np.asarray(p, np.float64).reshape(-1, 3)
    return _d2(p, closest_points(p, a, b, c)[0])


def _chunked_d2(q, a, b, c):
    out = np.empty(a.shape[0])
    for j0 in range(0, a.shape[0], CHUNK):
        j1 = min(a.shape[0], j0 + CHUNK)
        out[j0:j1] = triangle_d2(np.broadcast_to(q, (j1 - j0, 3)), a[j0:j1], b[j0:j1], c[j0:j1])
    return out


def query(points, verts, tris, max_dist=np.inf):
    """(dist [n] float64, tri [n] int32, closest [n,3] float64) of the minimum d2 over every triangle, ties to the lowest
    triangle index, dist = sqrt(d2); dist > max_dist gives (+inf, -1, NaN).

    The routine runs on the triangles that can attain the minimum: a triangle is skipped when the distance to its bounding box
    exceeds the distance to the nearest mesh vertex (an upper bound of the minimum) by a margin of 1e-6 relative plus 1e-9
    times the mesh's largest |coordinate|, millions of times the routine's rounding error.  Unlike the kernel's BVH this test
    looks at every triangle on its own, so it shares nothing with the search it checks."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    v = np.asarray(verts, np.float32).astype(np.float64)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    lo, hi = np.minimum(np.minimum(a, b), c), np.maximum(np.maximum(a, b), c)
    used = np.unique(t)
    vu = v[used]
    slack = 1e-9 * np.abs(v).max()
    n = p.shape[0]
    dist = np.full(n, np.inf)
    tri = np.full(n, -1, np.int32)
    closest = np.full((n, 3), np.nan)
    for i in range(n):
        q = p[i]
        upper = np.sqrt(((vu - q) ** 2).sum(1).min())
        g = np.maximum(np.maximum(lo - q, q - hi), 0.0)
        cand = np.flatnonzero(np.sqrt((g * g).sum(1)) <= upper * (1 + 1e-6) + slack)
        d2 = _chunked_d2(q, a[cand], b[cand], c[cand])
        k = int(np.argmin(d2))                      # first occurrence: the lowest triangle index
        d = np.sqrt(d2[k])
        if d <= max_dist:
            j = cand[k]
            dist[i], tri[i] = d, j
            closest[i] = closest_points(q[None], a[j:j + 1], b[j:j + 1], c[j:j + 1])[0][0]
    return dist, tri, closest
