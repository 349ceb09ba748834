"""numpy fp64 restatement of include/nero_align.h: the transform, the point-to-plane terms (normal, residual, Jacobian row),
the moments, the truncated score and the fixed-order pairwise tree of the block partials and of their reduction, operation
for operation; closest points come from nero_oracle_meshdist.query (brute force), and register() runs the host logic of
nero_b200/align.py on them, so the product's iterates are compared bit for bit.  numpy evaluates every float64 operation
correctly rounded and never contracts a * b + c."""
import numpy as np

import nero_oracle_meshdist as OD
from nero_b200 import align as A

BLOCK = A.BLOCK


def _dot(u, v):
    return (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]


def _cross(u, v):
    return np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                     u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], 1)


def transform(points, mats):
    """[K n, 3]: y_r = ((m_r0 x + m_r1 y) + m_r2 z) + m_r3 for each of mats [K,3,4]."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    m = np.asarray(mats, np.float64).reshape(-1, 3, 4)
    return np.concatenate([np.stack([((p[:, 0] * M[r, 0] + p[:, 1] * M[r, 1]) + p[:, 2] * M[r, 2]) + M[r, 3] for r in range(3)], 1)
                           for M in m])


def tree(x):
    """The pairwise tree along axis 1 of x [.., 2^k, ..]: level h adds element i + h to element i for i divisible by 2h."""
    while x.shape[1] > 1:
        x = x[:, 0::2] + x[:, 1::2]
    return x[:, 0]


def _chunks(x):
    """[rows, w] -> [ceil(rows / 256), 256, w], the last chunk padded with +0."""
    c = -(-x.shape[0] // BLOCK)
    pad = np.zeros((c * BLOCK, x.shape[1]))
    pad[:x.shape[0]] = x
    return pad.reshape(c, BLOCK, x.shape[1])


def block_partials(values):
    """[ceil(n / 256), w]: each block of 256 consecutive rows of values [n, w] summed by the tree."""
    return tree(_chunks(np.asarray(values, np.float64).reshape(values.shape[0], -1)))


def reduce(partial):
    """[segments, w] of partial [segments, blocks, w]: levels of 256-row chunks summed by the tree until one row is left."""
    out = []
    for seg in np.asarray(partial, np.float64):
        while seg.shape[0] > 1:
            seg = tree(_chunks(seg))
        out.append(seg[0])
    return np.stack(out)


def terms_values(y, tri, closest, verts, tris, center):
    """[n, 38]: each point's values of nero_align_terms (zeros for tri < 0; a 1 in column 37 for a zero cross product)."""
    y, q = np.asarray(y, np.float64).reshape(-1, 3), np.asarray(closest, np.float64).reshape(-1, 3)
    tri = np.asarray(tri).reshape(-1)
    out = np.zeros((y.shape[0], A.TERMS))
    hit = np.flatnonzero(tri >= 0)
    v = np.asarray(verts, np.float32).astype(np.float64)
    t = np.asarray(tris, np.int64).reshape(-1, 3)[tri[hit]]
    a, b, c = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    m = _cross(b - a, c - a)
    deg = (m[:, 0] == 0.0) & (m[:, 1] == 0.0) & (m[:, 2] == 0.0)
    out[hit[deg], 37] = 1.0
    ok = ~deg
    rows, m, yy, qq = hit[ok], m[ok], y[hit[ok]], q[hit[ok]]
    l = np.sqrt(_dot(m, m))
    n = m / l[:, None]
    d = yy - np.asarray(center, np.float64)[None]
    r = _dot(n, yy - qq)
    J = np.concatenate([_cross(d, n), n, _dot(n, d)[:, None]], 1)
    vals = [J[:, i] * J[:, j] for i in range(7) for j in range(i, 7)] + [J[:, i] * r for i in range(7)] + [r * r, np.ones_like(r)]
    out[rows, :37] = np.stack(vals, 1)
    return out


def moments_values(points, origin):
    """[n, 10]: 1, d, and the upper triangle of d d^T, d = p - origin."""
    d = np.asarray(points, np.float64).reshape(-1, 3) - np.asarray(origin, np.float64)[None]
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    return np.stack([np.ones_like(x), x, y, z, x * x, x * y, x * z, y * y, y * z, z * z], 1)


def score_partials(dist, k, tau):
    """[k, ceil(m / 256)]: per segment of m distances, the block sums of min(d, tau)^2."""
    v = np.minimum(np.asarray(dist, np.float64).reshape(k, -1), tau)
    return np.stack([block_partials((x * x)[:, None])[:, 0] for x in v])


def bbox_center(points):
    p = np.asarray(points, np.float64)
    return (p.min(0) + p.max(0)) / 2


class Backend:
    """register()'s backend in numpy: source points [n,3], the target mesh and its samples [m,3]; brute-force queries."""

    def __init__(self, pts, verts, tris, tgt, coarse=A.COARSE_SAMPLES):
        self.pts, self.verts, self.tris, self.tgt = (np.asarray(pts, np.float64), np.asarray(verts, np.float32),
                                                     np.asarray(tris, np.int32), np.asarray(tgt, np.float64))
        self.src_origin, self.dst_origin = bbox_center(self.pts), bbox_center(self.tgt)
        n = self.pts.shape[0]
        self.coarse = min(coarse, n)
        self.sub = self.pts[np.arange(self.coarse, dtype=np.int64) * n // self.coarse]
        self.trace = []

    def moments(self, which):
        p, o = (self.pts, self.src_origin) if which == 'src' else (self.tgt, self.dst_origin)
        return reduce(block_partials(moments_values(p, o))[None])[0]

    def terms(self, M, tau, center):
        y = transform(self.pts, M)
        _, tri, q = OD.query(y, self.verts, self.tris, tau)
        sums = reduce(block_partials(terms_values(y, tri, q, self.verts, self.tris, center))[None])[0]
        self.trace.append((np.asarray(M).copy(), tau, sums))
        return sums

    def score(self, mats, tau):
        k = mats.shape[0]
        d = OD.query(transform(self.sub, mats), self.verts, self.tris, tau)[0]
        return reduce(score_partials(d, k, tau)[:, :, None])[:, 0]


def align(pts, verts, tris, tgt, rigid=False, init='identity', max_distance=None, max_iters=50, coarse=A.COARSE_SAMPLES):
    """nero_b200.align.align on given source points and target samples -> (result dict, backend with its trace)."""
    b = Backend(pts, verts, tris, tgt, coarse)
    return A.register(b, rigid, init, max_distance, max_iters), b
