"""Register a mesh or point cloud to a reference mesh on the GPU (k_align.cu, include/nero_align.h): a trimmed
point-to-plane similarity ICP over the reference's BVH, started from the identity, a principal-axis search or a given matrix.

meshdist.compare measures two meshes in one frame.  Two reconstructions of one object (two SfM runs, two captures) or a
reconstruction and a scan are not in one frame: they differ by a rotation, a translation and a scale, which the metrics
would report as error.  align() estimates that similarity, and compare_meshes.py --align measures in the registered frame.

Convention
----------
  * The estimated map is y = s R x + t from source to target: R a proper rotation, s > 0 (rigid=True fixes s = 1 exactly).
    `matrix` is the float64 4 x 4 [[s R, t], [0, 1]].
  * Target: a MeshDistance (a triangle mesh with its BVH).  Source: a mesh (verts, tris), replaced by `samples`
    evaluate.sample_surface samples (seed `seed`, drawn once), or points [n,3] (a point cloud, evaluate.read_points_ply).
    The target's statistics come from `samples` samples of its own (seed `seed` + 1): its centroid c, fixed for the run,
    and its size L = sqrt(tr C), C the samples' covariance (the RMS distance from c).
  * One iteration at transform T_k: the source points mapped in float64 (nero_align_transform), queried with
    nero_meshdist_query at max_dist tau_k with closest points; for each point within tau_k, the unit normal n of the returned
    triangle from its original vertices (a zero cross product skips the point and counts it as degenerate), the residual
    r = n . (y - q) and the row J = [(y - c) x n, n, n . (y - c)] of the update y' = c + (1 + sigma)(I + [w]x)(y - c) + dt.
    nero_align_terms and nero_align_reduce sum J^T J (upper triangle), J^T r, r^2 and the counts in a fixed order, so two
    runs give the same bytes and oracle/nero_oracle_align.py reproduces every bit.
  * Host step (step(), shared with the oracle): the columns of w and sigma are scaled by 1 / L, so every parameter is a
    length; the system (A + lambda tr(A) / k I) z = -b (k = 7, or 6 when rigid) is solved with numpy; w is applied by
    Rodrigues' formula and sigma as exp(sigma): s' = e^sigma s, R' = R(w) R, t' = e^sigma R(w)(t - c) + c + dt.
    tau_{k+1} = max(tau_min, min(tau_k, 3 rms_k)); the run stops when max(|w|, |dt| / L, |sigma|) < TOLERANCE or after
    max_iters.
  * Undetermined degrees of freedom: the eigenvectors of the scaled J^T J over the rows used whose eigenvalue is below
    UNDETERMINED times the largest, each named by the block holding most of its weight (rotation, translation, scale).  A
    sphere leaves three rotations free and a torus one; the damping keeps the step along them near zero, so the other
    parameters stay meaningful.
  * init='auto': the moments (count, sum, second moments about the points' bounding-box centre, nero_align_moments) of the
    source points and of the target samples give their means and covariances; numpy.linalg.eigh gives the principal axes
    E (columns made a proper rotation); s0 = sqrt(tr C_dst / tr C_src) (1 when rigid); the 24 candidates
    R_i = E_dst G_i E_src^T, G_i the proper signed permutations, t_i = mu_dst - s0 R_i mu_src.  Each is scored on the same
    COARSE_SAMPLES source points (indices floor(j n / m)) as the mean of min(d, tau)^2 with tau = COARSE_TAU L, all 24 in one
    query; the lowest score wins, ties to the lowest index.

TAU0, TAU_MIN, DAMPING, TOLERANCE, UNDETERMINED, COARSE_TAU, COARSE_SAMPLES and the default sample count are choices, not
tuned values.
"""
import itertools

import numpy as np

TERMS, MOMENTS, BLOCK = 38, 10, 256      # include/nero_align.h
COARSE_SAMPLES = 16384                    # source points scored per coarse candidate
COARSE_TAU = 0.1                          # coarse score truncation, times L
TAU0 = 0.1                                # first inlier distance, times L (max_distance overrides it)
TAU_MIN = 1e-3                            # least inlier distance, times L
DAMPING = 1e-9                            # lambda
TOLERANCE = 1e-10                         # largest step component (radians, L, log-scale) that ends the run
UNDETERMINED = 1e-2                       # eigenvalue ratio below which a direction is reported as undetermined: an exact
                                          # symmetry gives 0, the facets of a 24^3 marching-cubes sphere about 1e-3


def _group():
    """The 24 proper signed permutation matrices: permutations in lexicographic order, then signs (+ before -) x, y, z."""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            G = np.zeros((3, 3))
            G[np.arange(3), perm] = signs
            if np.linalg.det(G) > 0:
                out.append(G)
    return out


GROUP = _group()


def matrix(s, R, t):
    M = np.eye(4)
    M[:3, :3] = s * R
    M[:3, 3] = t
    return M


def decompose(M):
    """(s, R, t) of a 4 x 4 similarity: s = cbrt(det A), R = A / s orthonormalised by SVD.  Raises ValueError unless det A > 0."""
    M = np.asarray(M, np.float64)
    if M.shape != (4, 4) or not np.isfinite(M).all():
        raise ValueError(f'a transform must be a finite 4 x 4 matrix, got shape {M.shape}')
    A = M[:3, :3]
    det = np.linalg.det(A)
    if not det > 0:
        raise ValueError(f'a transform must keep orientation (det > 0), got det {det}')
    s = float(np.cbrt(det))
    U, _, Vt = np.linalg.svd(A / s)
    return s, U @ Vt, M[:3, 3].copy()


def inverse(M):
    s, R, t = decompose(M)
    return matrix(1.0 / s, R.T, -(R.T @ t) / s)


def rodrigues(w):
    th = float(np.sqrt(w @ w))
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    if th < 1e-4:
        a, b = 1.0 - th * th / 6.0, 0.5 - th * th / 24.0
    else:
        a, b = np.sin(th) / th, (1.0 - np.cos(th)) / (th * th)
    return np.eye(3) + a * K + b * (K @ K)


def moment_stats(sums, origin):
    """(mean [3], covariance [3,3]) from the NERO_ALIGN_MOMENTS sums about origin."""
    n = sums[0]
    m = sums[1:4] / n
    S = np.array([[sums[4], sums[5], sums[6]], [sums[5], sums[7], sums[8]], [sums[6], sums[8], sums[9]]]) / n
    return np.asarray(origin, np.float64) + m, S - np.outer(m, m)


def system(sums, length, rigid):
    """(A, b) of the scaled normal equations (k x k, k) from the NERO_ALIGN_TERMS sums."""
    A = np.zeros((7, 7))
    iu = np.triu_indices(7)
    A[iu] = sums[:28]
    A.T[iu] = sums[:28]
    S = np.array([1.0 / length] * 3 + [1.0] * 3 + [1.0 / length])
    k = 6 if rigid else 7
    return (S[:, None] * A * S[None, :])[:k, :k], (S * sums[28:35])[:k], S[:k]


def step(sums, length, rigid):
    """The damped Gauss-Newton step x = (w, dt, sigma) (sigma = 0 when rigid) of one iteration's sums."""
    A, b, S = system(sums, length, rigid)
    k = A.shape[0]
    z = np.linalg.solve(A + DAMPING * np.trace(A) / k * np.eye(k), -b)
    x = np.zeros(7)
    x[:k] = S * z
    return x


def compose(s, R, t, x, center):
    """The transform after step x about center: s' = e^sigma s, R' = R(w) R, t' = e^sigma R(w)(t - c) + c + dt."""
    e = np.exp(x[6])
    Rw = rodrigues(x[:3])
    return e * s, Rw @ R, e * (Rw @ (t - center)) + center + x[3:6]


def undetermined(sums, length, rigid):
    """The directions of the scaled, per-row J^T J with eigenvalue < UNDETERMINED times the largest."""
    A, _, _ = system(sums, length, rigid)
    ev, V = np.linalg.eigh(A / max(sums[36], 1.0))
    out = []
    for i in np.flatnonzero(ev < UNDETERMINED * ev[-1]):
        v = V[:, i]
        w = [float(v[:3] @ v[:3]), float(v[3:6] @ v[3:6]), float(v[6:] @ v[6:])]
        out.append({'kind': ('rotation', 'translation', 'scale')[int(np.argmax(w))], 'eigenvalue': float(ev[i] / ev[-1]),
                    'vector': [float(a) for a in v]})
    return out


def candidates(src_stats, dst_stats, rigid):
    """The 24 coarse starts (s0, R_i, t_i) from the (mean, covariance) of both sides."""
    (ms, Cs), (md, Cd) = src_stats, dst_stats
    Es, Ed = np.linalg.eigh(Cs)[1], np.linalg.eigh(Cd)[1]
    Es[:, 2] *= np.sign(np.linalg.det(Es))
    Ed[:, 2] *= np.sign(np.linalg.det(Ed))
    s0 = 1.0 if rigid else float(np.sqrt(np.trace(Cd) / np.trace(Cs)))
    return [(s0, Ed @ G @ Es.T, md - s0 * (Ed @ G @ Es.T) @ ms) for G in GROUP]


def register(backend, rigid, init, max_distance, max_iters):
    """The host logic of align(), shared with the oracle.  backend gives NumPy sums: moments('src' | 'dst'),
    terms(M [3,4], tau, center), score(mats [K,3,4], tau) and the attributes src_origin, dst_origin, coarse (points per candidate)."""
    center, C = moment_stats(backend.moments('dst'), backend.dst_origin)
    length = float(np.sqrt(np.trace(C)))
    if not length > 0:
        raise ValueError('the target has no extent')
    out = {}
    if isinstance(init, str) and init == 'auto':
        cands = candidates(moment_stats(backend.moments('src'), backend.src_origin), (center, C), rigid)
        mats = np.stack([matrix(*c)[:3] for c in cands])
        scores = backend.score(mats, COARSE_TAU * length) / backend.coarse
        best = int(np.argmin(scores))
        s, R, t = cands[best]
        out['coarse_scores'], out['coarse_best'] = [float(v) for v in scores], best
    elif isinstance(init, str) and init == 'identity':
        s, R, t = 1.0, np.eye(3), np.zeros(3)
    elif isinstance(init, str):
        raise ValueError(f"init must be 'identity', 'auto' or a 4 x 4 matrix, got {init!r}")
    else:
        s, R, t = decompose(init)
        if rigid:
            s = 1.0
    tau = float(max_distance) if max_distance is not None else TAU0 * length
    tau_min = min(TAU_MIN * length, tau)
    taus, inliers, rmss, degenerate = [], [], [], []
    converged, sums = False, None
    for _ in range(int(max_iters)):
        sums = backend.terms(matrix(s, R, t)[:3], tau, center)
        used = sums[36]
        if used < (6 if rigid else 7):
            raise RuntimeError(f'align: {int(used)} source points within {tau:g} of the target: too few to fit the transform '
                               '(start closer, or raise max_distance)')
        rms = float(np.sqrt(sums[35] / used))
        x = step(sums, length, rigid)
        s, R, t = compose(s, R, t, x, center)
        taus.append(tau)
        inliers.append(int(used))
        rmss.append(rms)
        degenerate.append(int(sums[37]))
        tau = max(tau_min, min(tau, 3.0 * rms))
        if max(float(np.abs(x[:3]).max()), float(np.abs(x[3:6]).max()) / length, abs(float(x[6]))) < TOLERANCE:
            converged = True
            break
    M = matrix(s, R, t)
    out.update({'matrix': M, 'scale': float(s), 'rotation': R, 'translation': t, 'iterations': len(taus), 'tau': taus,
                'inliers': inliers, 'rms': rmss, 'degenerate': degenerate, 'converged': converged, 'center': center,
                'length': length, 'undetermined': undetermined(sums, length, rigid) if sums is not None else []})
    return out


# ------------------------------------------------------------------------------------------------------------ GPU side

def _launch(name, *args, launches=1):
    from . import ops
    ops.K(name, *args, launches=launches)


def transform(points, mats):
    """CUDA float64 [K n, 3]: the K transforms mats [K,3,4] (or one [3,4] / [4,4]) applied to points [n,3]."""
    import torch
    p = torch.as_tensor(points)
    dev = p.device if p.device.type == 'cuda' else torch.device('cuda')
    p = p.detach().to(dev, torch.float64).contiguous()
    if p.ndim != 2 or p.shape[1] != 3:
        raise ValueError(f'points must be [n,3], got {tuple(p.shape)}')
    m = np.asarray(mats, np.float64)
    m = m[None] if m.ndim == 2 else m
    if m.ndim != 3 or m.shape[1] not in (3, 4) or m.shape[2] != 4 or m.shape[0] < 1:
        raise ValueError(f'transforms must be [K,3,4], got {m.shape}')
    mt = torch.from_numpy(np.ascontiguousarray(m[:, :3])).to(dev)
    out = torch.empty(m.shape[0] * p.shape[0], 3, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        _launch('nero_align_transform', p, p.shape[0], mt, m.shape[0], out, launches=int(p.shape[0] > 0))
    return out


def apply(matrix_, points):
    """points [n,3] (numpy or tensor) mapped by the 4 x 4 matrix in float64 on the GPU -> CUDA float64 [n,3]."""
    return transform(points, np.asarray(matrix_, np.float64)[:3])


def terms(points, tri, closest, md, center):
    """Block partials [ceil(n / 256), 38] of nero_align_terms (CUDA float64)."""
    import torch
    n = points.shape[0]
    partial = torch.empty(max(1, -(-n // BLOCK)), TERMS, dtype=torch.float64, device=points.device)
    _launch('nero_align_terms', points, n, tri, closest, md.verts, md.tris, *(float(c) for c in center), partial, launches=int(n > 0))
    return partial


def moments(points, origin):
    """Block partials [ceil(n / 256), 10] of nero_align_moments (CUDA float64)."""
    import torch
    n = points.shape[0]
    partial = torch.empty(max(1, -(-n // BLOCK)), MOMENTS, dtype=torch.float64, device=points.device)
    _launch('nero_align_moments', points, n, *(float(o) for o in origin), partial, launches=int(n > 0))
    return partial


def score(dist, k, tau):
    """Block partials [k, ceil(m / 256)] of nero_align_score over dist [k m] (CUDA float64)."""
    import torch
    m = dist.shape[0] // k
    partial = torch.empty(k, -(-m // BLOCK), dtype=torch.float64, device=dist.device)
    _launch('nero_align_score', dist, m, k, float(tau), partial)
    return partial


def reduce(partial, segments, width):
    """nero_align_reduce: [segments, width] fixed-order sums of partial [segments, blocks, width] (overwritten)."""
    import torch
    blocks = partial.numel() // (segments * width)
    out = torch.empty(segments, width, dtype=torch.float64, device=partial.device)
    _launch('nero_align_reduce', partial, segments, blocks, width, out)
    return out


def bbox_center(points):
    """(lo + hi) / 2 of points [n,3] in float64 (the origin of the moments)."""
    lo, hi = points.amin(0).double().cpu().numpy(), points.amax(0).double().cpu().numpy()
    return (lo + hi) / 2


class _Gpu:
    """The backend of register() on the GPU: the source points, the target samples and the target's BVH."""

    def __init__(self, pts, dst, tgt):
        import torch
        self.pts, self.dst, self.tgt = pts, dst, tgt
        self.src_origin, self.dst_origin = bbox_center(pts), bbox_center(tgt)
        n = pts.shape[0]
        self.coarse = min(COARSE_SAMPLES, n)
        self.sub = pts[torch.from_numpy(np.arange(self.coarse, dtype=np.int64) * n // self.coarse).to(pts.device)].contiguous()
        dev = pts.device
        self.y = torch.empty(n, 3, dtype=torch.float64, device=dev)
        self.dist = torch.empty(n, dtype=torch.float64, device=dev)
        self.tri = torch.empty(n, dtype=torch.int32, device=dev)
        self.closest = torch.empty(n, 3, dtype=torch.float64, device=dev)
        self.status = torch.zeros(1, dtype=torch.int32, device=dev)

    def _query(self, y, tau, dist, tri, closest):
        d = self.dst
        _launch('nero_meshdist_query', y, y.shape[0], d.nodes, d.tri_ids, d.verts, d.tris, float(tau), dist, tri, closest, self.status)

    def _checked(self, sums):
        out = sums.cpu().numpy()
        if int(self.status.item()) != 0:
            raise RuntimeError('nero_meshdist_query: a traversal overran its stack (the BVH is deeper than the kernel supports)')
        return out

    def moments(self, which):
        p, o = (self.pts, self.src_origin) if which == 'src' else (self.tgt, self.dst_origin)
        return self._checked(reduce(moments(p, o), 1, MOMENTS))[0]

    def terms(self, M, tau, center):
        y = transform(self.pts, M)
        self._query(y, tau, self.dist, self.tri, self.closest)
        return self._checked(reduce(terms(y, self.tri, self.closest, self.dst, center), 1, TERMS))[0]

    def score(self, mats, tau):
        import torch
        y = transform(self.sub, mats)
        n = y.shape[0]
        dist = torch.empty(n, dtype=torch.float64, device=y.device)
        tri = torch.empty(n, dtype=torch.int32, device=y.device)
        self._query(y, tau, dist, tri, None)
        return self._checked(reduce(score(dist, mats.shape[0], tau), mats.shape[0], 1))[:, 0]


def source_points(src, samples, seed):
    """The source as CUDA float64 [n,3]: `samples` surface samples of a mesh (verts, tris), or the given points."""
    import torch
    from .evaluate import sample_surface
    if isinstance(src, (tuple, list)) and len(src) == 2:
        return sample_surface(src[0], src[1], samples, seed)
    p = torch.as_tensor(src)
    p = p.detach().to(p.device if p.device.type == 'cuda' else torch.device('cuda'), torch.float64).contiguous()
    if p.ndim != 2 or p.shape[1] != 3 or p.shape[0] < 7:
        raise ValueError(f'source points must be [n,3] with n >= 7, got {tuple(p.shape)}')
    if not bool(torch.isfinite(p).all()):
        raise ValueError('source points must be finite')
    return p


def check_args(init, samples, seed, max_distance, max_iters):
    if isinstance(init, str):
        if init not in ('identity', 'auto'):
            raise ValueError(f"init must be 'identity', 'auto' or a 4 x 4 matrix, got {init!r}")
    else:
        decompose(init)
    if int(samples) != samples or samples < 256:
        raise ValueError(f'samples must be an integer >= 256, got {samples}')
    if not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 32 - 1:
        raise ValueError(f'seed must be an integer in [0, 2^32 - 1), got {seed}')
    if max_distance is not None and not (np.isfinite(max_distance) and max_distance > 0):
        raise ValueError(f'max_distance must be positive and finite, got {max_distance}')
    if int(max_iters) != max_iters or max_iters < 1:
        raise ValueError(f'max_iters must be an integer >= 1, got {max_iters}')


def align(src, dst, *, rigid=False, init='identity', samples=200_000, seed=0, max_distance=None, max_iters=50):
    """Register src (a mesh (verts, tris) or points [n,3]) to dst (a MeshDistance): the similarity y = s R x + t of the module
    docstring -> dict with matrix (4 x 4), scale, rotation, translation, iterations, per-iteration tau / inliers / rms /
    degenerate, converged, undetermined, the run's center and length, and with init='auto' the 24 coarse_scores and
    coarse_best."""
    from .meshdist import MeshDistance
    from .evaluate import sample_surface
    if not isinstance(dst, MeshDistance):
        raise TypeError(f'dst must be a MeshDistance, got {type(dst).__name__}')
    check_args(init, samples, seed, max_distance, max_iters)
    pts = source_points(src, samples, seed)
    return register(_Gpu(pts, dst, sample_surface(dst.verts, dst.tris, samples, seed + 1)), bool(rigid), init, max_distance, max_iters)
