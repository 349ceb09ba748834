"""numpy fp64 restatement of the structure-from-motion kernels of k_sfm.cu (include/nero_sfm.h), in the protocol of
nero_b200/sfm.py: track building, the Lambda Twist P3P solver and its RANSAC, multi-view DLT triangulation, and the
pieces of one Levenberg-Marquardt iteration of bundle adjustment (residuals and Jacobians, the Schur elimination of the
points, the reduced camera system and the back-substitution).

There is no reference code to pin the kernels against: the reference workflow runs COLMAP's CPU mapper.  This file states
what the kernels compute instead, with their operation order where a result is compared bit for bit (tracks, P3P
winners) and their algorithm elsewhere (fp64 results agree to rounding).
"""
import numpy as np

import nero_oracle_objprep as OOp


# ------------------------------------------------------------------------------------------------ small linear algebra
def jacobi(A, sweeps):
    """Cyclic Jacobi of the symmetric matrix A -> (diagonal after the sweeps, eigenvectors as columns)."""
    A = np.array(A, np.float64)
    n = A.shape[0]
    V = np.eye(n)
    for _ in range(sweeps):
        for p in range(n - 1):
            for q in range(p + 1, n):
                apq = A[p, q]
                if apq == 0.0:
                    continue
                with np.errstate(over='ignore'):
                    theta = (A[q, q] - A[p, p]) / (2.0 * apq)
                    t = (1.0 if theta >= 0.0 else -1.0) / (abs(theta) + np.sqrt(theta * theta + 1.0))
                c = 1.0 / np.sqrt(t * t + 1.0)
                s = t * c
                Ap, Aq = A[:, p].copy(), A[:, q].copy()
                A[:, p], A[:, q] = c * Ap - s * Aq, s * Ap + c * Aq
                Ap, Aq = A[p, :].copy(), A[q, :].copy()
                A[p, :], A[q, :] = c * Ap - s * Aq, s * Ap + c * Aq
                Vp, Vq = V[:, p].copy(), V[:, q].copy()
                V[:, p], V[:, q] = c * Vp - s * Vq, s * Vp + c * Vq
    return np.diag(A).copy(), V


def rodrigues(w):
    th = np.linalg.norm(w)
    K = np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    if th < 1e-12:
        return np.eye(3) + K
    return np.eye(3) + np.sin(th) / th * K + (1 - np.cos(th)) / th ** 2 * K @ K


def _hat(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


# ------------------------------------------------------------------------------------------------ tracks
def tracks(edges, n):
    """Union-find components of n nodes under edges [E, 2] -> (label [n] = the smallest node of its component,
    track [n] = the rank of that label among the roots)."""
    parent = np.arange(n)

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x
    for a, b in np.asarray(edges, np.int64).reshape(-1, 2):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    label = np.array([find(v) for v in range(n)], np.int64)
    roots = np.nonzero(label == np.arange(n))[0]
    rank = np.full(n, -1, np.int64)
    rank[roots] = np.arange(roots.shape[0])
    return label, rank[label]


# ------------------------------------------------------------------------------------------------ P3P (Lambda Twist)
def _real_roots_cubic(c3, c2, c1, c0):
    r = np.roots([c3, c2, c1, c0])
    return np.sort(r[np.abs(r.imag) <= 1e-9 * (1 + np.abs(r.real))].real)


def p3p(y, x):
    """Poses (R, t), x_cam = R x + t, of unit bearings y [3, 3] toward world points x [3, 3]: at most 4, each with
    positive depths.  Lambda Twist: the pencil D1 + g D2 of the two homogeneous conics, one real root g of its cubic, the
    plane pair of the degenerate conic, the positive solutions of each plane, two Gauss-Newton steps on the depths, and
    the rotation from the two difference vectors and their cross product."""
    y = np.asarray(y, np.float64)
    x = np.asarray(x, np.float64)
    b12, b13, b23 = -2 * y[0] @ y[1], -2 * y[0] @ y[2], -2 * y[1] @ y[2]
    a12, a13, a23 = [float(np.sum((x[i] - x[j]) ** 2)) for i, j in ((0, 1), (0, 2), (1, 2))]
    M12 = np.array([[1, b12 / 2, 0], [b12 / 2, 1, 0], [0, 0, 0]])
    M13 = np.array([[1, 0, b13 / 2], [0, 0, 0], [b13 / 2, 0, 1]])
    M23 = np.array([[0, 0, 0], [0, 1, b23 / 2], [0, b23 / 2, 1]])
    D1 = M12 * a23 - M23 * a12
    D2 = M13 * a23 - M23 * a13
    det = np.linalg.det
    c3 = det(D2)
    c0 = det(D1)
    c2 = det(np.stack([D1[:, 0], D2[:, 1], D2[:, 2]], 1)) + det(np.stack([D2[:, 0], D1[:, 1], D2[:, 2]], 1)) + \
        det(np.stack([D2[:, 0], D2[:, 1], D1[:, 2]], 1))
    c1 = det(np.stack([D2[:, 0], D1[:, 1], D1[:, 2]], 1)) + det(np.stack([D1[:, 0], D2[:, 1], D1[:, 2]], 1)) + \
        det(np.stack([D1[:, 0], D1[:, 1], D2[:, 2]], 1))
    g = _real_roots_cubic(c3, c2, c1, c0)
    if g.shape[0] == 0:
        return []
    g = g[-1]
    D0 = D1 + g * D2
    ev, E = np.linalg.eigh(D0)
    order = np.argsort(-np.abs(ev))
    s1, s2 = ev[order[0]], ev[order[1]]
    u1, u2 = E[:, order[0]], E[:, order[1]]
    if s1 * s2 > 0 or s1 == 0:
        return []
    s = np.sqrt(-s2 / s1)
    out = []
    for sg in (1.0, -1.0):
        nrm = u1 - sg * s * u2                               # lambda . nrm = 0
        k = int(np.argmax(np.abs(nrm)))
        i, j = [m for m in range(3) if m != k]
        # lambda_k = w_i lambda_i + w_j lambda_j
        wi, wj = -nrm[i] / nrm[k], -nrm[j] / nrm[k]
        # quadratic in tau = lambda_i / lambda_j from lambda^T D2 lambda = 0
        e = np.zeros((3, 2))
        e[i, 0], e[j, 1], e[k] = 1, 1, (wi, wj)
        Q = e.T @ D2 @ e
        for tau in _quad_roots(Q[0, 0], 2 * Q[0, 1], Q[1, 1]):
            d = e @ np.array([tau, 1.0])
            q = d @ M23 @ d
            if q <= 0:
                continue
            lam = d * np.sqrt(a23 / q)
            if lam[j] < 0:
                lam = -lam
            if np.all(lam > 0):
                lam = _refine_depths(lam, b12, b13, b23, a12, a13, a23)
                out.append(_pose_from_depths(lam, y, x))
    return out


def _quad_roots(a, b, c):
    disc = b * b - 4 * a * c
    if disc < 0:
        return []
    sq = np.sqrt(disc)
    if a == 0:
        return [] if b == 0 else [-c / b]
    q = -0.5 * (b + (sq if b >= 0 else -sq))
    r1 = q / a
    r2 = c / q if q != 0 else r1
    return [r1, r2]


def _refine_depths(lam, b12, b13, b23, a12, a13, a23, steps=2):
    l = np.array(lam, np.float64)
    for _ in range(steps):
        r = np.array([l[0] ** 2 + l[1] ** 2 + b12 * l[0] * l[1] - a12, l[0] ** 2 + l[2] ** 2 + b13 * l[0] * l[2] - a13,
                      l[1] ** 2 + l[2] ** 2 + b23 * l[1] * l[2] - a23])
        J = np.array([[2 * l[0] + b12 * l[1], 2 * l[1] + b12 * l[0], 0], [2 * l[0] + b13 * l[2], 0, 2 * l[2] + b13 * l[0]],
                      [0, 2 * l[1] + b23 * l[2], 2 * l[2] + b23 * l[1]]])
        dt = np.linalg.det(J)
        if dt == 0:
            break
        l = l - np.linalg.solve(J, r)
    return l


def _pose_from_depths(lam, y, x):
    Y = lam[:, None] * y
    a, b = Y[0] - Y[1], Y[0] - Y[2]
    c, d = x[0] - x[1], x[0] - x[2]
    My = np.stack([a, b, np.cross(a, b)], 1)
    Mx = np.stack([c, d, np.cross(c, d)], 1)
    R = My @ np.linalg.inv(Mx)
    return R, Y[0] - R @ x[0]


def draw_key(seed, image, hyp, draw):
    with np.errstate(over='ignore'):
        h = OOp._mix(np.uint32(seed) * np.uint32(0x9e3779b9) + np.uint32(0x7f4a7c15))
        h = OOp._mix(h ^ np.uint32(image))
        h = OOp._mix(h ^ np.uint32(hyp))
        return int(OOp._mix(h ^ np.uint32(draw)))


def bearings(xy, f, cx, cy):
    v = np.stack([(xy[:, 0] - cx) / f, (xy[:, 1] - cy) / f, np.ones(xy.shape[0])], 1)
    return v / np.linalg.norm(v, axis=1, keepdims=True)


def inliers(R, t, xy, X, f, cx, cy, max_err2):
    Y = X @ R.T + t
    with np.errstate(all='ignore'):
        e = (f * Y[:, 0] / Y[:, 2] + cx - xy[:, 0]) ** 2 + (f * Y[:, 1] / Y[:, 2] + cy - xy[:, 1]) ** 2
    return (Y[:, 2] > 0) & (e <= max_err2)


def p3p_ransac(xy, X, f, cx, cy, image, hypotheses, seed, max_err2, max_draws=32):
    """-> (pose [12] (R row-major, t), winning hypothesis, its count, inlier bool [n], counts [H]).  Hypothesis h draws 3
    distinct correspondences by draw_key(seed, image, h, d) mod n; its best solution (ties: the first) is its count."""
    n = xy.shape[0]
    y = bearings(xy, f, cx, cy)
    counts = np.full(hypotheses, -1, np.int64)
    poses = np.zeros((hypotheses, 12))
    for h in range(hypotheses):
        idx = []
        for d in range(max_draws):
            if len(idx) == 3:
                break
            m = draw_key(seed, image, h, d) % n
            if m not in idx:
                idx.append(m)
        if len(idx) < 3:
            continue
        for R, t in p3p(y[idx], X[idx]):
            c = int(inliers(R, t, xy, X, f, cx, cy, max_err2).sum())
            if c > counts[h]:
                counts[h] = c
                poses[h] = np.concatenate([R.reshape(-1), t])
    w = int(np.argmax(counts))                              # the first of the largest
    pose = poses[w]
    inl = inliers(pose[:9].reshape(3, 3), pose[9:], xy, X, f, cx, cy, max_err2) if counts[w] >= 0 else np.zeros(n, bool)
    return pose, w, int(max(counts[w], 0)), inl, counts


# ------------------------------------------------------------------------------------------------ triangulation
def triangulate(poses, f, pp, xy):
    """DLT point of one track: poses [m, 12], focal [m], principal points [m, 2], observations xy [m, 2] -> X [3].  Rows
    x^ P3 - P1, y^ P3 - P2 on normalised coordinates, their 4 x 4 normal matrix summed in observation order, the
    eigenvector of its smallest Jacobi diagonal entry (10 sweeps)."""
    A = np.zeros((4, 4))
    for P, fk, c, x in zip(poses, f, pp, xy):
        Pm = np.concatenate([P[:9].reshape(3, 3), P[9:, None]], 1)
        u, v = (x[0] - c[0]) / fk, (x[1] - c[1]) / fk
        for row in (u * Pm[2] - Pm[0], v * Pm[2] - Pm[1]):
            A += np.outer(row, row)
    d, V = jacobi(A, 10)
    e = V[:, int(np.argmin(d))]
    return e[:3] / e[3]


def track_stats(X, poses, f, pp, xy):
    """(depths [m], reprojection errors [m] (px), the largest pairwise angle (radians) between the rays to X)."""
    R = poses[:, :9].reshape(-1, 3, 3)
    t = poses[:, 9:]
    Y = np.einsum('mij,j->mi', R, X) + t
    err = np.hypot(f * Y[:, 0] / Y[:, 2] + pp[:, 0] - xy[:, 0], f * Y[:, 1] / Y[:, 2] + pp[:, 1] - xy[:, 1])
    C = -np.einsum('mji,mj->mi', R, t)
    r = X - C
    r = r / np.linalg.norm(r, axis=1, keepdims=True)
    cos = np.clip(r @ r.T, -1, 1)
    return Y[:, 2], err, float(np.arccos(cos.min())) if r.shape[0] > 1 else 0.0


# ------------------------------------------------------------------------------------------------ bundle adjustment
def linearize(pose, focal, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    """Per observation: residual r [2] (projection - observation), Jc [2, 7] (rotation update w (left, exp(w) R), t,
    focal) and Jp [2, 3] (the point)."""
    n = obs_img.shape[0]
    res, Jc, Jp = np.zeros((n, 2)), np.zeros((n, 2, 7)), np.zeros((n, 2, 3))
    for o in range(n):
        i, p = obs_img[o], obs_pt[o]
        c = img_cam[i]
        R, t = pose[i, :9].reshape(3, 3), pose[i, 9:]
        RX = R @ X[p]
        Y = RX + t
        f = focal[c]
        iz = 1.0 / Y[2]
        u, v = Y[0] * iz, Y[1] * iz
        res[o] = (f * u + pp[c, 0] - obs_xy[o, 0], f * v + pp[c, 1] - obs_xy[o, 1])
        dY = f * iz * np.array([[1, 0, -u], [0, 1, -v]])
        Jc[o, :, :3] = dY @ -_hat(RX)
        Jc[o, :, 3:6] = dY
        Jc[o, :, 6] = (u, v)
        Jp[o] = dY @ R
    return res, Jc, Jp


def eliminate_points(pt_off, res, Jc, Jp, lam, fix_points=False):
    """Per point: V = sum Jp^T Jp (diagonal times 1 + lam), V^-1 (adjugate; 0 when fixed or singular), g = sum Jp^T r;
    per observation Y = W V^-1 with W = Jc^T Jp [7, 3]."""
    P = pt_off.shape[0] - 1
    Vinv, gp = np.zeros((P, 3, 3)), np.zeros((P, 3))
    Y = np.zeros((Jc.shape[0], 7, 3))
    for p in range(P):
        V = np.zeros((3, 3))
        g = np.zeros(3)
        for o in range(pt_off[p], pt_off[p + 1]):
            V += Jp[o].T @ Jp[o]
            g += Jp[o].T @ res[o]
        V[np.diag_indices(3)] *= 1 + lam
        gp[p] = g
        d = np.linalg.det(V)
        if fix_points or not d > 0:
            continue
        Vinv[p] = np.linalg.inv(V)
        for o in range(pt_off[p], pt_off[p + 1]):
            Y[o] = (Jc[o].T @ Jp[o]) @ Vinv[p]
    return Vinv, gp, Y


def columns(nimg, ncam):
    """Column of each parameter of the reduced system: image k's (w, t) at 6 k, camera c's focal at 6 nimg + c."""
    return 6 * nimg + ncam


def reduced_system(obs_img, img_cam, pt_off, res, Jc, Jp, Y, gp, lam, fixed, nimg, ncam):
    """S [n, n], b [n]: S = U (diagonal times 1 + lam) - sum_p sum_(o, o' of p) Y_o W_o'^T, b = -(g_c - sum_o Y_o g_p),
    with rows and columns of fixed parameters replaced by the identity (b = 0)."""
    n = columns(nimg, ncam)
    S, U, b = np.zeros((n, n)), np.zeros((n, n)), np.zeros(n)
    obs_pt = np.repeat(np.arange(pt_off.shape[0] - 1), np.diff(pt_off))
    cols = lambda o: list(range(6 * obs_img[o], 6 * obs_img[o] + 6)) + [6 * nimg + img_cam[obs_img[o]]]
    for p in range(pt_off.shape[0] - 1):
        for o in range(pt_off[p], pt_off[p + 1]):
            co = cols(o)
            U[np.ix_(co, co)] += Jc[o].T @ Jc[o]
            b[co] -= Jc[o].T @ res[o] - Y[o] @ gp[p]
            for o2 in range(pt_off[p], pt_off[p + 1]):
                S[np.ix_(co, cols(o2))] -= Y[o] @ (Jc[o2].T @ Jp[o2]).T
    S += U
    S[np.diag_indices(n)] += lam * np.diag(U)
    fx = np.asarray(fixed, bool)
    S[fx, :] = 0
    S[:, fx] = 0
    S[fx, fx] = 1
    b[fx] = 0
    d = np.diag(S).copy()
    S[np.diag_indices(n)] = np.where(d == 0, 1.0, d)
    return S, b


def back_substitute(obs_img, img_cam, pt_off, Jc, Jp, Vinv, gp, dc, nimg):
    """dX_p = -V_p^-1 (g_p + sum_o W_o^T dc_o)."""
    P = pt_off.shape[0] - 1
    dX = np.zeros((P, 3))
    for p in range(P):
        acc = gp[p].copy()
        for o in range(pt_off[p], pt_off[p + 1]):
            i = obs_img[o]
            d7 = np.concatenate([dc[6 * i:6 * i + 6], [dc[6 * nimg + img_cam[i]]]])
            acc += (Jc[o].T @ Jp[o]).T @ d7
        dX[p] = -Vinv[p] @ acc
    return dX


def apply_update(pose, focal, X, dc, dX, nimg):
    """New parameters: R <- exp(w) R, t <- t + dt, f <- f + df, X <- X + dX."""
    out = pose.copy()
    for i in range(pose.shape[0]):
        w, dt = dc[6 * i:6 * i + 3], dc[6 * i + 3:6 * i + 6]
        out[i, :9] = (rodrigues(w) @ pose[i, :9].reshape(3, 3)).reshape(-1)
        out[i, 9:] = pose[i, 9:] + dt
    return out, focal + dc[6 * nimg:], X + dX


def cost(pose, focal, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    r = linearize(pose, focal, pp, img_cam, X, obs_img, obs_pt, obs_xy)[0]
    return float((r ** 2).sum())


def residuals(pose, focal, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    """Residuals [2 n] of the model, for an independent solver."""
    R = pose[:, :9].reshape(-1, 3, 3)[obs_img]
    Y = np.einsum('nij,nj->ni', R, X[obs_pt]) + pose[obs_img, 9:]
    c = img_cam[obs_img]
    return np.concatenate([focal[c, None] * Y[:, :2] / Y[:, 2:] + pp[c] - obs_xy], 1).reshape(-1)


# ------------------------------------------------------------------------------------------------ synthetic problems
def synthetic_problem(n_cams=4, n_pts=200, noise=0.5, seed=0, shared_camera=False, perturb=True):
    """A seeded bundle-adjustment problem without images: cameras on an arc looking at a cloud of points, every point seen
    by 2..n_cams cameras, observations with Gaussian noise (px), and a perturbed start.  -> dict of the kernels' arrays
    (pose, focal, pp, img_cam, X, pt_off, obs_img, obs_xy, fixed with the gauge of nero_b200.sfm) and the truth."""
    rng = np.random.RandomState(seed)
    w, h, f = 640.0, 480.0, 560.0
    pose = np.zeros((n_cams, 12))
    for i in range(n_cams):
        a = np.radians(-30 + 60 * i / max(n_cams - 1, 1))
        C = np.array([4 * np.sin(a), 0.3 * rng.randn(), -4 * np.cos(a)])
        z = -C / np.linalg.norm(C)
        x = np.cross([0, 1, 0], z)
        x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        pose[i] = np.concatenate([R.reshape(-1), -R @ C])
    ncam = 1 if shared_camera else n_cams
    focal = f * (1 + 0.02 * rng.randn(ncam))
    pp = np.tile([w / 2, h / 2], (ncam, 1))
    img_cam = np.zeros(n_cams, np.int64) if shared_camera else np.arange(n_cams)
    X = rng.uniform(-1, 1, (n_pts, 3))
    obs_img, obs_xy, off = [], [], [0]
    for p in range(n_pts):
        k = rng.randint(2, n_cams + 1)
        cams = np.sort(rng.choice(n_cams, k, replace=False))
        for i in cams:
            R, t = pose[i, :9].reshape(3, 3), pose[i, 9:]
            Y = R @ X[p] + t
            c = img_cam[i]
            obs_img.append(i)
            obs_xy.append(focal[c] * Y[:2] / Y[2] + pp[c] + noise * rng.randn(2))
        off.append(len(obs_img))
    fixed = np.zeros(6 * n_cams + ncam, np.uint8)
    fixed[:6] = 1
    fixed[6 + 3 + int(np.argmax(np.abs(pose[1, 9:])))] = 1
    start = dict(pose=pose.copy(), focal=focal.copy(), X=X.copy())
    if perturb:
        for i in range(n_cams):
            if i == 0:
                continue
            start['pose'][i, :9] = (rodrigues(0.01 * rng.randn(3)) @ pose[i, :9].reshape(3, 3)).reshape(-1)
            dt = 0.02 * rng.randn(3)
            if i == 1:
                dt[int(np.argmax(np.abs(pose[1, 9:])))] = 0
            start['pose'][i, 9:] += dt
        start['focal'] = focal * (1 + 0.03 * rng.randn(ncam))
        start['X'] = X + 0.02 * rng.randn(n_pts, 3)
    return dict(pose=start['pose'], focal=start['focal'], pp=pp, img_cam=img_cam, X=start['X'], pt_off=np.asarray(off, np.int64),
                obs_img=np.asarray(obs_img, np.int64), obs_xy=np.asarray(obs_xy), fixed=fixed,
                truth=dict(pose=pose, focal=focal, X=X))


def lm_step(pr, lam):
    """One damped Gauss-Newton step of the oracle from problem dict pr -> (pose, focal, X, dict of the intermediates)."""
    obs_pt = np.repeat(np.arange(pr['X'].shape[0]), np.diff(pr['pt_off']))
    res, Jc, Jp = linearize(pr['pose'], pr['focal'], pr['pp'], pr['img_cam'], pr['X'], pr['obs_img'], obs_pt, pr['obs_xy'])
    Vinv, gp, Y = eliminate_points(pr['pt_off'], res, Jc, Jp, lam)
    nimg, ncam = pr['pose'].shape[0], pr['focal'].shape[0]
    S, b = reduced_system(pr['obs_img'], pr['img_cam'], pr['pt_off'], res, Jc, Jp, Y, gp, lam, pr['fixed'], nimg, ncam)
    dc = np.linalg.solve(S, b)
    dX = back_substitute(pr['obs_img'], pr['img_cam'], pr['pt_off'], Jc, Jp, Vinv, gp, dc, nimg)
    pose, focal, X = apply_update(pr['pose'], pr['focal'], pr['X'], dc, dX, nimg)
    return pose, focal, X, dict(res=res, Jc=Jc, Jp=Jp, Vinv=Vinv.reshape(-1, 9), gp=gp, Y=Y, S=S, b=b, dc=dc, dX=dX)
