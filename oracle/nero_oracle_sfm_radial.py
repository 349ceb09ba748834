"""numpy fp64 restatement of the SIMPLE_RADIAL bundle-adjustment kernels (include/nero_sfm_radial.h) in the protocol of
nero_b200/sfm.py: residuals and Jacobians through the distortion, the Schur elimination of the points, the reduced
camera system with two columns (f, k) per camera, the back-substitution and the cost.  The pinhole statements stay in
nero_oracle_sfm.py, whose track, P3P and triangulation functions the radial mapper reuses on undistorted keypoints.

Also a synthetic project rendered through the distortion: every pixel centre is inverted with
nero_oracle_undistort.undistort and its ray is cast into the table / box / sphere scene of nero_oracle_mvs.
"""
import os

import numpy as np

import nero_oracle_mvs as OM
import nero_oracle_objprep as OOp
import nero_oracle_sfm as OS
import nero_oracle_undistort as OU

NC = 8          # camera-side columns per observation: (w, t, f, k)


# ------------------------------------------------------------------------------------------------ bundle adjustment
def linearize(pose, focal, radial, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    """Per observation: residual r [2] (distorted projection - observation), Jc [2, 8] (rotation update w (left),
    t, f, k) and Jp [2, 3]."""
    n = obs_img.shape[0]
    res, Jc, Jp = np.zeros((n, 2)), np.zeros((n, 2, NC)), np.zeros((n, 2, 3))
    for o in range(n):
        i, p = obs_img[o], obs_pt[o]
        c = img_cam[i]
        R, t = pose[i, :9].reshape(3, 3), pose[i, 9:]
        RX = R @ X[p]
        Y = RX + t
        f, k = focal[c], radial[c]
        x, y = Y[0] / Y[2], Y[1] / Y[2]
        r2 = x * x + y * y
        d = 1.0 + k * r2
        res[o] = ((f * x) * d + pp[c, 0] - obs_xy[o, 0], (f * y) * d + pp[c, 1] - obs_xy[o, 1])
        dxy = f * np.array([[d + 2 * k * x * x, 2 * k * x * y], [2 * k * x * y, d + 2 * k * y * y]])
        dY = dxy @ (np.array([[1, 0, -x], [0, 1, -y]]) / Y[2])
        Jc[o, :, :3] = dY @ -OS._hat(RX)
        Jc[o, :, 3:6] = dY
        Jc[o, :, 6] = (x * d, y * d)
        Jc[o, :, 7] = (f * x * r2, f * y * r2)
        Jp[o] = dY @ R
    return res, Jc, Jp


def residuals(pose, focal, radial, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    """Residuals [2 n] of the model, vectorised, for an independent solver and for finite differences."""
    R = pose[:, :9].reshape(-1, 3, 3)[obs_img]
    Y = np.einsum('nij,nj->ni', R, X[obs_pt]) + pose[obs_img, 9:]
    c = img_cam[obs_img]
    xy = Y[:, :2] / Y[:, 2:]
    d = 1.0 + radial[c, None] * (xy ** 2).sum(1, keepdims=True)
    return ((focal[c, None] * xy) * d + pp[c] - obs_xy).reshape(-1)


def eliminate_points(pt_off, res, Jc, Jp, lam, fix_points=False):
    """nero_oracle_sfm.eliminate_points for 8-column Jc: Vinv [P, 3, 3], gp [P, 3], Y [n, 8, 3]."""
    P = pt_off.shape[0] - 1
    Vinv, gp = np.zeros((P, 3, 3)), np.zeros((P, 3))
    Y = np.zeros((Jc.shape[0], NC, 3))
    for p in range(P):
        s = slice(pt_off[p], pt_off[p + 1])
        V = np.einsum('oki,okj->ij', Jp[s], Jp[s])
        gp[p] = np.einsum('oki,ok->i', Jp[s], res[s])
        V[np.diag_indices(3)] *= 1 + lam
        if fix_points or not np.linalg.det(V) > 0:
            continue
        Vinv[p] = np.linalg.inv(V)
        Y[s] = np.einsum('oka,okb->oab', Jc[s], Jp[s]) @ Vinv[p]
    return Vinv, gp, Y


def columns(nimg, ncam):
    """Columns of the reduced system: image k's (w, t) at 6 k, camera c's f at 6 nimg + 2 c and k at 6 nimg + 2 c + 1."""
    return 6 * nimg + 2 * ncam


def reduced_system(obs_img, img_cam, pt_off, res, Jc, Jp, Y, gp, lam, fixed, nimg, ncam):
    """nero_oracle_sfm.reduced_system with the two camera columns (f, k)."""
    n = columns(nimg, ncam)
    S, U, b = np.zeros((n, n)), np.zeros((n, n)), np.zeros(n)
    cols = lambda o: list(range(6 * obs_img[o], 6 * obs_img[o] + 6)) + [6 * nimg + 2 * img_cam[obs_img[o]] + e for e in (0, 1)]
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


def camera_step(dc, i, img_cam, nimg):
    """The 8 camera-side entries (w, t, f, k) of dc for image i."""
    c = img_cam[i]
    return np.concatenate([dc[6 * i:6 * i + 6], dc[6 * nimg + 2 * c:6 * nimg + 2 * c + 2]])


def back_substitute(obs_img, img_cam, pt_off, Jc, Jp, Vinv, gp, dc, nimg):
    """dX_p = -V_p^-1 (g_p + sum_o W_o^T dc_o) with W_o = Jc_o^T Jp_o [8, 3]."""
    P = pt_off.shape[0] - 1
    dX = np.zeros((P, 3))
    for p in range(P):
        acc = gp[p].copy()
        for o in range(pt_off[p], pt_off[p + 1]):
            acc += (Jc[o].T @ Jp[o]).T @ camera_step(dc, obs_img[o], img_cam, nimg)
        dX[p] = -Vinv[p] @ acc
    return dX


def apply_update(pose, focal, radial, X, dc, dX, nimg):
    """New parameters: R <- exp(w) R, t <- t + dt, f <- f + df, k <- k + dk, X <- X + dX."""
    out = pose.copy()
    for i in range(pose.shape[0]):
        out[i, :9] = (OS.rodrigues(dc[6 * i:6 * i + 3]) @ pose[i, :9].reshape(3, 3)).reshape(-1)
        out[i, 9:] = pose[i, 9:] + dc[6 * i + 3:6 * i + 6]
    return out, focal + dc[6 * nimg::2], radial + dc[6 * nimg + 1::2], X + dX


def cost(pose, focal, radial, pp, img_cam, X, obs_img, obs_pt, obs_xy):
    return float((residuals(pose, focal, radial, pp, img_cam, X, obs_img, obs_pt, obs_xy) ** 2).sum())


def lm_step(pr, lam):
    """One damped Gauss-Newton step from problem dict pr (with 'radial') -> (pose, focal, radial, X, intermediates)."""
    obs_pt = np.repeat(np.arange(pr['X'].shape[0]), np.diff(pr['pt_off']))
    res, Jc, Jp = linearize(pr['pose'], pr['focal'], pr['radial'], pr['pp'], pr['img_cam'], pr['X'], pr['obs_img'], obs_pt, pr['obs_xy'])
    Vinv, gp, Y = eliminate_points(pr['pt_off'], res, Jc, Jp, lam)
    nimg, ncam = pr['pose'].shape[0], pr['focal'].shape[0]
    S, b = reduced_system(pr['obs_img'], pr['img_cam'], pr['pt_off'], res, Jc, Jp, Y, gp, lam, pr['fixed'], nimg, ncam)
    dc = np.linalg.solve(S, b)
    dX = back_substitute(pr['obs_img'], pr['img_cam'], pr['pt_off'], Jc, Jp, Vinv, gp, dc, nimg)
    pose, focal, radial, X = apply_update(pr['pose'], pr['focal'], pr['radial'], pr['X'], dc, dX, nimg)
    return pose, focal, radial, X, dict(res=res, Jc=Jc, Jp=Jp, Vinv=Vinv.reshape(-1, 9), gp=gp, Y=Y, S=S, b=b, dc=dc, dX=dX)


def synthetic_problem(n_cams=4, n_pts=200, noise=0.5, seed=0, shared_camera=False, perturb=True, radial=-0.15):
    """nero_oracle_sfm.synthetic_problem's cameras and points, observed through SIMPLE_RADIAL k = radial with Gaussian
    noise (px, its own seeded stream) -> the same dict plus 'radial' [ncam] (the start: k + 0.02 N(0, 1) when perturbed)
    and fixed [6 n_cams + 2 ncam] with the same gauge; truth gains 'radial'."""
    bp = OS.synthetic_problem(n_cams, n_pts, noise=0.0, seed=seed, shared_camera=shared_camera, perturb=perturb)
    tr = bp['truth']
    ncam = tr['focal'].shape[0]
    k = np.full(ncam, float(radial))
    obs_pt = np.repeat(np.arange(n_pts), np.diff(bp['pt_off']))
    rng = np.random.RandomState(seed + 1000)
    exact = residuals(tr['pose'], tr['focal'], k, bp['pp'], bp['img_cam'], tr['X'], bp['obs_img'], obs_pt, np.zeros_like(bp['obs_xy']))
    bp['obs_xy'] = exact.reshape(-1, 2) + noise * rng.randn(*bp['obs_xy'].shape)
    bp['radial'] = k + 0.02 * rng.randn(ncam) if perturb else k.copy()
    fixed = np.zeros(6 * n_cams + 2 * ncam, np.uint8)
    fixed[:6 * n_cams] = bp['fixed'][:6 * n_cams]
    bp['fixed'] = fixed
    tr['radial'] = k
    return bp


# ------------------------------------------------------------------------------------------------ distorted renders
def cast(pose, dc, cell=0.03):
    """nero_oracle_mvs.render's ray cast for camera-frame ray directions dc [n, 3] (z = 1) -> (rgb uint8 [n, 3], z-depth
    [n], 0 on a miss)."""
    up, e1, e2, o = OM.frame()
    P = np.asarray(pose, np.float64)
    R, t = P[:, :3], P[:, 3]
    C = -R.T @ t
    dw = dc @ R
    n = dw.shape[0]
    best = np.full(n, np.inf)
    surf = np.full(n, -1)
    with np.errstate(all='ignore'):
        tt = ((o - C) @ up) / (dw @ up)
        hit = C + tt[:, None] * dw - o
        rad = np.linalg.norm(hit - (hit @ up)[:, None] * up, axis=1)
        upd = (tt > 0) & (rad <= OM.TABLE_R) & (tt < best)
        best[upd], surf[upd] = tt[upd], 0
        B = np.stack([e1, e2, up])
        cl, dl = B @ (C - o), dw @ B.T
        lo, hi = np.asarray([-OM.BOX_HALF, -OM.BOX_HALF, 0.0]), np.asarray([OM.BOX_HALF, OM.BOX_HALF, OM.BOX_H])
        t1, t2 = (lo - cl) / dl, (hi - cl) / dl
        tn, tf = np.minimum(t1, t2).max(1), np.maximum(t1, t2).min(1)
        upd = (tn <= tf) & (tn > 0) & (tn < best)
        best[upd], surf[upd] = tn[upd], 1
        oc = C - (o + OM.SPHERE_H * up)
        a, b = (dw * dw).sum(1), dw @ oc
        disc = b * b - a * (oc @ oc - OM.SPHERE_R ** 2)
        ts = (-b - np.sqrt(disc)) / a
        upd = (disc >= 0) & (ts > 0) & (ts < best)
        best[upd], surf[upd] = ts[upd], 2
    hitp = C + np.where(np.isfinite(best), best, 0)[:, None] * dw
    rgb = np.zeros((n, 3))
    m = surf >= 0
    rgb[m] = OM.albedo(hitp[m], surf[m], cell)
    return np.clip(np.round(rgb * 255), 0, 255).astype(np.uint8), np.where(m, best, 0.0)


def render(pose, f, cx, cy, k, w, h, cell=0.03):
    """uint8 [h, w, 3] of SIMPLE_RADIAL camera (f, cx, cy, k): each pixel centre inverted, then its ray cast."""
    ys, xs = np.mgrid[0:h, 0:w]
    x, y, ok = OU.undistort(xs.reshape(-1) + 0.5, ys.reshape(-1) + 0.5, f, cx, cy, k)
    assert ok.all(), 'the distortion is not invertible over the image'
    rgb, _ = cast(pose, np.stack([x, y, np.ones_like(x)], 1), cell)
    return rgb.reshape(h, w, 3)


def _render_job(a):
    return render(*a)


def project(root, n_views, w, h, k, seed=0, cell=0.03, focal=0.9, workers=1):
    """<root>/images/img_XXX.png of nero_oracle_mvs.project's views (same poses for the same seed), rendered through
    SIMPLE_RADIAL (f = focal w, w / 2, h / 2, k).  No model is written.  -> dict(names, poses [n, 3, 4], K, k, up)."""
    import cv2
    sc = OOp.scene(n_table=10, n_obj=10, outlier_frac=0.0, n_cams=n_views, seed=seed)
    f, cx, cy = focal * w, w / 2, h / 2
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    names = [f'img_{i:03d}.png' for i in range(n_views)]
    jobs = [(P, f, cx, cy, k, w, h, cell) for P in sc['poses']]
    if workers > 1:
        import multiprocessing
        with multiprocessing.get_context('fork').Pool(workers) as pool:
            imgs = pool.map(_render_job, jobs)
    else:
        imgs = [render(*a) for a in jobs]
    for name, img in zip(names, imgs):
        cv2.imwrite(os.path.join(root, 'images', name), np.ascontiguousarray(img[..., ::-1]))
    K = np.asarray([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)
    return dict(names=names, poses=sc['poses'], K=K, k=float(k), up=sc['up'], center=sc['center'])
