"""Structure from motion on the GPU: the kernels of k_sfm.cu against the fp64 oracle (oracle/nero_oracle_sfm.py), the
bundle adjustment against scipy's least-squares solver, and the whole mapper on the synthetic table / box / sphere
projects: accuracy against the true cameras, run-to-run identity of the model, a disconnected database, and the workflow
from images to the prepared object with no COLMAP and no true poses."""
import importlib.util
import os
import shutil

import numpy as np
import pytest
import torch

import nero_oracle_mvs as OM
import nero_oracle_sfm as OS
from nero_b200 import features as Ft
from nero_b200 import objprep as OP
from nero_b200 import sfm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _rel(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / max(np.abs(np.asarray(b)).max(), 1e-300))


def _problem(bp, fix_points=False):
    return sfm.Problem(bp['pose'], bp['focal'], bp['pp'], bp['img_cam'], bp['X'], bp['pt_off'], bp['obs_img'], bp['obs_xy'], bp['fixed'],
                       fix_points)


@pytest.mark.parametrize('shared', [False, True])
def test_bundle_adjustment_kernels_match_the_oracle(shared):
    bp = OS.synthetic_problem(5, 150, seed=4, shared_camera=shared)
    pr = _problem(bp)
    if shared:     # the focal segments span many chunks: the two-stage sums are exercised
        assert int((pr.seg_chunk[1:] - pr.seg_chunk[:-1]).max()) > 2 and int((pr.rseg_chunk[1:] - pr.rseg_chunk[:-1]).max()) > 1
    pr.linearize()
    lam = 1e-3
    pr.eliminate(lam)
    S, b = pr.reduce(lam)
    dc = torch.linalg.solve(S, b)
    pose, focal, X = pr.backsub(dc)
    opose, ofocal, oX, o = OS.lm_step(bp, lam)
    got = dict(res=pr.res, Jc=pr.Jc, Jp=pr.Jp, Vinv=pr.Vinv, gp=pr.gp, Y=pr.Y, S=S, b=b)
    for k, v in got.items():
        err = _rel(v.cpu().numpy().reshape(o[k].shape), o[k])
        print(f'{k}: {err:.2e}')
        assert err <= 1e-12, f'{k} differs from the oracle by {err:.2e} (relative)'
    assert _rel(dc.cpu().numpy(), o['dc']) <= 1e-9
    assert _rel(X.cpu().numpy() - bp['X'], o['dX']) <= 1e-9
    assert _rel(pose.cpu().numpy(), opose) <= 1e-9 and _rel(focal.cpu().numpy(), ofocal) <= 1e-9
    # back-substitution alone, from the oracle's own camera step
    _, _, X2 = pr.backsub(torch.from_numpy(o['dc']).cuda())
    assert _rel(X2.cpu().numpy() - bp['X'], o['dX']) <= 1e-12
    c = pr.cost()
    obs_pt = np.repeat(np.arange(bp['X'].shape[0]), np.diff(bp['pt_off']))
    oc = OS.cost(bp['pose'], bp['focal'], bp['pp'], bp['img_cam'], bp['X'], bp['obs_img'], obs_pt, bp['obs_xy'])
    assert abs(c - oc) <= 1e-12 * oc


def test_tracks_are_exact():
    rng = np.random.RandomState(7)
    n = 5000
    edges = rng.randint(0, n, (3000, 2))
    label, track, T = sfm.build_tracks(edges, n)
    olabel, otrack = OS.tracks(edges, n)
    assert np.array_equal(label, olabel) and np.array_equal(track, otrack) and T == otrack.max() + 1


def test_triangulation_matches_the_oracle():
    bp = OS.synthetic_problem(6, 300, noise=0.5, seed=5, perturb=False)
    X, st = sfm.triangulate(bp['pt_off'], bp['obs_img'], bp['obs_xy'], bp['pose'], bp['img_cam'], bp['focal'], bp['pp'])
    for p in range(X.shape[0]):
        s = slice(bp['pt_off'][p], bp['pt_off'][p + 1])
        c = bp['img_cam'][bp['obs_img'][s]]
        oX = OS.triangulate(bp['pose'][bp['obs_img'][s]], bp['focal'][c], bp['pp'][c], bp['obs_xy'][s])
        d, e, a = OS.track_stats(oX, bp['pose'][bp['obs_img'][s]], bp['focal'][c], bp['pp'][c], bp['obs_xy'][s])
        assert _rel(X[p], oX) <= 1e-9, p
        assert abs(st[p, 0] - d.min()) <= 1e-9 * abs(d.min()) and abs(st[p, 1] - e.max()) <= 1e-6 and abs(st[p, 2] - a) <= 1e-9
    assert np.median(np.linalg.norm(X - bp['truth']['X'], axis=1)) <= 0.01


def test_p3p_ransac_matches_the_oracle_with_outliers():
    rng = np.random.RandomState(11)
    R = OS.rodrigues(0.4 * rng.randn(3))
    t = np.array([0.2, -0.1, 5.0])
    f, cx, cy = 600.0, 320.0, 240.0
    n = 400
    Xc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(3, 7, n)], 1)
    X = (Xc - t) @ R
    xy = f * Xc[:, :2] / Xc[:, 2:] + [cx, cy]
    out = rng.rand(n) < 0.3
    xy[out] = rng.uniform([0, 0], [640, 480], (int(out.sum()), 2))
    pose, h, cnt, inl, counts = sfm.p3p_ransac(xy, X, f, cx, cy, 17, hypotheses=256)
    opose, oh, ocnt, oinl, ocounts = OS.p3p_ransac(xy, X, f, cx, cy, 17, 256, sfm.SEED, sfm.ABS_POSE_MAX_ERROR ** 2)
    print(f'winner {h} ({cnt}) vs oracle {oh} ({ocnt}); {(counts == ocounts).mean():.3f} of the counts equal')
    assert (h, cnt) == (oh, ocnt) and np.array_equal(inl, oinl)
    assert (counts == ocounts).mean() >= 0.99
    Rg = pose[:9].reshape(3, 3)
    ang = np.degrees(np.arccos(np.clip((np.trace(Rg @ R.T) - 1) / 2, -1, 1)))
    assert ang <= 0.01 and np.abs(pose[9:] - t).max() <= 1e-6 * np.linalg.norm(t) and inl[~out].all()


def _scipy_problem(bp, free):
    """scipy's view of the problem: the free parameters (rotation vectors w with R = exp(w) R_start, t, f, X offsets) ->
    residuals, and their analytic Jacobian (the left Jacobian of SO(3) maps the kernels' rotation columns to w)."""
    nimg, ncam, P = bp['pose'].shape[0], bp['focal'].shape[0], bp['X'].shape[0]
    obs_pt = np.repeat(np.arange(P), np.diff(bp['pt_off']))
    oi, n = bp['obs_img'], bp['obs_img'].shape[0]
    nfull = 6 * nimg + ncam + 3 * P

    def unpack(x):
        full = np.zeros(nfull)
        full[free] = x
        pose = bp['pose'].copy()
        for i in range(nimg):
            pose[i, :9] = (OS.rodrigues(full[6 * i:6 * i + 3]) @ bp['pose'][i, :9].reshape(3, 3)).reshape(-1)
            pose[i, 9:] = bp['pose'][i, 9:] + full[6 * i + 3:6 * i + 6]
        return full, pose, bp['focal'] + full[6 * nimg:6 * nimg + ncam], bp['X'] + full[6 * nimg + ncam:].reshape(-1, 3)

    def fun(x):
        _, pose, focal, X = unpack(x)
        return OS.residuals(pose, focal, bp['pp'], bp['img_cam'], X, oi, obs_pt, bp['obs_xy'])

    def left_jacobian(w):
        th = np.linalg.norm(w)
        K = OS._hat(w)
        if th < 1e-8:
            return np.eye(3) + K / 2
        return np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K

    def jac(x):
        full, pose, focal, X = unpack(x)
        R = pose[oi, :9].reshape(-1, 3, 3)
        RX = np.einsum('nij,nj->ni', R, X[obs_pt])
        Y = RX + pose[oi, 9:]
        c = bp['img_cam'][oi]
        iz = 1 / Y[:, 2]
        u, v = Y[:, 0] * iz, Y[:, 1] * iz
        fz = focal[c] * iz
        dY = np.zeros((n, 2, 3))
        dY[:, 0, 0], dY[:, 0, 2], dY[:, 1, 1], dY[:, 1, 2] = fz, -fz * u, fz, -fz * v
        Jl = np.stack([left_jacobian(full[6 * i:6 * i + 3]) for i in range(nimg)])[oi]
        Hm = -np.stack([OS._hat(r) for r in RX])
        J = np.zeros((n, 2, nfull))
        rows = np.arange(n)
        for k in range(3):
            J[rows, :, 6 * oi + k] = np.einsum('nij,njk->nik', dY, Hm @ Jl)[:, :, k]
            J[rows, :, 6 * oi + 3 + k] = dY[:, :, k]
            J[rows, :, 6 * nimg + ncam + 3 * obs_pt + k] = np.einsum('nij,njk->nik', dY, R)[:, :, k]
        J[rows, 0, 6 * nimg + c] = u
        J[rows, 1, 6 * nimg + c] = v
        return J.reshape(2 * n, nfull)[:, free]
    return fun, jac, unpack


def test_bundle_adjustment_converges_to_scipys_solution():
    from scipy.optimize import least_squares
    bp = OS.synthetic_problem(8, 500, noise=0.5, seed=8)
    pr = _problem(bp)
    info = pr.solve(200, tol=1e-15)
    pose, focal, X = pr.result()
    free = np.nonzero(np.concatenate([bp['fixed'] == 0, np.ones(3 * bp['X'].shape[0], bool)]))[0]
    fun, jac, unpack = _scipy_problem(bp, free)
    sol = least_squares(fun, np.zeros(free.shape[0]), jac=jac, method='lm', ftol=1e-15, xtol=1e-15, gtol=1e-15)
    _, spose, sfocal, sX = unpack(sol.x)
    scost = float((sol.fun ** 2).sum())
    print(f'LM: {info["iterations"]} iterations, cost {info["cost0"]:.6f} -> {info["cost"]:.9f}; scipy ({sol.nfev} evaluations, status '
          f'{sol.status}) {scost:.9f}; pose {_rel(pose, spose):.2e}, focal {_rel(focal, sfocal):.2e}, points {_rel(X, sX):.2e}')
    assert abs(info['cost'] - scost) <= 1e-6 * scost
    assert _rel(pose, spose) <= 1e-6 and _rel(focal, sfocal) <= 1e-6 and _rel(X, sX) <= 1e-6


# ------------------------------------------------------------------------------------------------ the mapper
def _align(C_est, C_true):
    """Similarity (s, R, t) with s R C_est + t ~ C_true (Umeyama)."""
    me, mt = C_est.mean(0), C_true.mean(0)
    A, B = C_est - me, C_true - mt
    U, S, Vt = np.linalg.svd(B.T @ A)
    D = np.eye(3)
    D[2, 2] = np.sign(np.linalg.det(U @ Vt))
    R = U @ D @ Vt
    s = (S * np.diag(D)).sum() / (A ** 2).sum()
    return s, R, mt - s * R @ me


def _accuracy(model_dir, pr):
    import nero_oracle_objprep as OOp  # noqa: F401  (the project's scene)
    views, pts = OP.read_colmap_model(model_dir)
    names = pr['names']
    ids = sorted(views)
    k = [names.index(views[i][0]) for i in ids]
    P = [views[i][1].astype(np.float64) for i in ids]
    C = np.array([-p[:, :3].T @ p[:, 3] for p in P])
    Ct = np.array([-pr['poses'][j][:, :3].T @ pr['poses'][j][:, 3] for j in k])
    s, R, t = _align(C, Ct)
    _, D, _, _ = OP.scene_scale({i: (views[i][0], pr['poses'][j].astype(np.float32), views[i][2]) for i, j in zip(ids, k)})
    cerr = np.linalg.norm(s * C @ R.T + t - Ct, axis=1).max() / D
    rerr = max(np.degrees(np.arccos(np.clip((np.trace(pr['poses'][j][:, :3] @ (p[:, :3] @ R.T).T) - 1) / 2, -1, 1))) for p, j in zip(P, k))
    near = (OM.surface_distance(s * pts @ R.T + t) <= 0.005 * D).mean()
    return dict(registered=len(ids), centre=cerr, rotation=rerr, near=near)


@pytest.fixture(scope='module')
def twelve(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('sfm12'))
    pr = OM.project(root, 12, 640, 480, per_view=10, workers=4)
    shutil.rmtree(os.path.join(root, 'sparse'))
    tool('match_features').main(['--root', root])
    return root, pr


@pytest.mark.parametrize('same', [False, True])
def test_accuracy_on_twelve_views(twelve, tmp_path, same):
    root, pr = twelve
    db = os.path.join(root, 'database.db')
    if same:
        db = str(tmp_path / 'same.db')
        Ft.build_database(os.path.join(root, 'images'), db, same_camera=True)
    out = str(tmp_path / 'model')
    s = tool('map_sparse').main(['--root', root, '--database', db, '--output', out])
    acc = _accuracy(out, pr)
    f_true = pr['K'][0, 0]
    ferr = max(abs(f - f_true) / f_true for f in s['focals'].values())
    print(f'same_camera={same}: {acc}, focal errors up to {100 * ferr:.3f} %, mean error {s["mean_error"]:.3f} px, {s["points"]} points')
    assert acc['registered'] == 12 and not s['unregistered']
    assert acc['rotation'] <= 0.2 and acc['centre'] <= 0.005
    assert ferr <= (0.01 if same else 0.02)
    assert s['mean_error'] <= 1.0 and acc['near'] >= 0.9


def test_model_is_identical_across_runs(twelve, tmp_path):
    root, _ = twelve
    outs = []
    for k in range(2):
        out = str(tmp_path / f'm{k}')
        sfm.map_sparse(os.path.join(root, 'database.db'), out, os.path.join(root, 'images'))
        outs.append({n: open(os.path.join(out, f'{n}.bin'), 'rb').read() for n in ('cameras', 'images', 'points3D')})
    assert outs[0] == outs[1]


def test_disconnected_database_gives_the_larger_model(twelve, tmp_path):
    """Two projects in one database with no pair between them: the larger one is reconstructed, the other reported."""
    import sqlite3
    root, _ = twelve
    other = str(tmp_path / 'other')
    OM.project(other, 6, 640, 480, seed=1, per_view=10, workers=4)
    Ft.build_database(os.path.join(other, 'images'), os.path.join(other, 'database.db'))
    parts = []
    for r, off, prefix in ((root, 0, ''), (other, 12, 'other_')):
        con = sqlite3.connect(os.path.join(r, 'database.db'))
        parts.append(dict(
            off=off, prefix=prefix,
            cams=con.execute('SELECT camera_id, model, width, height, params, prior_focal_length FROM cameras').fetchall(),
            imgs=con.execute('SELECT image_id, name, camera_id FROM images').fetchall(),
            kps={i: np.frombuffer(b, np.float32).reshape(rr, c) for i, rr, c, b in con.execute('SELECT image_id, rows, cols, data FROM keypoints')},
            geos=[(Ft.pair_ids(p), np.frombuffer(d, np.uint32).reshape(rr, 2), np.frombuffer(F, np.float64).reshape(3, 3))
                  for p, rr, d, F in con.execute('SELECT pair_id, rows, data, F FROM two_view_geometries')]))
        con.close()
    cams, imgs, kps, geos = [], [], {}, {}
    for p in parts:
        o = p['off']
        cams += [(c + o, m, w, h, np.frombuffer(pa, np.float64), pf) for c, m, w, h, pa, pf in p['cams']]
        imgs += [(i + o, p['prefix'] + n, c + o) for i, n, c in p['imgs']]
        kps.update({i + o: k for i, k in p['kps'].items()})
        for (a, b), m, F in p['geos']:
            geos[a + o, b + o] = dict(matches=m, config=3, F=F, E=F, H=np.zeros((3, 3)), qvec=np.array([1.0, 0, 0, 0]), tvec=np.zeros(3))
    db = str(tmp_path / 'both.db')
    Ft.write_database(db, imgs, cams, kps, {}, {k: g['matches'] for k, g in geos.items()}, geos)
    s = sfm.map_sparse(db, str(tmp_path / 'model'))
    print(f'registered {s["registered"]}, not registered {s["unregistered"]}')
    assert s['registered'] == list(range(1, 13)) and s['unregistered'] == list(range(13, 19))


def test_workflow_without_colmap_or_true_poses(tmp_path, capsys):
    from nero_b200 import objprep as OPr
    from nero_b200.evaluate import read_points_ply
    root = str(tmp_path)
    pr = OM.project(root, 12, 640, 480, seed=3, workers=4)
    shutil.rmtree(os.path.join(root, 'sparse'))
    tool('match_features').main(['--root', root])
    tool('map_sparse').main(['--root', root])
    tool('dense_points').main(['--root', root])
    tool('prepare_custom_object').main(['--root', root, '--min-component', '0.1'])
    up = np.loadtxt(os.path.join(root, 'meta_info.txt'))[0]
    views, _ = OPr.read_colmap_model(os.path.join(root, 'sparse', '0'))
    ids = sorted(views)
    k = [pr['names'].index(views[i][0]) for i in ids]
    C = np.array([-views[i][1][:, :3].astype(np.float64).T @ views[i][1][:, 3] for i in ids])
    Ct = np.array([-pr['poses'][j][:, :3].T @ pr['poses'][j][:, 3] for j in k])
    s, R, t = _align(C, Ct)
    up_w = R @ up
    ang = np.degrees(np.arccos(np.clip(up_w @ pr['up'] / np.linalg.norm(up_w), -1, 1)))
    obj = read_points_ply(os.path.join(root, 'object_point_cloud.ply'))
    obj_w = s * obj @ R.T + t
    _, D, _, _ = OPr.scene_scale({i: (views[i][0], pr['poses'][j].astype(np.float32), views[i][2]) for i, j in zip(ids, k)})
    lo, hi = OM.object_bbox()
    err = max(np.abs(obj_w.min(0) - lo).max(), np.abs(obj_w.max(0) - hi).max())
    print(capsys.readouterr().out)
    print(f'up error {ang:.4f} deg, bounding-box error {err / (OPr.VOXEL_FRAC * D):.2f} voxels, {obj.shape[0]} object points')
    assert ang <= 1.0 and err <= 2 * OPr.VOXEL_FRAC * D
