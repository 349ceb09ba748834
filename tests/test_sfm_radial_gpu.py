"""SIMPLE_RADIAL structure from motion on the GPU: the radial bundle-adjustment kernels against the fp64 oracle
(oracle/nero_oracle_sfm_radial.py), the adjustment against scipy's least-squares solver with the k column, and the
mapper on projects rendered through the distortion: accuracy against the true cameras and k, run-to-run identity of the
model, and the workflow from distorted images to the prepared object with no COLMAP and no true poses."""
import os

import numpy as np
import pytest
import torch

import nero_oracle_mvs as OM
import nero_oracle_sfm as OS
import nero_oracle_sfm_radial as OR
from nero_b200 import features as Ft
from nero_b200 import sfm
from test_sfm_gpu import _accuracy, _align, _rel, tool

pytestmark = pytest.mark.gpu
K_TRUE = -0.05          # the lens of the mapper projects


def _problem(bp):
    return sfm.Problem(bp['pose'], bp['focal'], bp['pp'], bp['img_cam'], bp['X'], bp['pt_off'], bp['obs_img'], bp['obs_xy'], bp['fixed'],
                       radial=bp['radial'])


@pytest.mark.parametrize('shared', [False, True])
def test_radial_bundle_adjustment_kernels_match_the_oracle(shared):
    bp = OR.synthetic_problem(5, 150, seed=4, shared_camera=shared, radial=-0.15)
    pr = _problem(bp)
    if shared:     # the camera segments span many chunks: the two-stage sums are exercised
        assert int((pr.seg_chunk[1:] - pr.seg_chunk[:-1]).max()) > 2 and int((pr.rseg_chunk[1:] - pr.rseg_chunk[:-1]).max()) > 1
    pr.linearize()
    lam = 1e-3
    pr.eliminate(lam)
    S, b = pr.reduce(lam)
    dc = torch.linalg.solve(S, b)
    pose, focal, X, radial = pr.backsub(dc)
    opose, ofocal, ok, oX, o = OR.lm_step(bp, lam)
    got = dict(res=pr.res, Jc=pr.Jc, Jp=pr.Jp, Vinv=pr.Vinv, gp=pr.gp, Y=pr.Y, S=S, b=b)
    for k, v in got.items():
        err = _rel(v.cpu().numpy().reshape(o[k].shape), o[k])
        print(f'{k}: {err:.2e}')
        assert err <= 1e-12, f'{k} differs from the oracle by {err:.2e} (relative)'
    assert _rel(dc.cpu().numpy(), o['dc']) <= 1e-9
    assert _rel(X.cpu().numpy() - bp['X'], o['dX']) <= 1e-9
    assert _rel(pose.cpu().numpy(), opose) <= 1e-9 and _rel(focal.cpu().numpy(), ofocal) <= 1e-9 and _rel(radial.cpu().numpy(), ok) <= 1e-9
    _, _, X2, _ = pr.backsub(torch.from_numpy(o['dc']).cuda())
    assert _rel(X2.cpu().numpy() - bp['X'], o['dX']) <= 1e-12
    c = pr.cost()
    oc = OR.cost(bp['pose'], bp['focal'], bp['radial'], bp['pp'], bp['img_cam'], bp['X'], bp['obs_img'],
                 np.repeat(np.arange(bp['X'].shape[0]), np.diff(bp['pt_off'])), bp['obs_xy'])
    assert abs(c - oc) <= 1e-12 * oc
    # the filter's distorted reprojection errors against the oracle's residuals
    err, _ = sfm.reprojection(bp['pt_off'], bp['obs_img'], bp['obs_xy'], bp['pose'], bp['img_cam'], bp['focal'], bp['pp'], bp['X'],
                              bp['radial'])
    assert np.abs(err[:, 1] - np.hypot(*o['res'].T)).max() <= 1e-9


def _scipy_problem(bp, free):
    """scipy's view: free parameters (w with R = exp(w) R_start, t, f, k, X offsets) -> residuals and the analytic Jacobian
    (the oracle's columns, rotation columns through the left Jacobian of SO(3))."""
    nimg, ncam, P = bp['pose'].shape[0], bp['focal'].shape[0], bp['X'].shape[0]
    obs_pt = np.repeat(np.arange(P), np.diff(bp['pt_off']))
    oi, n = bp['obs_img'], bp['obs_img'].shape[0]
    nc = 6 * nimg + 2 * ncam
    nfull = nc + 3 * P

    def unpack(x):
        full = np.zeros(nfull)
        full[free] = x
        pose = bp['pose'].copy()
        for i in range(nimg):
            pose[i, :9] = (OS.rodrigues(full[6 * i:6 * i + 3]) @ bp['pose'][i, :9].reshape(3, 3)).reshape(-1)
            pose[i, 9:] = bp['pose'][i, 9:] + full[6 * i + 3:6 * i + 6]
        return full, pose, bp['focal'] + full[6 * nimg:nc:2], bp['radial'] + full[6 * nimg + 1:nc:2], bp['X'] + full[nc:].reshape(-1, 3)

    def fun(x):
        _, pose, focal, radial, X = unpack(x)
        return OR.residuals(pose, focal, radial, bp['pp'], bp['img_cam'], X, oi, obs_pt, bp['obs_xy'])

    def left_jacobian(w):
        th = np.linalg.norm(w)
        K = OS._hat(w)
        if th < 1e-8:
            return np.eye(3) + K / 2
        return np.eye(3) + (1 - np.cos(th)) / th ** 2 * K + (th - np.sin(th)) / th ** 3 * K @ K

    def jac(x):
        full, pose, focal, radial, X = unpack(x)
        _, Jc, Jp = OR.linearize(pose, focal, radial, bp['pp'], bp['img_cam'], X, oi, obs_pt, bp['obs_xy'])
        Jl = np.stack([left_jacobian(full[6 * i:6 * i + 3]) for i in range(nimg)])[oi]
        J = np.zeros((n, 2, nfull))
        rows = np.arange(n)
        c = bp['img_cam'][oi]
        Jw = np.einsum('nij,njk->nik', Jc[:, :, :3], Jl)
        for k in range(3):
            J[rows, :, 6 * oi + k] = Jw[:, :, k]
            J[rows, :, 6 * oi + 3 + k] = Jc[:, :, 3 + k]
            J[rows, :, nc + 3 * obs_pt + k] = Jp[:, :, k]
        J[rows, :, 6 * nimg + 2 * c] = Jc[:, :, 6]
        J[rows, :, 6 * nimg + 2 * c + 1] = Jc[:, :, 7]
        return J.reshape(2 * n, nfull)[:, free]
    return fun, jac, unpack


def test_radial_bundle_adjustment_converges_to_scipys_solution():
    from scipy.optimize import least_squares
    bp = OR.synthetic_problem(6, 300, noise=0.5, seed=8, radial=-0.15)
    pr = _problem(bp)
    info = pr.solve(200, tol=1e-15)
    pose, focal, X = pr.result()
    radial = pr.radial.cpu().numpy()
    free = np.nonzero(np.concatenate([bp['fixed'] == 0, np.ones(3 * bp['X'].shape[0], bool)]))[0]
    fun, jac, unpack = _scipy_problem(bp, free)
    sol = least_squares(fun, np.zeros(free.shape[0]), jac=jac, method='lm', ftol=1e-15, xtol=1e-15, gtol=1e-15)
    _, spose, sfocal, sradial, sX = unpack(sol.x)
    scost = float((sol.fun ** 2).sum())
    print(f'LM: {info["iterations"]} iterations, cost {info["cost0"]:.6f} -> {info["cost"]:.9f}; scipy ({sol.nfev} evaluations, status '
          f'{sol.status}) {scost:.9f}; pose {_rel(pose, spose):.2e}, focal {_rel(focal, sfocal):.2e}, k {_rel(radial, sradial):.2e}, '
          f'points {_rel(X, sX):.2e}; k {radial} (true {bp["truth"]["radial"]})')
    assert abs(info['cost'] - scost) <= 1e-6 * scost
    assert _rel(pose, spose) <= 1e-6 and _rel(focal, sfocal) <= 1e-6 and _rel(radial, sradial) <= 1e-6 and _rel(X, sX) <= 1e-6


# ------------------------------------------------------------------------------------------------ the mapper
@pytest.fixture(scope='module')
def radial12(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('sfm_radial12'))
    pr = OR.project(root, 12, 640, 480, K_TRUE, workers=4)
    tool('match_features').main(['--root', root, '--camera-model', 'SIMPLE_RADIAL'])
    return root, pr


def _map(root, db, out, model):
    return tool('map_sparse').main(['--root', root, '--database', db, '--output', out, '--camera-model', model])


@pytest.mark.parametrize('same', [False, True])
def test_radial_mapper_accuracy_on_twelve_views(radial12, tmp_path, same):
    root, pr = radial12
    db = os.path.join(root, 'database.db')
    if same:
        db = str(tmp_path / 'same.db')
        Ft.build_database(os.path.join(root, 'images'), db, same_camera=True, camera_model='SIMPLE_RADIAL')
    s = _map(root, db, str(tmp_path / 'model'), 'SIMPLE_RADIAL')
    acc = _accuracy(str(tmp_path / 'model'), pr)
    f_true = pr['K'][0, 0]
    ferr = max(abs(f - f_true) / f_true for f in s['focals'].values())
    kerr = max(abs(k - K_TRUE) for k in s['radial'].values())
    # the pinhole mapper on the same images, for the record: what estimating k buys
    pdb = str(tmp_path / 'pinhole.db')
    Ft.build_database(os.path.join(root, 'images'), pdb, same_camera=same)
    try:
        ps = _map(root, pdb, str(tmp_path / 'pinhole'), 'SIMPLE_PINHOLE')
        pacc = _accuracy(str(tmp_path / 'pinhole'), pr)
        pf = max(abs(f - f_true) / f_true for f in ps['focals'].values())
        pinhole = f'{pacc}, focal errors up to {100 * pf:.3f} %, mean error {ps["mean_error"]:.3f} px, {ps["points"]} points'
    except RuntimeError as e:
        pinhole = f'failed: {e}'
    print(f'same_camera={same}: SIMPLE_RADIAL {acc}, focal errors up to {100 * ferr:.3f} %, |k - k_true| up to {kerr:.5f}, mean error '
          f'{s["mean_error"]:.3f} px, {s["points"]} points, warnings {s["warnings"]}\n  SIMPLE_PINHOLE on the same images: {pinhole}')
    # measured on one H100 (DESIGN.md section 4m'): centre 0.58 % / 0.14 % of D, |k - k_true| 0.0216 / 0.0107.  Twelve
    # 640 x 480 views pin k loosely (48 views at 1600 x 1200 give 0.0022), so the k and centre bars carry that margin.
    assert acc['registered'] == 12 and not s['unregistered']
    assert acc['rotation'] <= 0.2 and acc['centre'] <= 0.0075
    assert ferr <= (0.01 if same else 0.02) and kerr <= (0.015 if same else 0.03)
    assert s['mean_error'] <= 1.0 and acc['near'] >= 0.9
    if not pinhole.startswith('failed'):
        assert acc['near'] > pacc['near']


def test_radial_model_is_identical_across_runs(radial12, tmp_path):
    root, _ = radial12
    outs = []
    for k in range(2):
        out = str(tmp_path / f'm{k}')
        sfm.map_sparse(os.path.join(root, 'database.db'), out, os.path.join(root, 'images'), camera_model='SIMPLE_RADIAL')
        outs.append({n: open(os.path.join(out, f'{n}.bin'), 'rb').read() for n in ('cameras', 'images', 'points3D')})
    assert outs[0] == outs[1]


def test_radial_workflow_without_colmap_or_true_poses(tmp_path, capsys):
    from nero_b200 import objprep as OPr
    from nero_b200.evaluate import read_points_ply
    root, und = str(tmp_path / 'raw'), str(tmp_path / 'und')
    pr = OR.project(root, 12, 640, 480, K_TRUE, seed=3, workers=4)
    tool('match_features').main(['--root', root, '--camera-model', 'SIMPLE_RADIAL'])
    tool('map_sparse').main(['--root', root, '--camera-model', 'SIMPLE_RADIAL'])
    tool('undistort_images').main(['--root', root, '--output', und])
    tool('dense_points').main(['--root', und])
    tool('prepare_custom_object').main(['--root', und, '--min-component', '0.1'])
    up = np.loadtxt(os.path.join(und, 'meta_info.txt'))[0]
    views, _ = OPr.read_colmap_model(os.path.join(und, 'sparse', '0'))
    ids = sorted(views)
    k = [pr['names'].index(views[i][0]) for i in ids]
    C = np.array([-views[i][1][:, :3].astype(np.float64).T @ views[i][1][:, 3] for i in ids])
    Ct = np.array([-pr['poses'][j][:, :3].T @ pr['poses'][j][:, 3] for j in k])
    s, R, t = _align(C, Ct)
    up_w = R @ up
    ang = np.degrees(np.arccos(np.clip(up_w @ pr['up'] / np.linalg.norm(up_w), -1, 1)))
    obj = read_points_ply(os.path.join(und, 'object_point_cloud.ply'))
    obj_w = s * obj @ R.T + t
    _, D, _, _ = OPr.scene_scale({i: (views[i][0], pr['poses'][j].astype(np.float32), views[i][2]) for i, j in zip(ids, k)})
    lo, hi = OM.object_bbox()
    err = max(np.abs(obj_w.min(0) - lo).max(), np.abs(obj_w.max(0) - hi).max())
    print(capsys.readouterr().out)
    print(f'up error {ang:.4f} deg, bounding-box error {err / (OPr.VOXEL_FRAC * D):.2f} voxels, {obj.shape[0]} object points')
    assert ang <= 1.0 and err <= 2 * OPr.VOXEL_FRAC * D
