"""SIMPLE_RADIAL structure from motion without a GPU: the radial header's symbols, the oracle's Jacobian against finite
differences of its residuals, the radial oracle at k = 0 against the pinhole one, the distorted render at k = 0 against
the pinhole render, and map_sparse.py's --camera-model refusals, which all come before any GPU work."""
import os
import re
import subprocess
import sys

import numpy as np

import nero_oracle_mvs as OM
import nero_oracle_sfm as OS
import nero_oracle_sfm_radial as OR
from nero_b200 import features as Ft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_radial_sfm_symbol():
    from nero_b200 import ops
    header = open(os.path.join(ROOT, 'include', 'nero_sfm_radial.h')).read()
    names = set(re.findall(r'\bint\s+(nero_sfm_radial_\w+)\s*\(', header))
    assert names == set(ops.SFM_RADIAL_PROTOS) and len(names) == 6
    assert not names & set(ops.SFM_PROTOS) and len(ops.SFM_PROTOS) == 9
    out = subprocess.run(['nm', '-D', '--defined-only', ops._LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r'\bT\s+(nero_sfm_radial_\w+)', out))
    assert names == exported, f'header {sorted(names)}, library {sorted(exported)}'


def _obs_pt(bp):
    return np.repeat(np.arange(bp['X'].shape[0]), np.diff(bp['pt_off']))


def test_oracle_jacobian_matches_central_differences():
    bp = OR.synthetic_problem(3, 30, seed=2, shared_camera=False, radial=-0.15)
    obs_pt = _obs_pt(bp)
    args = lambda pose, focal, radial, X: (pose, focal, radial, bp['pp'], bp['img_cam'], X, bp['obs_img'], obs_pt, bp['obs_xy'])
    res, Jc, Jp = OR.linearize(*args(bp['pose'], bp['focal'], bp['radial'], bp['X']))
    assert np.allclose(res.reshape(-1), OR.residuals(*args(bp['pose'], bp['focal'], bp['radial'], bp['X'])), rtol=0, atol=1e-10)
    n = res.shape[0]
    Jc_fd, Jp_fd = np.zeros_like(Jc), np.zeros_like(Jp)
    oi = bp['obs_img']
    for q in range(8):
        for i in range(bp['pose'].shape[0]):
            c = bp['img_cam'][i]
            h = 1e-6 * (bp['focal'][c] if q == 6 else 1.0)
            diff = []
            for sg in (1.0, -1.0):
                pose, focal, radial = bp['pose'].copy(), bp['focal'].copy(), bp['radial'].copy()
                if q < 3:
                    w = np.zeros(3)
                    w[q] = sg * h
                    pose[i, :9] = (OS.rodrigues(w) @ pose[i, :9].reshape(3, 3)).reshape(-1)
                elif q < 6:
                    pose[i, 6 + q] += sg * h
                elif q == 6:
                    focal[c] += sg * h
                else:
                    radial[c] += sg * h
                diff.append(OR.residuals(*args(pose, focal, radial, bp['X'])).reshape(n, 2))
            sel = oi == i
            Jc_fd[sel, :, q] = ((diff[0] - diff[1]) / (2 * h))[sel]
    for p in range(bp['X'].shape[0]):
        for q in range(3):
            diff = []
            for sg in (1.0, -1.0):
                X = bp['X'].copy()
                X[p, q] += sg * 1e-6
                diff.append(OR.residuals(*args(bp['pose'], bp['focal'], bp['radial'], X)).reshape(n, 2))
            sel = obs_pt == p
            Jp_fd[sel, :, q] = ((diff[0] - diff[1]) / 2e-6)[sel]
    for q in range(8):
        err = np.abs(Jc[:, :, q] - Jc_fd[:, :, q]).max() / np.abs(Jc[:, :, q]).max()
        assert err <= 1e-7, f'camera column {q}: {err:.2e}'
    assert np.abs(Jp - Jp_fd).max() / np.abs(Jp).max() <= 1e-7


def test_radial_oracle_at_k_zero_is_the_pinhole_oracle():
    """k = 0 and held: residuals, the (w, t, f) and point columns and the step equal the pinhole oracle's."""
    for shared in (False, True):
        bp = OS.synthetic_problem(4, 60, seed=3, shared_camera=shared)
        rp = dict(bp, radial=np.zeros(bp['focal'].shape[0]))
        nimg, ncam = bp['pose'].shape[0], bp['focal'].shape[0]
        fixed = np.zeros(6 * nimg + 2 * ncam, np.uint8)
        fixed[:6 * nimg] = bp['fixed'][:6 * nimg]
        fixed[6 * nimg:] = np.stack([bp['fixed'][6 * nimg:], np.ones(ncam, np.uint8)], 1).reshape(-1)
        rp['fixed'] = fixed
        pose, focal, X, o = OS.lm_step(bp, 1e-3)
        rpose, rfocal, rk, rX, ro = OR.lm_step(rp, 1e-3)
        rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
        assert rel(ro['res'], o['res']) <= 1e-14
        assert rel(ro['Jc'][:, :, :7], o['Jc']) <= 1e-13 and rel(ro['Jp'], o['Jp']) <= 1e-13
        keep = np.concatenate([np.arange(6 * nimg), 6 * nimg + 2 * np.arange(ncam)])
        assert rel(ro['dc'][keep], o['dc']) <= 1e-9 and np.all(ro['dc'][6 * nimg + 1::2] == 0)
        assert rel(rpose, pose) <= 1e-12 and rel(rfocal, focal) <= 1e-12 and rel(rX, X) <= 1e-12 and np.all(rk == 0)


def test_distorted_render_at_k_zero_is_the_pinhole_render():
    P = np.concatenate([np.eye(3), [[0.1], [-0.2], [-3.0]]], 1)
    w, h, f = 48, 36, 0.9 * 48
    K = np.array([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1]])
    ref = OM.render(P, K, w, h)['rgb']
    got = OR.render(P, f, w / 2, h / 2, 0.0, w, h)
    assert (got == ref).all(-1).mean() >= 0.99 and (got.astype(int) - ref).std() < 5


def _database(path, model):
    cams, cam_of = Ft.cameras_for([(64, 48)] * 3, camera_model=model)
    kp = {i: np.random.RandomState(i).rand(10, 6).astype(np.float32) * 40 for i in (1, 2, 3)}
    m = np.stack([np.arange(10), np.arange(10)], 1).astype(np.uint32)
    geos = {(1, 2): dict(matches=m, config=3, F=np.eye(3), E=np.eye(3), H=np.zeros((3, 3)), qvec=np.array([1.0, 0, 0, 0]),
                         tvec=np.zeros(3))}
    Ft.write_database(str(path), [(k + 1, f'img_{k}.png', cam_of[k]) for k in range(3)], cams, kp, {}, {(1, 2): m}, geos)


def _run(root, *extra):
    """Exit code and stderr of map_sparse.py in a process that sees no GPU."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'map_sparse.py'), '--root', str(root), *extra], env=env,
                       capture_output=True, text=True, timeout=300)
    return r.returncode, r.stderr


def test_camera_model_refusals_come_before_any_gpu_work(tmp_path):
    root = tmp_path / 'obj'
    (root / 'images').mkdir(parents=True)
    _database(root / 'database.db', 'SIMPLE_PINHOLE')
    rc, err = _run(root, '--camera-model', 'SIMPLE_RADIAL')
    assert rc == 2 and 'camera 1 is SIMPLE_PINHOLE' in err and 'match_features.py --camera-model SIMPLE_RADIAL' in err, err
    rc, err = _run(root, '--camera-model', 'OPENCV')
    assert rc == 2 and 'invalid choice' in err and 'OPENCV' in err, err
    os.remove(root / 'database.db')
    _database(root / 'database.db', 'SIMPLE_RADIAL')
    rc, err = _run(root)
    assert rc == 2 and 'SIMPLE_PINHOLE cameras only' in err and 'SIMPLE_RADIAL' in err and '--camera-model SIMPLE_RADIAL' in err, err


def test_check_database_takes_the_camera_model():
    from nero_b200 import sfm
    import pytest
    cams = {1: (Ft.SIMPLE_RADIAL, 64, 48, np.array([80.0, 32, 24, 0.0])), 2: (Ft.SIMPLE_RADIAL, 64, 48, np.array([80.0, 32, 24, np.nan]))}
    db = dict(cameras=cams, pairs={(1, 2): None})
    with pytest.raises(ValueError, match='camera 2: SIMPLE_RADIAL needs 4 finite'):
        sfm.check_database(db, 'SIMPLE_RADIAL')
    with pytest.raises(ValueError, match="camera model 'RADIAL'"):
        sfm.check_database(db, 'RADIAL')
    del cams[2]
    sfm.check_database(db, 'SIMPLE_RADIAL')
