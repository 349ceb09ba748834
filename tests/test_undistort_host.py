"""CPU: the SIMPLE_RADIAL convention of nero_b200/undistort.py against oracle/nero_oracle_undistort.py (inverse, camera rule,
warp identity at k = 0), COLMAP model records, the SIMPLE_RADIAL database cameras, the undistorter's refusals before any
GPU work, and the header's exports."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_mvs as OM
import nero_oracle_undistort as OU
from nero_b200 import features as Ft
from nero_b200 import objprep as OP
from nero_b200 import undistort as U

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize('k', [-0.2, -0.05, 0.0, 0.05, 0.2])
def test_inverse_undoes_the_distortion_across_the_valid_range(k):
    rng = np.random.RandomState(7)
    rmax = 0.95 / np.sqrt(-3 * k) if k < 0 else 1.5        # the monotone branch ends at r = 1 / sqrt(-3 k)
    r, th = rng.uniform(0, rmax, 20000), rng.uniform(0, 2 * np.pi, 20000)
    x, y = np.r_[0.0, r * np.cos(th)], np.r_[0.0, r * np.sin(th)]
    f, cx, cy = 700.0, 331.5, 247.25
    u, v = OU.distort(x, y, f, cx, cy, k)
    xx, yy, ok = U.undistort_host(u, v, f, cx, cy, k)
    assert ok.all()
    assert np.abs(xx - x).max() <= 1e-12 and np.abs(yy - y).max() <= 1e-12
    ox, oy, ook = OU.undistort(u, v, f, cx, cy, k)
    assert np.array_equal(xx, ox) and np.array_equal(yy, oy) and np.array_equal(ok, ook)


@pytest.mark.parametrize('k', [-0.2, -0.05])
def test_points_beyond_the_monotone_range_are_invalid(k):
    rs = 1 / np.sqrt(-3 * k)
    rd_max = rs * (1 + k * rs * rs)                          # the largest distorted radius of the monotone branch
    rd = np.linspace(1.0001 * rd_max, 4 * rd_max, 500)
    f = 500.0
    _, _, ok = U.undistort_host(f * rd, np.zeros_like(rd), f, 0.0, 0.0, k)
    assert not ok.any()
    assert not OU.undistort(f * rd, np.zeros_like(rd), f, 0.0, 0.0, k)[2].any()


def test_camera_rule():
    w, h, f = 640, 480, 576.0
    for cx, cy in ((320.0, 240.0), (317.3, 251.9), (0.1 * w, 0.9 * h)):
        assert U.camera(w, h, f, cx, cy, 0.0) == (w, h, cx, cy)
    for k in (-0.2, -0.08, -0.01, 0.01, 0.08, 0.2):
        got = U.camera(w, h, f, 312.0, 250.0, k)
        assert got == OU.camera(w, h, f, 312.0, 250.0, k)
        assert (got[0] > w and got[1] > h) if k < 0 else (got[0] < w and got[1] < h)
    for k in (-1.0, -0.6, 10.0, np.nan):                     # corners outside the invertible range, or a < 0.5 ratio
        with pytest.raises(ValueError, match='camera 7'):
            U.camera(w, h, f, 320.0, 240.0, k, name='camera 7')


def test_warp_oracle_is_the_identity_at_k_zero():
    rng = np.random.RandomState(3)
    img = rng.randint(0, 256, (37, 53, 3)).astype(np.uint8)
    for f, cx, cy in ((60.0, 26.5, 18.5), (41.3, 20.1, 19.7)):
        W, H, cx2, cy2 = U.camera(53, 37, f, cx, cy, 0.0)
        assert np.array_equal(OU.warp(img, f, cx, cy, 0.0, W, H, cx2, cy2), img)


def _model(tmp_path, cams, fmt=None):
    pts = {1: ((0.1, 0.2, 3.0), [1, 2, 3], 0.5, [1, 2], [0, 1]), 5: ((-0.4, 0.0, 2.5), [9, 8, 7], 0.25, [2], [0])}
    images = {1: ((1.0, 0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 1, 'a.png', np.asarray([[10.5, 20.25], [30.0, 40.0]]), [1, 1]),
              2: ((0.99, 0.1, 0.0, 0.0), (0.1, 0.2, 0.3), list(cams)[-1], 'b.png', np.asarray([[1.0, 2.0], [3.0, 4.0]]), [5, 1])}
    path = str(tmp_path / 'sparse' / '0')
    if fmt is None:                                          # the package's writer, which knows every model id
        OP.write_colmap_model(path, cams, images, pts)
    else:
        OM.OOp.write_colmap_model(path, cams, images, pts, fmt)
    return path, images, pts


@pytest.mark.parametrize('fmt', ['bin', 'txt'])
@pytest.mark.parametrize('model', ['SIMPLE_RADIAL', 'SIMPLE_PINHOLE'])
def test_model_records_round_trip(tmp_path, fmt, model):
    par = [576.0, 320.0, 240.0, -0.08] if model == 'SIMPLE_RADIAL' else [576.0, 320.0, 240.0]
    cams = {1: (model, 640, 480, par), 3: ('PINHOLE', 640, 480, [500.0, 510.0, 320.0, 240.0])}
    path, images, pts = _model(tmp_path, cams, fmt)
    c, im, pt = OP.read_colmap_records(path)
    assert c == cams
    assert list(im) == list(images) and list(pt) == list(pts)
    for iid in images:
        q, t, cid, name, xys, p3d = images[iid]
        assert np.allclose(im[iid][0], q) and np.allclose(im[iid][1], t) and im[iid][2:4] == (cid, name)
        assert np.array_equal(im[iid][4], xys) and np.array_equal(im[iid][5], p3d)
    for pid in pts:
        assert np.allclose(pt[pid][0], pts[pid][0]) and list(pt[pid][1]) == pts[pid][1] and pt[pid][2] == pts[pid][2]
        assert list(pt[pid][3]) == pts[pid][3] and list(pt[pid][4]) == pts[pid][4]
    if fmt == 'bin':                                         # written back, the files are the same bytes
        out = str(tmp_path / 'again')
        OP.write_colmap_model(out, c, im, pt)
        for n in ('cameras', 'images', 'points3D'):
            assert open(os.path.join(out, f'{n}.bin'), 'rb').read() == open(os.path.join(path, f'{n}.bin'), 'rb').read()


def test_database_cameras_of_the_simple_radial_model(tmp_path):
    sizes = [(640, 480), (640, 480), (800, 600)]
    for same in (False, True):
        base, _ = Ft.cameras_for(sizes, same)
        cams, cam_of = Ft.cameras_for(sizes, same, 'SIMPLE_RADIAL')
        assert cam_of == Ft.cameras_for(sizes, same)[1]
        for (c0, m0, w0, h0, p0, pr0), (c, m, w, h, p, pr) in zip(base, cams):
            assert (c, w, h, pr) == (c0, w0, h0, pr0) and m0 == 0 and m == 2
            assert np.array_equal(p, np.r_[p0, 0.0])
    with pytest.raises(ValueError, match='OPENCV'):
        Ft.cameras_for(sizes, False, 'OPENCV')
    cams, cam_of = Ft.cameras_for(sizes[:2], False, 'SIMPLE_RADIAL')
    db = str(tmp_path / 'database.db')
    kp = {1: np.zeros((0, 6), np.float32), 2: np.zeros((0, 6), np.float32)}
    Ft.write_database(db, [(1, 'a.png', 1), (2, 'b.png', 2)], cams, kp, {1: np.zeros((0, 128), np.uint8), 2: np.zeros((0, 128), np.uint8)},
                      {}, {})
    from nero_b200 import sfm
    got = sfm.read_database(db)['cameras']
    assert sorted(got) == [1, 2] and all(m == 2 and list(p) == [800.0, 320.0, 240.0, 0.0] for m, _, _, p in got.values())
    assert np.array_equal(Ft.camera_K(cams[0]), Ft.camera_K(Ft.cameras_for(sizes[:2])[0][0]))


def _refusal(*args):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'undistort_images.py'), *args], env=env, capture_output=True,
                       text=True, timeout=300)
    return r.returncode, r.stderr


def test_undistorter_refusals_come_before_any_gpu_work(tmp_path):
    root = tmp_path / 'obj'
    (root / 'images').mkdir(parents=True)
    out = str(tmp_path / 'out')
    rc, err = _refusal('--root', str(root), '--output', out)
    assert rc == 2 and 'no COLMAP model' in err
    path, _, _ = _model(root, {1: ('OPENCV_FISHEYE', 640, 480, [500.0, 500.0, 320.0, 240.0, 0.1, 0.0, 0.0, 0.0])})
    rc, err = _refusal('--root', str(root), '--output', out)
    assert rc != 0 and 'OPENCV_FISHEYE' in err and 'SIMPLE_RADIAL' in err
    _model(root, {1: ('SIMPLE_RADIAL', 640, 480, [576.0, 320.0, 240.0, -0.9])})
    rc, err = _refusal('--root', str(root), '--output', out)
    assert rc != 0 and 'camera 1' in err and 'invertible' in err
    os.makedirs(out)
    rc, err = _refusal('--root', str(root), '--output', out)
    assert rc == 2 and 'already exists' in err and '--force' in err
    assert os.listdir(out) == []


def test_library_exports_every_symbol_of_the_undistort_header():
    import __graft_entry__ as g
    lib = ctypes.CDLL(g.build())
    txt = open(os.path.join(ROOT, 'include', 'nero_undistort.h')).read()
    syms = sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))
    assert syms == ['nero_undistort_image', 'nero_undistort_points']
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/nero_undistort.h but not exported'
    from nero_b200 import ops
    for s in syms:
        assert len(getattr(ops.lib, s).argtypes) == len(ops.UNDISTORT_PROTOS[s])
    # bad arguments are refused before any launch
    buf = ctypes.c_void_p(16)
    assert ops.lib.nero_undistort_points(buf, 4, 0.0, 1.0, 1.0, 0.0, buf, buf, None) == 1
    assert ops.lib.nero_undistort_points(buf, -1, 1.0, 1.0, 1.0, 0.0, buf, buf, None) == 1
    assert ops.lib.nero_undistort_points(None, 0, 1.0, 1.0, 1.0, 0.0, None, None, None) == 0
    assert ops.lib.nero_undistort_image(buf, 4, 4, 1.0, 2.0, 2.0, float('nan'), buf, 4, 4, 2.0, 2.0, None) == 1
    assert ops.lib.nero_undistort_image(buf, 0, 4, 1.0, 2.0, 2.0, 0.0, buf, 4, 4, 2.0, 2.0, None) == 1
    assert ops.lib.nero_undistort_image(None, 4, 4, 1.0, 2.0, 2.0, 0.0, buf, 4, 4, 2.0, 2.0, None) == 1


def test_feature_refinement_takes_an_octave_without_candidates():
    """An octave with no DoG extrema has an empty keypoint buffer (a NULL pointer); the refinement has nothing to do and
    returns 0 rather than refusing it, so feature extraction works on images with few extrema."""
    from nero_b200 import ops
    buf = ctypes.c_void_p(16)
    assert ops.lib.nero_features_refine(buf, 64, 64, 6, None, 0, 0, 1.6, 0.02, 10.0, None, None) == 0
    assert ops.lib.nero_features_refine(buf, 64, 64, 6, buf, 3, 0, 1.6, 0.02, 10.0, None, None) == 1
