"""GPU: the kernels of k_undistort.cu against oracle/nero_oracle_undistort.py bit for bit, and tools/undistort_images.py on a
SIMPLE_RADIAL project whose images are rendered exactly through the distortion (no resampling in the truth)."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_undistort as OU
from nero_b200 import features as Ft
from nero_b200 import mvs
from nero_b200 import objprep as OP
from nero_b200 import undistort as U

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_warp_matches_the_oracle_bit_for_bit():
    rng = np.random.RandomState(11)
    for it in range(8):
        w, h = int(rng.randint(40, 160)), int(rng.randint(30, 120))
        f = float(rng.uniform(0.7, 1.3) * w)
        cx, cy = float(w / 2 + rng.uniform(-5, 5)), float(h / 2 + rng.uniform(-5, 5))
        k = float(rng.uniform(-0.2, 0.2))
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        W, H, cx2, cy2 = U.camera(w, h, f, cx, cy, k)
        got = U.image(img, f, cx, cy, k, W, H, cx2, cy2).cpu().numpy()
        assert got.shape == (H, W, 3)
        assert np.array_equal(got, OU.warp(img, f, cx, cy, k, W, H, cx2, cy2)), (it, k)
        j, i = np.mgrid[0:H, 0:W]                            # every output pixel centre lands inside the input
        u, v = OU.distort(((i + 0.5) - cx2) / f, ((j + 0.5) - cy2) / f, f, cx, cy, k)
        assert (u >= 0).all() and (u <= w).all() and (v >= 0).all() and (v <= h).all(), (it, k)
        W0, H0, cx0, cy0 = U.camera(w, h, f, cx, cy, 0.0)
        assert np.array_equal(U.image(img, f, cx, cy, 0.0, W0, H0, cx0, cy0).cpu().numpy(), img)


def test_keypoint_inversion_matches_the_oracle():
    rng = np.random.RandomState(5)
    for k in (-0.2, -0.05, 0.0, 0.05, 0.2):
        f, cx, cy = 800.0, 401.5, 299.25
        xy = np.stack([rng.uniform(-900, 1700, 50000), rng.uniform(-700, 1300, 50000)], 1)
        xy[:3] = [[cx, cy], [0.0, 0.0], [cx + 1e-9, cy]]
        xn, ok = U.points(xy, f, cx, cy, k)
        xn, ok = xn.cpu().numpy(), ok.cpu().numpy()
        ox, oy, ook = OU.undistort(xy[:, 0], xy[:, 1], f, cx, cy, k)
        assert np.array_equal(ok, ook), k
        assert np.array_equal(xn[ok, 0], ox[ok]) and np.array_equal(xn[ok, 1], oy[ok]), k
        if k >= 0:
            assert ok.all()
        else:
            assert 0 < ok.sum() < ok.shape[0]
    assert U.points(np.zeros((0, 2)), 1.0, 0.0, 0.0, 0.1)[0].shape == (0, 2)


def _project(root, k, w=320, h=240, n=3, names=None):
    """A SIMPLE_RADIAL model of n views of pattern(): images rendered through the distortion, keypoints the distorted
    projections of random points in front of every camera, one shared camera."""
    f, cx, cy = 0.9 * w, w / 2 + 1.25, h / 2 - 0.75
    rng = np.random.RandomState(2)
    names = names or [f'v{i}.png' for i in range(n)]
    os.makedirs(os.path.join(root, 'images'), exist_ok=True)
    X = np.stack([rng.uniform(-0.3, 0.3, 40), rng.uniform(-0.2, 0.2, 40), rng.uniform(2.5, 3.5, 40)], 1)
    images = {}
    for i, name in enumerate(names):
        import cv2
        cv2.imwrite(os.path.join(root, 'images', name), np.ascontiguousarray(OU.render_pattern(w, h, f, cx, cy, k)[..., ::-1]),
                    [cv2.IMWRITE_JPEG_QUALITY, 100])
        t = np.asarray([0.01 * i, -0.02 * i, 0.0])
        Y = X + t
        u, v = OU.distort(Y[:, 0] / Y[:, 2], Y[:, 1] / Y[:, 2], f, cx, cy, k)
        images[i + 1] = ((1.0, 0.0, 0.0, 0.0), tuple(t), 1, name, np.stack([u, v], 1), np.arange(1, 41))
    points = {p + 1: (tuple(X[p]), [10, 20, 30], 0.1, list(range(1, len(names) + 1)), [p] * len(names)) for p in range(40)}
    OP.write_colmap_model(os.path.join(root, 'sparse', '0'), {1: ('SIMPLE_RADIAL', w, h, [f, cx, cy, k])}, images, points)
    return X, (f, cx, cy)


def test_undistorter_on_the_true_model(tmp_path):
    k = -0.08
    X, (f, cx, cy) = _project(str(tmp_path / 'obj'), k, names=['a.png', 'b.jpg', 'c.png'])
    outs = []
    for run in range(2):
        out = str(tmp_path / f'out{run}')
        tool('undistort_images').main(['--root', str(tmp_path / 'obj'), '--output', out])
        outs.append(out)
    cams, images, pts = OP.read_colmap_records(os.path.join(outs[0], 'sparse', '0'))
    model, W, H, (f2, cx2, cy2) = cams[1]
    assert model == 'SIMPLE_PINHOLE' and f2 == f and (W, H, cx2, cy2) == U.camera(320, 240, f, cx, cy, k)
    assert W > 320 and H > 240
    _, _, pts0 = OP.read_colmap_records(os.path.join(str(tmp_path / 'obj'), 'sparse', '0'))
    assert list(pts) == list(pts0)
    j, i = np.mgrid[0:H, 0:W]
    truth = np.clip(np.floor(OU.pattern(((i + 0.5) - cx2) / f, ((j + 0.5) - cy2) / f) + 0.5), 0, 255)
    for iid, (q, t, cid, name, xys, p3d) in images.items():
        Y = X + np.asarray(t)
        proj = np.stack([f * Y[:, 0] / Y[:, 2] + cx2, f * Y[:, 1] / Y[:, 2] + cy2], 1)
        err = np.abs(xys - proj[p3d - 1]).max()
        assert err <= 0.05, (name, err)
        got = mvs.read_rgb(os.path.join(outs[0], 'images', name))
        src = mvs.read_rgb(os.path.join(str(tmp_path / 'obj'), 'images', name))
        mad = np.abs(got.astype(np.float64) - truth).mean()
        print(f'{name}: mean |undistorted - truth| = {mad:.3f}, POINTS2D error {err:.2e} px')
        assert mad <= 1.0, (name, mad)
        if name.endswith('.png'):                              # PNG is lossless: the oracle's bytes
            assert np.array_equal(got, OU.warp(src, f, cx, cy, k, W, H, cx2, cy2))
        assert np.array_equal(got, mvs.read_rgb(os.path.join(outs[1], 'images', name)))
    for n in ('cameras', 'images', 'points3D'):
        a, b = (open(os.path.join(o, 'sparse', '0', f'{n}.bin'), 'rb').read() for o in outs)
        assert a == b, n
    for name in ('a.png', 'c.png'):
        a, b = (open(os.path.join(o, 'images', name), 'rb').read() for o in outs)
        assert a == b, name


def test_pinhole_cameras_pass_through(tmp_path):
    root = tmp_path / 'obj'
    X, (f, cx, cy) = _project(str(root), 0.0, n=2)
    cams, images, pts = OP.read_colmap_records(str(root / 'sparse' / '0'))
    cams[1] = ('SIMPLE_PINHOLE', 320, 240, [f, cx, cy])
    OP.write_colmap_model(str(root / 'sparse' / '0'), cams, images, pts)
    out = str(tmp_path / 'out')
    info = tool('undistort_images').main(['--root', str(root), '--output', out])
    assert info['copied'] == 2 and info['warped'] == 0
    for name in ('v0.png', 'v1.png'):
        assert open(os.path.join(out, 'images', name), 'rb').read() == open(str(root / 'images' / name), 'rb').read()
    for n in ('cameras', 'images', 'points3D'):
        assert open(os.path.join(out, 'sparse', '0', f'{n}.bin'), 'rb').read() == \
            open(str(root / 'sparse' / '0' / f'{n}.bin'), 'rb').read()


def test_radial_k_zero_project_returns_the_input_arrays(tmp_path):
    root = tmp_path / 'obj'
    _project(str(root), 0.0, n=2)
    out = str(tmp_path / 'out')
    tool('undistort_images').main(['--root', str(root), '--output', out])
    cams, images, _ = OP.read_colmap_records(os.path.join(out, 'sparse', '0'))
    cams0, images0, _ = OP.read_colmap_records(str(root / 'sparse' / '0'))
    assert cams[1] == ('SIMPLE_PINHOLE', 320, 240, cams0[1][3][:3])
    for name in ('v0.png', 'v1.png'):
        assert np.array_equal(mvs.read_rgb(os.path.join(out, 'images', name)), mvs.read_rgb(str(root / 'images' / name)))
    for iid in images:
        assert np.abs(images[iid][4] - images0[iid][4]).max() <= 1e-9



def test_invalid_keypoints_refuse_the_project_before_any_output(tmp_path):
    root = tmp_path / 'obj'
    _project(str(root), -0.08, n=2)
    cams, images, pts = OP.read_colmap_records(str(root / 'sparse' / '0'))
    q, t, cid, name, xys, p3d = images[2]
    xys = xys.copy()
    xys[3] = [-5000.0, -5000.0]                                  # far beyond the invertible range of k = -0.08
    images[2] = (q, t, cid, name, xys, p3d)
    OP.write_colmap_model(str(root / 'sparse' / '0'), cams, images, pts)
    out = str(tmp_path / 'out')
    with pytest.raises(SystemExit, match='image 2'):
        tool('undistort_images').main(['--root', str(root), '--output', out])
    assert not os.path.exists(out) or not any(files for _, _, files in os.walk(out))


def test_database_with_simple_radial_cameras(tmp_path):
    """match_features on smooth images whose coarse octaves have no extrema, with SIMPLE_RADIAL cameras."""
    root = tmp_path / 'obj'
    _project(str(root), -0.05, n=2)
    db = str(tmp_path / 'database.db')
    info = Ft.build_database(str(root / 'images'), db, max_features=500, camera_model='SIMPLE_RADIAL')
    assert info['names'] == ['v0.png', 'v1.png']
    from nero_b200 import sfm
    cams = sfm.read_database(db)['cameras']
    assert sorted(cams) == [1, 2]
    for m, w, h, p in cams.values():
        assert m == 2 and (w, h) == (320, 240) and list(p) == [400.0, 160.0, 120.0, 0.0]
