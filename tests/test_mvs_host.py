"""Dense multi-view stereo, host side: the track reader, source selection and depth ranges, the grey image's scaling of K,
the oracle's PatchMatch on a textured plane, and the tool's argument checks."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_mvs as OM
import nero_oracle_objprep as OOp
from nero_b200 import mvs
from nero_b200 import objprep as OP

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.parametrize('fmt', ['bin', 'txt'])
def test_track_reader_round_trip(tmp_path, fmt):
    sc = OOp.scene(n_table=500, n_obj=300, n_cams=6, seed=2)
    cams, images, points = OOp.scene_model(sc)
    points = {pid: (p[0], p[1], p[2], [100 - 2 * (k % 6), 100 - 2 * ((k + 1) % 6), 98][:2 + k % 2], [k, 0, 3][:2 + k % 2])
              for k, (pid, p) in enumerate(points.items())}
    OOp.write_colmap_model(str(tmp_path), cams, images, points, fmt)
    views, pts, tracks = OP.read_colmap_model(str(tmp_path), tracks=True)
    assert len(tracks) == pts.shape[0] == len(points)
    for t, p in zip(tracks, points.values()):
        assert t.dtype == np.int64 and t.tolist() == list(p[3])
    plain = OP.read_colmap_model(str(tmp_path))
    assert len(plain) == 2 and np.array_equal(plain[1], pts) and plain[0].keys() == views.keys()


def _cams(centres, target=(0.0, 0.0, 0.0)):
    return np.stack([OOp.look_at(c, target, np.asarray([0.0, 0.0, 1.0])) for c in centres])


def test_source_selection_and_depth_range():
    # 5 cameras on a circle of radius 4 at 0, 10, 20, 90 degrees and one 0.1 degree from the first
    ang = np.radians([0.0, 10.0, 20.0, 90.0, 0.1])
    centres = np.stack([4 * np.cos(ang), 4 * np.sin(ang), np.full(5, 0.5)], 1)
    poses = _cams(centres)
    ids = [11, 12, 13, 14, 15]
    rng = np.random.RandomState(0)
    pts = rng.rand(40, 3) * 0.2 - 0.1
    tracks = [np.asarray(ids, np.int64)] * 30 + [np.asarray([11, 13], np.int64)] * 10
    score, plan = mvs.select_sources(pts, tracks, poses, ids)
    # view 0: 10 deg (view 1) and 20 deg (view 2) pass; 90 deg exceeds 60; 0.1 deg is below 2
    assert score[0].tolist() == [0, 30, 40, 0, 0]
    assert plan[0]['sources'] == [2, 1] and plan[0]['skip'] is None
    assert plan[4]['sources'] == [1, 2]                         # view 4 shares 30 points with both: ties in name order
    assert plan[3]['skip'] is not None and plan[3]['sources'] == []
    z = pts @ poses[0][2, :3] + poses[0][2, 3]
    p1, p99 = np.percentile(z, [1, 99])
    assert plan[0]['range'] == (0.75 * p1, 1.25 * p99)
    assert plan[0]['track'] == 40
    _, few = mvs.select_sources(pts[:9], tracks[:9], poses, ids)
    assert 'sparse points' in few[0]['skip']
    _, cap = mvs.select_sources(pts, tracks, poses, ids, sources=1)
    assert cap[0]['sources'] == [2] and cap[0]['skip'] is not None


def test_grey_scale_and_K():
    assert mvs.grey_scale(1600, 1200) == 1 and mvs.grey_scale(1601, 900) == 2 and mvs.grey_scale(4032, 3024) == 3
    assert mvs.grey_scale(100, 3300, 1600) == 3
    K = np.asarray([[1000.0, 0, 800.5], [0, 1010.0, 600.25], [0, 0, 1]], np.float32)
    Ks = mvs.scale_K(K, 2)
    assert Ks.dtype == np.float64 and np.array_equal(Ks, [[500.0, 0, 400.25], [0, 505.0, 300.125], [0, 0, 1]])
    # pixel (x, y) of the grey image covers block pixels [s x, s x + s): its centre s (x + 1/2) maps to x + 1/2 under K / s
    X = np.asarray([0.3, -0.2, 2.0])
    full = K.astype(np.float64) @ X
    half = Ks @ X
    assert np.allclose(full[:2] / full[2] / 2, half[:2] / half[2])
    rgb = np.arange(5 * 7 * 3, dtype=np.int64).reshape(5, 7, 3).astype(np.uint8) * 3
    g = OM.grey(rgb, 2)
    assert g.shape == (2, 3) and g.dtype == np.float32
    blk = rgb[2:4, 4:6].astype(np.int64)
    assert g[1, 2] == np.float32((299 * blk[..., 0] + 587 * blk[..., 1] + 114 * blk[..., 2]).sum()) / np.float32(255000 * 4)
    assert mvs.kinv32(Ks) == tuple(float(np.float32(v)) for v in (1 / 500.0, 1 / 505.0, -400.25 / 500.0, -300.125 / 505.0))


def test_oracle_patchmatch_recovers_a_textured_plane():
    w, h, f = 64, 48, 60.0
    K = np.asarray([[f, 0, w / 2], [0, f, h / 2], [0, 0, 1.0]])
    poses = [np.concatenate([np.eye(3), [[tx], [0.0], [0.0]]], 1) for tx in (0.0, -0.3, 0.3)]
    n = np.asarray([0.2, -0.1, -1.0])
    n /= np.linalg.norm(n)
    q = n @ [0.0, 0.0, 3.0]

    def render(P):
        C = -P[:, :3].T @ P[:, 3]
        ys, xs = np.mgrid[0:h, 0:w]
        d = np.stack([(xs + 0.5 - w / 2) / f, (ys + 0.5 - h / 2) / f, np.ones((h, w))], -1).reshape(-1, 3) @ P[:, :3]
        t = (q - C @ n) / (d @ n)
        a = 0.1 + 0.85 * OM.value_noise(C + t[:, None] * d, 0.08)
        return np.round(a * 255).astype(np.uint8).reshape(h, w)[..., None].repeat(3, -1), t.reshape(h, w)

    views = [render(P) for P in poses]
    g = [OM.grey(im, 1) for im, _ in views]
    geo = mvs.pm_table(K, poses[0], [K, K], poses[1:])
    v = OM.View(g[0], mvs.kinv32(K), OM.ref_stats(g[0], 4, 2), g[1:], geo, 2.0, 4.5, 4, 2, 0, 0)
    states = OM.patchmatch(v, 4)
    assert len(states) == 9
    costs = [float(c.mean()) for _, c in states]
    assert all(b <= a for a, b in zip(costs, costs[1:]))       # a pass never raises a pixel's cost
    d = states[-1][0][..., 0]
    err = np.abs(d - views[0][1]) / views[0][1]
    assert np.median(err) < 0.01 and (err < 0.01).mean() > 0.6, (np.median(err), (err < 0.01).mean())
    nrm = states[-1][0][..., 1:]
    assert np.allclose(np.linalg.norm(nrm, axis=-1), 1, atol=1e-5)


def test_dense_points_arguments(tmp_path, capsys):
    DP = tool('dense_points')
    root = str(tmp_path)
    with pytest.raises(SystemExit):
        DP.parse_args(['--root', os.path.join(root, 'missing')])
    with pytest.raises(SystemExit):
        DP.parse_args(['--root', root])                       # no model
    os.makedirs(os.path.join(root, 'sparse', '0'))
    with pytest.raises(SystemExit):
        DP.parse_args(['--root', root])                       # no images
    os.makedirs(os.path.join(root, 'images'))
    f = DP.parse_args(['--root', root])
    assert f.sparse == os.path.join(root, 'sparse', '0') and f.output == os.path.join(root, 'points.ply')
    assert (f.max_size, f.sources, f.iterations, f.radius, f.step) == (mvs.MAX_SIZE, mvs.SOURCES, mvs.ITERATIONS, mvs.RADIUS, mvs.STEP)
    for bad in (['--sources', '1'], ['--sources', '17'], ['--max-size', '0'], ['--iterations', '-1'], ['--step', '0'],
                ['--radius', '65'], ['--seed', '-1'], ['--voxel', '0']):
        with pytest.raises(SystemExit):
            DP.parse_args(['--root', root] + bad)
    open(os.path.join(root, 'points.ply'), 'w').close()
    with pytest.raises(SystemExit):
        DP.parse_args(['--root', root])
    assert DP.parse_args(['--root', root, '--force']).force
    assert 'already exists' in capsys.readouterr().err
