"""GPU: the custom-object kernels (include/nero_objprep.h) against the numpy oracle bit for bit, the whole pipeline on a
synthetic scene against its ground truth, and tools/prepare_custom_object.py end to end on a synthetic project."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_objprep as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _np(t):
    return t.cpu().numpy()


def _scene_points(n, seed):
    sc = O.scene(n_table=int(n * 0.55) + 10, n_obj=int(n * 0.35) + 10, seed=seed)
    return sc, np.ascontiguousarray(sc['points'][:n])


def _check_kernels(p, sphere, H, tol, seed, above, voxel, frac):
    import torch
    from nero_b200 import objprep as OP
    plane, info = OP.fit_support_plane(p, tol, sphere, None, H, seed)
    keep = O.crop(p, sphere)
    assert np.array_equal(_np(info['keep']).astype(bool), keep)
    assert np.array_equal(_np(info['kept_index']), np.nonzero(keep)[0])
    kept = p[keep]
    planes, sample, valid = O.hypotheses(kept, H, seed)
    assert np.array_equal(_np(info['sample']), sample) and np.array_equal(_np(info['valid']).astype(bool), valid)
    assert np.array_equal(_np(info['planes']), planes, equal_nan=True)
    counts = O.counts(kept, planes, tol)
    assert np.array_equal(_np(info['counts']), counts)
    assert info['best'] == int(np.argmax(counts))
    pl = planes[info['best']]
    kg = torch.from_numpy(kept).cuda()
    for rp, cen, S, cnt in info['refits']:                      # each round's sums from the GPU's previous plane
        _, s = O.moments(kept, pl, tol, np.zeros(3))
        assert s[0] == cnt and np.array_equal(s[1:4] / s[0], cen)
        part, m = O.moments(kept, pl, tol, cen)
        gpart, gm = OP._moments(kg, pl, tol, cen)
        assert np.array_equal(_np(gpart), part) and np.array_equal(gm, m)
        assert np.array_equal(np.asarray([[m[4], m[5], m[6]], [m[5], m[7], m[8]], [m[6], m[8], m[9]]]), S)
        pl = rp
    obj, iinfo = OP.isolate_object(p, plane, above, voxel, sphere, None, frac)
    ref = O.isolate(p, keep, plane, above, kept.min(0), voxel, frac)
    assert np.array_equal(_np(iinfo['flag']).astype(bool), ref['flag']) and np.array_equal(_np(iinfo['keys']), ref['keys'])
    assert np.array_equal(_np(iinfo['ukeys']), ref['ukeys']) and np.array_equal(_np(iinfo['vcount']), ref['vcount'])
    assert np.array_equal(_np(iinfo['label']), ref['label'])
    assert np.array_equal(_np(iinfo['comp_count']), ref['comp_count'])
    assert np.array_equal(_np(iinfo['voxel_keep']).astype(bool), ref['voxel_keep'])
    assert np.array_equal(_np(iinfo['point_keep']).astype(bool), ref['point_keep'])
    assert np.array_equal(_np(iinfo['index']), ref['index']) and np.array_equal(_np(obj), p[ref['index']])
    return info, iinfo


@pytest.mark.parametrize('n,H', [(1000, 1024), (4096 * 3 + 77, 300), (2_000_000, 16)])
def test_kernels_match_oracle(n, H):
    sc, p = _scene_points(n, seed=n % 7)
    sphere = list(sc['center']) + [1.5]
    info, iinfo = _check_kernels(p, sphere, H, 0.006, 11, 0.012, 0.03, 0.5)
    assert info['kept'] < n and iinfo['kept'] > 0


def test_three_points_and_degenerate_hypotheses():
    p = np.asarray([[0.0, 0.0, 1.0], [1.0, 0.0, 1.0], [0.0, 1.0, 1.0]])
    info, _ = _check_kernels(p, None, 64, 1e-9, 3, -1.0, 0.5, 1.0)
    v = _np(info['valid']).astype(bool)
    assert v.any() and not v.all()                              # draws with a repeated index are invalid
    assert (_np(info['counts'])[v] == 3).all() and (_np(info['counts'])[~v] == 0).all()


def test_collinear_cloud_is_refused():
    from nero_b200 import objprep as OP
    line = np.stack([np.arange(50.0), 2 * np.arange(50.0), np.full(50, 3.0)], 1)
    with pytest.raises(ValueError):
        OP.fit_support_plane(line, 0.1)


def test_bad_clouds_raise():
    from nero_b200 import objprep as OP
    with pytest.raises(ValueError):
        OP.fit_support_plane(np.zeros((2, 3)), 0.1)
    p = np.random.RandomState(0).rand(100, 3)
    with pytest.raises(ValueError):
        OP.fit_support_plane(p, 0.1, sphere=[5.0, 5.0, 5.0, 0.5])       # fully cropped
    with pytest.raises(ValueError):
        OP.fit_support_plane(p, 0.1, box=[2, 2, 2, 3, 3, 3])
    with pytest.raises(ValueError):
        OP.isolate_object(p, [0, 0, 1, 0.0], 0.1, 0.05, sphere=[5.0, 5.0, 5.0, 0.5])
    with pytest.raises(ValueError):
        OP.isolate_object(p, [0, 0, 1, -2.0], 0.1, 0.05)               # nothing above the plane


def test_pipeline_on_synthetic_scene():
    from nero_b200 import objprep as OP
    sc = O.scene(seed=2)
    views = {i: (f'v{i:02d}', P.astype(np.float32), np.eye(3, dtype=np.float32)) for i, P in enumerate(sc['poses'])}
    center, D, names, centers = OP.scene_scale(views)
    sphere = list(center) + [OP.CROP_FRAC * D]
    tol = OP.TOL_FRAC * D
    plane, info = OP.fit_support_plane(sc['points'], tol, sphere, None, 1024, 0, centers)
    ang = np.degrees(np.arccos(min(1.0, plane[:3] @ sc['up'])))
    assert ang < 0.5, f'up is {ang} degrees from the truth'
    obj, iinfo = OP.isolate_object(sc['points'], plane, OP.ABOVE_TOLS * tol, OP.VOXEL_FRAC * D, sphere, None, 1.0)
    k = _np(iinfo['point_keep']).astype(bool)
    lab = sc['label']
    recall = (k & (lab == 1)).sum() / (lab == 1).sum()
    foreign = (k & (lab != 1)).sum() / k.sum()
    assert recall >= 0.99 and foreign <= 0.01, (recall, foreign)
    f = OP.forward_direction(center, centers[0], plane[:3])
    norm = OP.normalization(_np(obj), plane[:3], f, centers)
    assert np.linalg.norm(norm['ref_points'], axis=1).max() <= 1 + 1e-12
    assert not norm['inside'].any() and norm['camera_dist'].min() > 1


def _tool():
    spec = importlib.util.spec_from_file_location('prepare_custom_object', os.path.join(ROOT, 'tools', 'prepare_custom_object.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tool_end_to_end(tmp_path, capsys):
    from nero_b200 import objprep as OP
    from nero_b200.evaluate import read_points_ply, write_points_ply
    sc = O.scene(n_table=60000, n_obj=40000, seed=4)
    root = tmp_path / 'synthetic'
    cams, images, points = O.scene_model(sc)
    O.write_colmap_model(str(root / 'colmap' / 'sparse' / '0'), cams, images, points, 'bin')
    write_points_ply(str(root / 'colmap' / 'point.ply'), sc['points'])
    tool = _tool()
    tool.main(['--root', str(root), '--preview', 'img_003.jpg'])
    out = capsys.readouterr().out
    assert 'plane: normal' in out and 'closest normalised camera distance' in out
    first = {f: (root / f).read_bytes() for f in tool.OUTPUTS}
    assert (root / 'object_preview.png').read_bytes()[:8] == b'\x89PNG\r\n\x1a\n'
    with pytest.raises(SystemExit):
        tool.main(['--root', str(root)])                               # refuses to overwrite
    tool.main(['--root', str(root), '--force'])
    assert all((root / f).read_bytes() == b for f, b in first.items()), 'two runs wrote different files'
    d = np.loadtxt(str(root / 'meta_info.txt'))
    assert d.shape == (2, 3) and np.degrees(np.arccos(min(1.0, d[0] @ sc['up']))) < 0.5 and abs(d[0] @ d[1]) < 1e-9
    pts = read_points_ply(str(root / 'object_point_cloud.ply'))
    views, _ = OP.read_colmap_model(str(root / 'colmap' / 'sparse' / '0'))
    norm = OP.normalization(pts, d[0], d[1], OP.camera_centers(views)[1])
    assert not norm['inside'].any()
    # --up and --forward-image override the fit and the default camera
    tool.main(['--root', str(root), '--force', '--up', '0', '0', '1', '--forward-image', 'img_010.jpg'])
    d2 = np.loadtxt(str(root / 'meta_info.txt'))
    assert np.array_equal(d2[0], [0, 0, 1]) and abs(d2[1][2]) < 1e-12
