"""CPU: the COLMAP reader and the normalisation of nero_b200.objprep against NeRO's own read_model, _parse_colmap and
_normalize (tests/golden/objprep_colmap.npz, oracle/make_golden_objprep.py), the written files, known answers of the
custom-object oracle (oracle/nero_oracle_objprep.py) and the argument checks of tools/prepare_custom_object.py."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_objprep as O
from nero_b200 import objprep as OP
from nero_b200.evaluate import read_points_ply, write_points_ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, 'tests', 'golden', 'objprep_colmap.npz'))


def _model(tmp_path, fmt):
    d = tmp_path / fmt
    d.mkdir()
    for n in ('cameras', 'images', 'points3D'):
        (d / f'{n}.{fmt}').write_bytes(GOLD[f'{n}_{fmt}'].tobytes())
    return str(d)


@pytest.mark.parametrize('fmt', ['bin', 'txt'])
def test_reader_matches_reference(tmp_path, fmt):
    views, pts = OP.read_colmap_model(_model(tmp_path, fmt))
    assert list(views) == GOLD[f'ids_{fmt}'].tolist()
    assert [v[0] for v in views.values()] == GOLD[f'names_{fmt}'].tolist()
    poses = np.stack([v[1] for v in views.values()])
    Ks = np.stack([v[2] for v in views.values()])
    assert poses.dtype == np.float32 and Ks.dtype == np.float32
    assert np.array_equal(poses, GOLD[f'poses_{fmt}']) and np.array_equal(Ks, GOLD[f'Ks_{fmt}'])
    assert np.array_equal(pts, GOLD[f'points_{fmt}'])


def test_fixture_covers_the_camera_models():
    models = set()
    for ln in GOLD['cameras_txt'].tobytes().decode().splitlines():
        if ln and not ln.startswith('#'):
            models.add(ln.split()[1])
    assert models == {'PINHOLE', 'SIMPLE_RADIAL', 'SIMPLE_PINHOLE'}


@pytest.mark.parametrize('fmt', ['bin', 'txt'])
def test_unsupported_camera_model(tmp_path, fmt):
    cams = {1: ('OPENCV', 64, 48, [50.0, 50.0, 32.0, 24.0, 0.0, 0.0, 0.0, 0.0])}
    images = {1: (np.asarray([1.0, 0, 0, 0]), np.zeros(3), 1, 'a.png', np.zeros((0, 2)), np.zeros(0, np.int64))}
    O.write_colmap_model(str(tmp_path), cams, images, {}, fmt)
    with pytest.raises(NotImplementedError):
        OP.read_colmap_model(str(tmp_path))


def test_missing_model(tmp_path):
    with pytest.raises(FileNotFoundError):
        OP.read_colmap_model(str(tmp_path))


@pytest.mark.parametrize('fmt', ['bin', 'txt'])
def test_normalization_matches_reference(tmp_path, fmt):
    (tmp_path / 'o.ply').write_bytes(GOLD['ply'].tobytes())
    (tmp_path / 'm.txt').write_bytes(GOLD['meta_info'].tobytes())
    d = np.loadtxt(str(tmp_path / 'm.txt'))
    n = OP.normalization(read_points_ply(str(tmp_path / 'o.ply')), d[0], d[1])
    assert n['scale'] == GOLD[f'scale_rect_{fmt}']
    assert np.array_equal(n['offset'], GOLD[f'offset_rect_{fmt}'])
    np.testing.assert_allclose(n['R'], GOLD[f'R_rect_{fmt}'], rtol=0, atol=4e-16)
    np.testing.assert_allclose(n['ref_points'], GOLD[f'ref_points_{fmt}'], rtol=0, atol=4e-16)
    assert np.abs(n['ref_points']).max() <= 1 + 1e-12


def test_written_files_round_trip(tmp_path):
    write_points_ply(str(tmp_path / 'o.ply'), GOLD['obj'])
    OP.write_meta_info(str(tmp_path / 'm.txt'), GOLD['up'], GOLD['forward'])
    assert (tmp_path / 'o.ply').read_bytes() == GOLD['ply'].tobytes()
    assert (tmp_path / 'm.txt').read_bytes() == GOLD['meta_info'].tobytes()
    assert np.array_equal(read_points_ply(str(tmp_path / 'o.ply')), GOLD['obj'])
    d = np.loadtxt(str(tmp_path / 'm.txt'))
    assert d.shape == (2, 3) and np.array_equal(d[0], GOLD['up']) and np.array_equal(d[1], GOLD['forward'])


def test_object_center_and_forward():
    sc = O.scene(n_table=100, n_obj=100, n_cams=12, seed=5)
    views = {i: (f'v{i:02d}', P.astype(np.float32), np.eye(3, dtype=np.float32)) for i, P in enumerate(sc['poses'])}
    o, D, names, centers = OP.scene_scale(views)
    assert np.abs(o - sc['center']).max() < 1e-5 and abs(D - 3.0) < 1e-5 and names == sorted(names)
    f = OP.forward_direction(o, centers[0], sc['up'])
    assert abs(f @ sc['up']) < 1e-12 and abs(np.linalg.norm(f) - 1) < 1e-12 and f @ (centers[0] - o) > 0
    with pytest.raises(ValueError):
        OP.project_forward(3 * sc['up'], sc['up'])
    with pytest.raises(ValueError):
        OP.object_center(centers[:3], np.tile(sc['up'], (3, 1)))


# ------------------------------------------------------------------------------------------------ oracle known answers
def test_oracle_plane_counts():
    # 5 points on z = 1, 2 at z = 1.5, 1 at z = 0.995: the plane through the first three counts within tol
    p = np.asarray([[0, 0, 1], [1, 0, 1], [0, 1, 1], [2, 3, 1], [-1, 4, 1], [0, 0, 1.5], [1, 1, 1.5], [3, 3, 0.995]], np.float64)
    planes = np.asarray([[0, 0, 1, -1.0], [0, 0, -1, 1.5], [np.nan] * 4])
    assert O.counts(p, planes, 0.0).tolist() == [5, 2, 0]
    assert O.counts(p, planes, 0.01).tolist() == [6, 2, 0]
    _, out = O.moments(p, planes[0], 0.0, np.zeros(3))
    assert out[0] == 5 and np.array_equal(out[1:4], [2.0, 8.0, 5.0])
    _, out = O.moments(p, planes[0], 0.0, [0.4, 1.6, 1.0])
    assert abs(out[1]) < 1e-12 and abs(out[2]) < 1e-12 and out[9] == 0.0


def test_oracle_hypotheses():
    rng = np.random.RandomState(0)
    plane = np.concatenate([rng.rand(500, 2), np.full((500, 1), 2.0)], 1)
    planes, sample, valid = O.hypotheses(plane, 64, seed=7)
    assert valid.all() and ((sample >= 0) & (sample < 500)).all()
    assert np.allclose(np.abs(planes[:, 2]), 1) and np.allclose(planes[:, 3] * planes[:, 2], -2)
    # collinear points (exactly representable) and repeated points give only invalid hypotheses, written as NaN
    line = np.stack([np.arange(40.0), 2 * np.arange(40.0), np.full(40, 3.0)], 1)
    for pts in (line, np.tile([[1.0, 2.0, 3.0]], (40, 1))):
        planes, _, valid = O.hypotheses(pts, 32, seed=1)
        assert not valid.any() and np.isnan(planes).all() and not O.counts(pts, planes, 1.0).any()
    # the hash draws the same points whatever H is
    assert np.array_equal(O.hypotheses(plane, 8, 7)[1], O.hypotheses(plane, 64, 7)[1][:8])


def test_oracle_voxel_components():
    # two 26-connected groups (a diagonal chain and a separate voxel), keyed at an origin of 0
    vox = np.asarray([[0, 0, 0], [1, 1, 1], [2, 2, 2], [5, 0, 0], [5, 0, 2]], np.int64)
    keys = np.sort((vox[:, 0] << 42) | (vox[:, 1] << 21) | vox[:, 2])
    lab = O.voxel_components(keys)
    groups = {}
    for k, l in zip(keys, lab):
        groups.setdefault(int(l), []).append(int(k))
    assert sorted(len(g) for g in groups.values()) == [1, 1, 3] and all(l == min(np.searchsorted(keys, g)) for l, g in groups.items())
    cc, keep = O.component_select(lab, np.asarray([4, 1, 1, 1, 1]), 0.5)
    assert cc[0] == 6 and cc[3] == 1 and cc[4] == 1 and keep.tolist() == [True, True, True, False, False]


# ------------------------------------------------------------------------------------------------ the tool
def _tool():
    spec = importlib.util.spec_from_file_location('prepare_custom_object', os.path.join(ROOT, 'tools', 'prepare_custom_object.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tool_defaults_and_argument_errors(tmp_path):
    tool = _tool()
    root = tmp_path / 'kettle'
    with pytest.raises(SystemExit):
        tool.parse_args(['--root', str(root)])                       # no such directory
    root.mkdir()
    with pytest.raises(SystemExit):
        tool.parse_args(['--root', str(root)])                       # no model
    (root / 'sparse' / '0').mkdir(parents=True)
    f = tool.parse_args(['--root', str(root)])
    assert f.sparse == str(root / 'sparse' / '0') and f.points is None and f.hypotheses == 1024 and f.min_component == 1.0
    (root / 'colmap' / 'sparse' / '0').mkdir(parents=True)
    (root / 'points.ply').write_bytes(b'ply\n')
    f = tool.parse_args(['--root', str(root)])
    assert f.sparse == str(root / 'colmap' / 'sparse' / '0') and f.points == str(root / 'points.ply')
    (root / 'colmap' / 'point.ply').write_bytes(b'ply\n')
    assert tool.parse_args(['--root', str(root)]).points == str(root / 'colmap' / 'point.ply')
    for bad in (['--min-component', '1.5'], ['--hypotheses', '0'], ['--seed', '-1'], ['--crop-sphere', '0', '0', '0', '0'],
                ['--crop-box', '1', '0', '0', '0', '1', '1'], ['--tol', '0'], ['--voxel', '-1'], ['--up', '0', '0', '0'],
                ['--forward', '1', '0', '0', '--forward-image', 'a.jpg'], ['--points', str(root / 'none.ply')],
                ['--sparse', str(root / 'none')]):
        with pytest.raises(SystemExit):
            tool.parse_args(['--root', str(root)] + bad)
    (root / 'meta_info.txt').write_text('0 0 1\n1 0 0\n')
    with pytest.raises(SystemExit):
        tool.parse_args(['--root', str(root)])                       # refuses to overwrite
    assert tool.parse_args(['--root', str(root), '--force']).force
