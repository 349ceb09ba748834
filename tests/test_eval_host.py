"""CPU: the shape-evaluation oracle against the reference glue's golden output, the rasteriser against a ray cast, the voxel
oracle, point-cloud PLY files, the GlossySynthetic readers and the kernels' register use.  No GPU needed."""
import os
import pickle
import re
import subprocess

import numpy as np
import pytest

import nero_oracle_eval as OE
from nero_b200 import evaluate as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = np.load(os.path.join(ROOT, 'tests', 'golden', 'eval_shape.npz'))


def golden_views():
    order = [int(i) for i in GOLD['ids']]
    h, w = (int(x) for x in GOLD['hw'])
    # the reference casts the stored cameras to float32 (GlossySyntheticDatabase.get_pose / get_K)
    return [(GOLD['poses'][k].astype(np.float32), GOLD['Ks'][k].astype(np.float32), (h, w)) for k in order], order


# ------------------------------------------------------------------------------------------------ golden fixture
def test_clip_space_vertices_match_reference():
    views, _ = golden_views()
    for (pose, K, (h, w)), clip in zip(views, GOLD['clip']):
        ours = OE.project_clip(GOLD['verts'].astype(np.float32), pose, K, h, w)
        # the reference projects in float32; the oracle in float64
        np.testing.assert_allclose(ours, clip, rtol=0, atol=1e-6)
        assert (clip[:, 3] == 1).all()


def test_predicted_points_match_reference():
    views, _ = golden_views()
    pts = []
    for pose, K, (h, w) in views:
        depth, mask = OE.render_depth(GOLD['verts'].astype(np.float32), GOLD['tris'], pose, K, h, w)
        pts.append(OE.depth_to_points(depth, mask, K, pose))
    pts = np.concatenate(pts, 0)
    ref = GOLD['pr_points_in']
    assert pts.shape == ref.shape
    # float32 depth round trip through clip-space z in the reference: about 1e-6 of the point's distance from the camera
    np.testing.assert_allclose(pts, ref, rtol=0, atol=1e-5)


def test_gt_points_match_reference():
    views, order = golden_views()
    pts = np.concatenate([OE.depth_to_points(d, d < 14.5, K, pose)
                          for d, (pose, K, _) in zip([GOLD['depth_png'][k].astype(np.float32) / 65535 * 15 for k in order], views)], 0)
    ref = GOLD['gt_points_in']
    assert pts.shape == ref.shape
    np.testing.assert_allclose(pts, ref, rtol=0, atol=2e-6)


def test_nearest_dist_and_chamfer_match_reference():
    d_gt = OE.nearest_dist(GOLD['pts_gt'], GOLD['pts_pr'])
    d_pr = OE.nearest_dist(GOLD['pts_pr'], GOLD['pts_gt'])
    np.testing.assert_allclose(d_gt, GOLD['dist_gt'], rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(d_pr, GOLD['dist_pr'], rtol=1e-6, atol=1e-7)
    c = (np.mean(GOLD['dist_gt']) + np.mean(GOLD['dist_pr'])) / 2
    assert c == GOLD['chamfer_exact']
    assert E.result_line('fixture_mesh', c) == f'fixture_mesh {float(GOLD["chamfer"]):.5f}'
    assert abs(OE.chamfer(GOLD['pts_gt'], GOLD['pts_pr'])[0] - c) < 1e-6


# ------------------------------------------------------------------------------------------------ rule 1
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_rasteriser_equals_ray_cast_depth(seed):
    rng = np.random.RandomState(seed)
    verts = rng.uniform(-0.6, 0.6, (30, 3))
    tris = rng.randint(0, 30, (40, 3))
    tris = tris[(tris[:, 0] != tris[:, 1]) & (tris[:, 1] != tris[:, 2]) & (tris[:, 0] != tris[:, 2])]
    pose = np.concatenate([np.eye(3), [[0.1], [-0.05], [2.0]]], 1)
    K = np.asarray([[22.0, 0, 13.3], [0, 25.0, 9.6], [0, 0, 1]])
    h, w = 20, 28
    rast = OE.rasterize(OE.project_clip(verts, pose, K, h, w), tris, h, w)
    rd, rid = OE.raycast_depth(verts, tris, pose, K, h, w)
    same = (rast[..., 3] - 1 == rid) & (rid >= 0)
    assert same.sum() > 100
    assert ((rast[..., 3] > 0) == (rid >= 0)).mean() > 0.97
    zr = (rast[..., 2] + 1) / 2 * (OE.FAR - OE.NEAR) + OE.NEAR
    np.testing.assert_allclose(zr[same], rd[same], rtol=1e-12, atol=0)


def test_half_pixel_and_clip_rules():
    # a fronto-parallel square at depth 2 covering pixel centres only: unprojected at integer coordinates
    verts = np.asarray([[-3, -3, 2], [3, -3, 2], [3, 3, 2], [-3, 3, 2]], np.float64)
    tris = np.asarray([[0, 1, 2], [0, 2, 3]])
    pose = np.concatenate([np.eye(3), np.zeros((3, 1))], 1)
    K = np.asarray([[4.0, 0, 4.0], [0, 4.0, 4.0], [0, 0, 1]])
    depth, mask = OE.render_depth(verts, tris, pose, K, 8, 8)
    assert mask.all() and np.allclose(depth, 2.0)
    pts = OE.depth_to_points(depth, mask, K, pose)
    np.testing.assert_allclose(pts[0], [(0 - 4) * 2 / 4, (0 - 4) * 2 / 4, 2])
    # behind the near plane or beyond the far plane: clipped
    for z in (0.4, 101.0):
        _, m = OE.render_depth(verts * [z / 2, z / 2, z / 2], tris, pose, K, 8, 8)
        assert not m.any()


# ------------------------------------------------------------------------------------------------ voxel oracle
def test_voxel_oracle_bound_means_order_and_range():
    p = np.asarray([[0.0, 0.0, 0.0], [0.004, 0.0, 0.0], [0.006, 0.0, 0.0], [0.0, 0.012, 0.0], [0.0, 0.0, 0.0149]])
    out = OE.voxel_down_sample(p, 0.01)
    # min bound = -0.005: x = 0.004 shares voxel 0 with 0, 0.006 is in voxel 1; z = 0.0149 < 0.015 stays in voxel 1
    # keys (0,0,0) < (0,0,1) < (0,1,0) < (1,0,0)
    np.testing.assert_array_equal(out, [[0.002, 0.0, 0.0], [0.0, 0.0, 0.0149], [0.0, 0.012, 0.0], [0.006, 0.0, 0.0]])
    rng = np.random.RandomState(3)
    q = rng.rand(2000, 3)
    o = OE.voxel_down_sample(q, 0.1)
    lo = q.min(0) - 0.05
    idx = np.floor((o - lo) / 0.1).astype(np.int64)
    key = (idx[:, 0] << 42) | (idx[:, 1] << 21) | idx[:, 2]
    assert (np.diff(key) > 0).all()
    assert abs(o.mean(0) - q.mean(0)).max() < 0.05
    with pytest.raises(ValueError):
        OE.voxel_down_sample(np.asarray([[0.0, 0, 0], [30000.0, 0, 0]]), 0.01)


# ------------------------------------------------------------------------------------------------ PLY
def _ply(path, fmt, props, rows, extra=''):
    head = f'ply\nformat {fmt} 1.0\ncomment test\nelement vertex {len(rows)}\n'
    head += ''.join(f'property {t} {n}\n' for t, n in props) + extra + 'end_header\n'
    with open(path, 'wb') as f:
        f.write(head.encode())
        if fmt == 'ascii':
            f.write(''.join(' '.join(repr(v) for v in r) + '\n' for r in rows).encode())
        else:
            f.write(np.asarray([tuple(r) for r in rows], dtype=[(n, '<' + {'float': 'f4', 'double': 'f8', 'uchar': 'u1'}[t])
                                                                for t, n in props]).tobytes())


@pytest.mark.parametrize('fmt', ['ascii', 'binary_little_endian'])
@pytest.mark.parametrize('ftype', ['float', 'double'])
def test_point_ply_reader(tmp_path, fmt, ftype):
    rng = np.random.RandomState(1)
    xyz = rng.randn(7, 3).astype(np.float32 if ftype == 'float' else np.float64)
    rows = [[float(v) for v in r] + [int(c)] for r, c in zip(xyz, rng.randint(0, 255, 7))]
    path = tmp_path / 'a.ply'
    props = [(ftype, 'x'), (ftype, 'y'), (ftype, 'z'), ('uchar', 'red')]
    _ply(path, fmt, props, rows, extra='element face 0\nproperty list uchar int vertex_indices\n')
    got = E.read_points_ply(str(path))
    assert got.dtype == np.float64
    np.testing.assert_array_equal(got, xyz.astype(np.float64))


def test_point_ply_reader_reads_meshes_and_rejects_others(tmp_path):
    from nero_b200.mesh import write_ply
    v = np.random.RandomState(2).rand(5, 3).astype(np.float32)
    write_ply(str(tmp_path / 'm.ply'), v, np.asarray([[0, 1, 2], [2, 3, 4]]))
    np.testing.assert_array_equal(E.read_points_ply(str(tmp_path / 'm.ply')), v.astype(np.float64))
    (tmp_path / 'b.ply').write_bytes(b'ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nend_header\n')
    with pytest.raises(ValueError):
        E.read_points_ply(str(tmp_path / 'b.ply'))
    (tmp_path / 'c.ply').write_bytes(b'ply\nformat ascii 1.0\nelement face 0\nproperty list uchar int vertex_indices\n'
                                     b'element vertex 0\nproperty float x\nproperty float y\nproperty float z\nend_header\n')
    with pytest.raises(ValueError):
        E.read_points_ply(str(tmp_path / 'c.ply'))


def test_point_ply_writer_round_trip_and_open3d_header(tmp_path):
    p = np.random.RandomState(4).randn(11, 3)
    path = str(tmp_path / 'eval_pts.ply')
    E.write_points_ply(path, p)
    np.testing.assert_array_equal(E.read_points_ply(path), p)
    data = open(path, 'rb').read()
    head, body = data.split(b'end_header\n', 1)
    lines = head.decode('ascii').split('\n')[:-1]
    # Open3D's reader (rply): magic, format line, then comment / element / property lines, then end_header
    assert lines[0] == 'ply' and lines[1] == 'format binary_little_endian 1.0'
    assert all(re.fullmatch(r'(comment .*|element vertex \d+|property double [xyz])', l) for l in lines[2:])
    assert [l for l in lines if l.startswith('property')] == ['property double x', 'property double y', 'property double z']
    assert len(body) == 11 * 24


# ------------------------------------------------------------------------------------------------ GlossySynthetic readers
def test_glossy_synthetic_directory(tmp_path):
    import cv2
    root = tmp_path / 'data' / 'GlossySynthetic' / 'obj'
    root.mkdir(parents=True)
    rng = np.random.RandomState(5)
    for k in range(3):
        pose = rng.randn(3, 4)
        K = np.asarray([[40.0 + k, 0, 10.0], [0, 41.0, 7.0], [0, 0, 1]])
        with open(root / f'{k}-camera.pkl', 'wb') as f:
            pickle.dump([pose, K], f)
        cv2.imwrite(str(root / f'{k}.png'), np.zeros((15, 21, 3), np.uint8))
        cv2.imwrite(str(root / f'{k}-depth.png'), (np.arange(15 * 21).reshape(15, 21) * 150 + k).astype(np.uint16))
    split = tmp_path / 'split.pkl'
    with open(split, 'wb') as f:
        pickle.dump([np.asarray(['2', '0']), ['1']], f)
    ids = E.split_test_ids(str(split))
    assert ids == ['2', '0']
    views = E.read_views(str(root), ids)
    assert views[0][2] == (15, 21) and views[0][0].dtype == np.float32 and views[0][1][0, 0] == np.float32(42.0)
    d = E.read_gt_depth(str(root), '2')
    raw = (np.arange(15 * 21).reshape(15, 21) * 150 + 2).astype(np.uint16)
    np.testing.assert_array_equal(d, raw.astype(np.float32) / 65535 * 15)
    assert d.dtype == np.float32


# ------------------------------------------------------------------------------------------------ compiled code
def test_eval_kernels_do_not_spill():
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    src = os.path.join(ROOT, 'nero_b200', 'csrc', 'k_eval.cu')
    out = subprocess.run([nvcc, '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17', '--expt-relaxed-constexpr',
                          '-Xptxas', '-v', '-c', src, '-o', os.devnull], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    kernels = re.findall(r"Compiling entry function '(\w+)'.*?(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                         out.stderr, re.S)
    names = {k[0] for k in kernels}
    for want in ('depth_render_kernel', 'points_count_kernel', 'block_offsets_kernel', 'points_emit_kernel', 'voxel_keys_kernel',
                 'voxel_mean_kernel', 'nearest_kernel'):
        assert any(want in n for n in names), want
    for name, stack, st, ld in kernels:
        assert st == '0' and ld == '0', name
        # only the ray caster has a stack frame: the 48-entry traversal stack of bvh_traverse.cuh
        assert int(stack) == 0 or ('depth_render_kernel' in name and int(stack) <= 48 * 4), (name, stack)
