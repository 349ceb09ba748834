"""Shape evaluation on the GPU: the depth kernel against the oracle rasteriser, point compaction, voxel down-sampling, nearest
distances, and the two tools end to end on a synthetic dataset of an analytic sphere."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_eval as OE
import nero_oracle_mat as OM
from nero_b200 import evaluate as E
from nero_b200.mesh import marching_cubes, write_ply

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def look_at(c, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """World -> camera [3,4], OpenCV axes, camera at c looking at target."""
    c = np.asarray(c, np.float64)
    z = np.asarray(target, np.float64) - c
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 0)
    return np.concatenate([R, (-R @ c)[:, None]], 1)


def sphere_mesh(radius, res=64):
    """GPU marching cubes of the SDF |x| - radius on a res^3 grid over [-1,1]^3, in world coordinates."""
    ax = np.linspace(-1.0, 1.0, res)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    v, t = marching_cubes((np.linalg.norm(x, axis=-1) - radius).astype(np.float32), 0.0)
    return (-1.0 + 2.0 * v / (res - 1)).astype(np.float32), t


def silhouette(cover):
    """Pixels whose 3x3 neighbourhood holds both covered and uncovered pixels."""
    p = np.pad(cover, 1, mode='edge')
    h, w = cover.shape
    nb = np.stack([p[i:i + h, j:j + w] for i in range(3) for j in range(3)])
    return nb.any(0) & ~nb.all(0)


CAMERAS = [((2.2, 0.4, 0.6), (40, 56), (50.0, 47.0, 29.3, 18.1)),
           ((-0.7, 1.9, -0.9), (48, 36), (44.0, 44.0, 16.2, 25.0)),
           ((0.3, -1.2, 2.1), (33, 61), (58.0, 55.0, 31.0, 15.5))]


def camera(i):
    c, (h, w), (fx, fy, cx, cy) = CAMERAS[i]
    return look_at(c).astype(np.float32), np.asarray([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32), h, w


@pytest.mark.parametrize('scene', ['two_spheres', 'mcubes'])
@pytest.mark.parametrize('view', [0, 1, 2])
def test_depth_kernel_matches_oracle_rasteriser(scene, view):
    verts, tris = OM.test_scene(2) if scene == 'two_spheres' else sphere_mesh(0.55, 40)
    pose, K, h, w = camera(view)
    got = E.DepthRenderer(verts, tris).render(pose, K, h, w).cpu().numpy()
    ref, cover = OE.render_depth(verts, tris, pose, K, h, w)
    mine = got > 0
    diff = mine != cover
    assert cover.mean() > 0.1
    assert diff.mean() <= 1e-3 or diff.sum() <= 2, f'{diff.sum()} pixels differ in coverage'
    assert not (diff & ~silhouette(cover)).any(), 'coverage differs away from the silhouette'
    both = mine & cover
    np.testing.assert_allclose(got[both], ref[both], rtol=1e-5, atol=0)
    assert (got[~mine] == 0).all()


def test_depth_kernel_far_clip_and_validation():
    verts, tris = OM.test_scene(2)
    pose, K, h, w = camera(0)
    r = E.DepthRenderer(verts, tris)
    far = 2.0                                      # cuts through the front of the two-sphere scene
    got = r.render(pose, K, h, w, far=far).cpu().numpy()
    ref, cover = OE.render_depth(verts, tris, pose, K, h, w, far=far)
    full = r.render(pose, K, h, w).cpu().numpy()
    assert ((full > far) & (got == 0)).sum() > 10, 'some pixels must be clipped by the far plane'
    assert ((got > 0) != cover).sum() <= max(2, 1e-3 * h * w) + silhouette(cover).sum()
    assert (got <= far).all()
    with pytest.raises(ValueError):
        r.render(pose, np.asarray([[50.0, 0.5, 20], [0, 50, 20], [0, 0, 1]]), h, w)


def test_points_match_oracle_order_and_values():
    verts, tris = OM.test_scene(2)
    r = E.DepthRenderer(verts, tris)
    depths, poses, Ks = [], [], []
    for i in (0, 1):
        pose, K, _, _ = camera(i)
        depths.append(r.render(pose, K, 40, 56))
        poses.append(pose)
        Ks.append(K)
    got = E.depth_to_points_cuda(torch.stack(depths), poses, Ks).cpu().numpy()
    ref = np.concatenate([OE.depth_to_points(d.cpu().numpy(), d.cpu().numpy() > 0, K, p) for d, p, K in zip(depths, poses, Ks)], 0)
    assert got.shape == ref.shape and got.shape[0] > 100
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())
    # three 640 x 640 views: 1 228 800 pixels in 1200 blocks, so the block offsets carry a sum across their 1024-block chunks
    K = np.asarray([[800.0, 0, 320], [0, 800.0, 320], [0, 0, 1]], np.float32)
    poses = [camera(i)[0] for i in range(3)]
    depths = torch.stack([r.render(p, K, 640, 640) for p in poses])
    assert (depths.reshape(-1)[:1024 * 1024] > 0).any() and (depths.reshape(-1)[1024 * 1024:] > 0).any()
    got = E.depth_to_points_cuda(depths, poses, [K] * 3).cpu().numpy()
    ref = np.concatenate([OE.depth_to_points(d.cpu().numpy(), d.cpu().numpy() > 0, K, p) for d, p in zip(depths, poses)], 0)
    assert got.shape == ref.shape
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())
    # the ground-truth mask (-inf, 14.5) of a 16-bit depth map
    raw = np.random.RandomState(0).randint(0, 65536, (37, 29)).astype(np.uint16)
    d = raw.astype(np.float32) / 65535 * 15
    pose, K, _, _ = camera(2)
    got = E.depth_to_points(d, K, pose, float('-inf'), 14.5)
    ref = OE.depth_to_points(d, d < 14.5, K, pose)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-6 * np.abs(ref).max())


def test_voxel_down_sampling_is_bit_identical_to_oracle():
    rng = np.random.RandomState(7)
    p = rng.rand(20000, 3) * [0.3, 0.2, 0.25]
    p = np.concatenate([p, p[:500]], 0)               # duplicate points
    got = E.voxel_down_sample(p, 0.01)
    ref = OE.voxel_down_sample(p, 0.01)
    np.testing.assert_array_equal(got, ref)
    lo = p.min(0) - 0.005
    idx = np.floor((got - lo) / 0.01).astype(np.int64)
    key = (idx[:, 0] << 42) | (idx[:, 1] << 21) | idx[:, 2]
    assert (np.diff(key) > 0).all()
    pts = E.depth_to_points_cuda(E.DepthRenderer(*OM.test_scene(2)).render(*camera(0)), camera(0)[0], camera(0)[1])
    np.testing.assert_array_equal(E.voxel_down_sample_cuda(pts, 0.01).cpu().numpy(), OE.voxel_down_sample(pts.cpu().numpy(), 0.01))
    with pytest.raises(ValueError):
        E.voxel_down_sample(np.asarray([[0.0, 0, 0], [30000.0, 0, 0]]), 0.01)


def _ref_torch_formula(q, t, bs=512):
    """eval_synthetic_shape.nearest_dist's formula: torch fp32 norm of the difference, minimum."""
    q = torch.from_numpy(np.asarray(q, np.float32)).cuda()
    t = torch.from_numpy(np.asarray(t, np.float32)).cuda()
    return torch.cat([torch.norm(q[i:i + bs, None, :] - t[None], dim=-1).min(1)[0] for i in range(0, q.shape[0], bs)]).cpu().numpy()


@pytest.mark.parametrize('n,m', [(1, 1), (1, 1500), (1000, 777), (1031, 2049), (4097, 3)])
def test_nearest_dist_exact(n, m):
    rng = np.random.RandomState(n + m)
    q = rng.randn(n, 3).astype(np.float32)
    t = rng.randn(m, 3).astype(np.float32)
    got = E.nearest_dist(q, t)
    ref = OE.nearest_dist(q, t)
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)
    tf = _ref_torch_formula(q, t)
    assert (np.abs(got - tf) <= 2 * np.spacing(tf)).all()


def test_nearest_dist_duplicates_ties_and_empty():
    t = np.asarray([[0, 0, 0], [0, 0, 0], [1, 0, 0], [-1, 0, 0]], np.float32)
    q = np.asarray([[0, 0, 0], [0.5, 0, 0], [0, 1, 0], [1, 0, 0]], np.float32)
    np.testing.assert_array_equal(E.nearest_dist(q, t), np.asarray([0, 0.5, 1, 0], np.float32))
    for a, b in ((np.zeros((0, 3)), t), (q, np.zeros((0, 3)))):
        with pytest.raises(ValueError):
            E.nearest_dist(a, b)


def test_nearest_dist_200k():
    rng = np.random.RandomState(11)
    q = torch.from_numpy(rng.rand(200_000, 3).astype(np.float32)).cuda()
    t = torch.from_numpy(rng.rand(200_003, 3).astype(np.float32)).cuda()
    got = E.nearest_dist_cuda(q, t)
    assert torch.equal(got, E.nearest_dist_cuda(q, t))
    sub = torch.from_numpy(rng.choice(200_000, 1500, replace=False)).cuda()
    qd, td = q[sub].double(), t.double()
    ref = torch.cat([torch.cdist(qd[i:i + 250], td, compute_mode='donot_use_mm_for_euclid_dist').min(1)[0] for i in range(0, qd.shape[0], 250)])
    np.testing.assert_allclose(got[sub].double().cpu().numpy(), ref.cpu().numpy(), rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ end to end
RADIUS, DELTA, RES = 0.5, 0.05, 96
RING = [(2.0 * np.cos(a) * np.cos(e), 2.0 * np.sin(a) * np.cos(e), 2.0 * np.sin(e))
        for e in (-0.5, 0.0, 0.5) for a in np.linspace(0, 2 * np.pi, 4, endpoint=False) + e]
GT_H, GT_W, GT_K = 240, 300, np.asarray([[280.0, 0, 150.3], [0, 280.0, 119.6], [0, 0, 1]])


def sphere_depth_png(pose, K, h, w, radius):
    """16-bit GlossySynthetic depth of an analytic sphere: camera z of the first hit of the ray through each pixel centre,
    v = round(z / 15 * 65535), 65535 where the ray misses."""
    o, d = OE.pixel_rays(pose, K, h, w)
    b = d @ o
    a = (d * d).sum(-1)
    disc = b * b - a * ((o * o).sum() - radius * radius)
    t = (-b - np.sqrt(np.maximum(disc, 0))) / a
    z = np.where(disc > 0, t, 15.0)                # d has camera z component 1, so t is the camera depth
    return np.round(np.clip(z, 0, 15) / 15 * 65535).astype(np.uint16).reshape(h, w)


def make_dataset(root, split):
    import cv2
    os.makedirs(root, exist_ok=True)
    for k, c in enumerate(RING):
        pose = look_at(c)
        with open(os.path.join(root, f'{k}-camera.pkl'), 'wb') as f:
            pickle.dump([pose, GT_K], f)
        cv2.imwrite(os.path.join(root, f'{k}.png'), np.zeros((GT_H, GT_W, 3), np.uint8))
        cv2.imwrite(os.path.join(root, f'{k}-depth.png'), sphere_depth_png(pose, GT_K, GT_H, GT_W, RADIUS))
    os.makedirs(os.path.dirname(split), exist_ok=True)
    with open(split, 'wb') as f:
        pickle.dump([np.asarray([str(k) for k in range(len(RING))][::-1]), []], f)


@pytest.fixture(scope='module')
def workspace(tmp_path_factory):
    ws = tmp_path_factory.mktemp('eval')
    make_dataset(str(ws / 'data' / 'GlossySynthetic' / 'ball'), str(ws / 'configs' / 'synthetic_split_128.pkl'))
    v, t = sphere_mesh(RADIUS + DELTA, RES)
    write_ply(str(ws / 'ball_pred.ply'), v, t)
    return ws


def test_chamfer_of_a_dilated_sphere(workspace):
    root = str(workspace / 'data' / 'GlossySynthetic' / 'ball')
    split = str(workspace / 'configs' / 'synthetic_split_128.pkl')
    ids = E.split_test_ids(split)
    views = E.read_views(root, ids)
    gt = E.gt_eval_points_cuda(root, ids, views)
    from nero_b200.material import read_ply
    verts, tris = read_ply(str(workspace / 'ball_pred.ply'))
    pr = E.mesh_eval_points_cuda(verts, tris, views)
    c, dg, dp = E.chamfer_distance(gt.cpu().numpy().astype(np.float32), pr.cpu().numpy().astype(np.float32))
    # Both clouds lie on concentric spheres DELTA apart, up to: the marching-cubes chord error (< h^2 / (8 R), h the grid
    # step, plus the vertex interpolation error of a linear fit to |x|, < h^2 / (2 R)) and 16-bit depth quantisation
    # (15 / 65535 / 2).  Unprojecting at (x, y) what was seen at (x + 1/2, y + 1/2) moves each view's points by at most
    # s = sqrt(2) / 2 * z_max / f, differently per view, so a point's nearest neighbour from another view can be up to 2 s
    # closer or farther.  Every point of one cloud has a point of the other within the diagonal of a voxel of the radial
    # direction, so DELTA - 2 s - eps <= chamfer <= sqrt(DELTA^2 + 3 voxel^2) + 2 s + eps.
    h = 2.0 / (RES - 1)
    s = np.sqrt(2) / 2 * (2.0 + RADIUS + DELTA) / GT_K[0, 0]
    eps = h * h / (8 * RADIUS) + h * h / (2 * RADIUS) + 15 / 65535 / 2 + 2 * s + 1e-4
    assert DELTA - eps <= c <= np.sqrt(DELTA ** 2 + 3 * E.VOXEL ** 2) + eps, (c, eps)
    # the oracle pipeline on the kernel's depth maps: points within 1e-6, voxel means of those points bit-identical, Chamfer
    r = E.DepthRenderer(verts, tris)
    dpr = [r.render(p, K, hh, ww).cpu().numpy() for p, K, (hh, ww) in views]
    dgt = [E.read_gt_depth(root, i) for i in ids]
    for dm, lo, hi, cloud in ((dpr, 0.0, np.inf, pr), (dgt, -np.inf, 14.5, gt)):
        mine = np.concatenate([E.depth_to_points(d, K, p, lo, hi) for d, (p, K, _) in zip(dm, views)], 0)
        ref = np.concatenate([OE.depth_to_points(d, (d > lo) & (d < hi), K, p) for d, (p, K, _) in zip(dm, views)], 0)
        np.testing.assert_allclose(mine, ref, rtol=0, atol=1e-6 * np.abs(ref).max())
        np.testing.assert_array_equal(cloud.cpu().numpy(), OE.voxel_down_sample(mine, 0.01))
    # the oracle's brute-force distance (nero_oracle_eval.nearest_dist) in float64, run with torch on the GPU for speed
    g32, p32 = gt.float().double(), pr.float().double()
    nn = lambda a, b: torch.cat([torch.cdist(a[i:i + 1024], b, compute_mode='donot_use_mm_for_euclid_dist').min(1)[0]
                                 for i in range(0, a.shape[0], 1024)]).cpu().numpy()
    oc = (nn(g32, p32).mean() + nn(p32, g32).mean()) / 2
    assert abs(c - oc) <= 1e-6 * oc
    # a second run gives the same bits
    c2, dg2, dp2 = E.chamfer_distance(E.gt_eval_points_cuda(root, ids, views).cpu().numpy().astype(np.float32),
                                      E.mesh_eval_points_cuda(verts, tris, views).cpu().numpy().astype(np.float32))
    assert c2 == c and np.array_equal(dg, dg2) and np.array_equal(dp, dp2)


def run_tool(ws, *args):
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get('PYTHONPATH', ''))
    out = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', args[0])] + list(args[1:]), cwd=str(ws), env=env,
                         capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    return out.stdout.strip().split('\n')[-1]


def test_eval_synthetic_shape_tool_writes_and_reuses_the_cache(workspace):
    cache = workspace / 'data' / 'GlossySynthetic' / 'ball' / 'eval_pts.ply'
    if cache.exists():
        cache.unlink()
    log = workspace / 'data' / 'geometry.log'
    if log.exists():
        log.unlink()
    a = run_tool(workspace, 'eval_synthetic_shape.py', '--object', 'ball', '--mesh', 'ball_pred.ply', '--batch_size', '7')
    head = cache.read_bytes().split(b'end_header\n')[0].decode()
    assert 'format binary_little_endian 1.0' in head and 'property double x' in head
    stamp = cache.stat().st_mtime_ns
    b = run_tool(workspace, 'eval_synthetic_shape.py', '--object', 'ball', '--mesh', 'ball_pred.ply')
    assert cache.stat().st_mtime_ns == stamp
    assert a == b and a.startswith('ball_pred ')
    assert log.read_text() == a + '\n' + b + '\n'
    assert abs(float(a.split()[1]) - DELTA) < 0.01


def test_eval_real_shape_tool_matches_oracle(workspace):
    rng = np.random.RandomState(3)
    p = rng.randn(3000, 3)
    g = rng.randn(2500, 3)
    E.write_points_ply(str(workspace / 'real_pr.ply'), p)
    write_ply(str(workspace / 'real_gt.ply'), g.astype(np.float32), np.zeros((0, 3), np.int64))
    line = run_tool(workspace, 'eval_real_shape.py', '--pr', 'real_pr.ply', '--gt', 'real_gt.ply')
    c = E.chamfer_distance(g.astype(np.float32), p)[0]
    oc = OE.chamfer(g.astype(np.float32), p.astype(np.float32))[0]
    assert abs(c - oc) <= 1e-6 * oc
    assert line == E.result_line('real_pr', c)
    assert (workspace / 'data' / 'geometry.log').read_text().endswith(line + '\n')
