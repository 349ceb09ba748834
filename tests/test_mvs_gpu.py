"""Dense multi-view stereo on the GPU: every kernel of k_mvs.cu against oracle/nero_oracle_mvs.py bit for bit, run-to-run
identity, accuracy on the synthetic table / box / sphere project, and tools/dense_points.py feeding
tools/prepare_custom_object.py end to end."""
import importlib.util
import os

import numpy as np
import pytest
import torch

import nero_oracle_mvs as OM
from nero_b200 import mvs
from nero_b200 import objprep as OP
from nero_b200.evaluate import depth_to_points_cuda, read_points_ply

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _run(root, **kw):
    views, pts, tracks = OP.read_colmap_model(os.path.join(root, 'sparse', '0'), tracks=True)
    return mvs.reconstruct(views, pts, tracks, mvs.image_reader(os.path.join(root, 'images')), **kw)


@pytest.fixture(scope='module')
def tiny(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('mvs_tiny'))
    pr = OM.project(root, 3, 48, 32, per_view=40)
    trace = {}
    cloud, info = _run(root, radius=2, step=1, iterations=2, trace=trace)
    return root, pr, cloud, info, trace


def test_kernels_match_oracle_bit_for_bit(tiny):
    root, pr, cloud, info, trace = tiny
    assert info['views_used'] == 3
    greys = [OM.grey(mvs.read_rgb(os.path.join(root, 'images', n)), 1) for n in info['names']]
    for g, og in zip(info['greys'], greys):
        assert np.array_equal(g.cpu().numpy(), og)
    for i, e in enumerate(info['plan']):
        src = e['sources']
        geo = mvs.pm_table(info['Ks'][i], info['poses'][i], [info['Ks'][j] for j in src], [info['poses'][j] for j in src])
        stats = OM.ref_stats(greys[i], 2, 1)
        assert np.array_equal(mvs.ref_stats(info['greys'][i], 2, 1).cpu().numpy(), stats)
        v = OM.View(greys[i], mvs.kinv32(info['Ks'][i]), stats, [greys[j] for j in src], geo, np.float32(e['range'][0]),
                    np.float32(e['range'][1]), 2, 1, mvs.SEED, i)
        states = OM.patchmatch(v, 2)
        assert len(trace[i]) == len(states) == 5
        for k, ((p, c), (op, oc)) in enumerate(zip(trace[i], states)):
            assert np.array_equal(p.cpu().numpy(), op), f'view {i}: hypotheses differ after step {k}'
            assert np.array_equal(c.cpu().numpy(), oc), f'view {i}: costs differ after step {k}'
    planes = [p.cpu().numpy() for p in info['planes']]
    costs = [c.cpu().numpy() for c in info['cost']]
    pts = []
    for i, e in enumerate(info['plan']):
        src = e['sources']
        geo = mvs.filter_table(info['poses'][i], [info['Ks'][j] for j in src], [info['poses'][j] for j in src])
        od, oc = OM.geometric_filter(info['Ks'][i], planes[i], costs[i], [(planes[j], costs[j]) for j in src], geo, mvs.MAX_COST,
                                     mvs.REPROJ ** 2, mvs.REL_DEPTH, np.cos(np.radians(mvs.NORMAL_DEG)), mvs.MIN_CONSISTENT)
        assert np.array_equal(info['count'][i].cpu().numpy(), oc) and np.array_equal(info['depth'][i].cpu().numpy(), od)
        pts.append(OM.unproject(od, info['Ks'][i], info['poses'][i]))
    ref = np.concatenate(pts, 0)
    out = cloud.cpu().numpy()
    assert out.shape == ref.shape and np.allclose(out, ref, rtol=0, atol=1e-5)
    # at 48 x 32 after 2 iterations the default thresholds keep few pixels or none: loose ones exercise every branch of the
    # filter and give fused points to compare
    fused, ofused = [], []
    for i, e in enumerate(info['plan']):
        src = e['sources']
        loose = (2.0, 3.0, 0.1, 0.5, 1)
        d, cnt = mvs.geometric_filter(info['Ks'][i], info['poses'][i], info['planes'][i], info['cost'][i],
                                      [(info['Ks'][j], info['poses'][j], info['planes'][j], info['cost'][j]) for j in src],
                                      loose[0], loose[1], loose[2], np.degrees(np.arccos(loose[3])), loose[4])
        geo = mvs.filter_table(info['poses'][i], [info['Ks'][j] for j in src], [info['poses'][j] for j in src])
        od, oc = OM.geometric_filter(info['Ks'][i], planes[i], costs[i], [(planes[j], costs[j]) for j in src], geo, loose[0],
                                     loose[1] ** 2, loose[2], float(np.cos(np.radians(np.degrees(np.arccos(loose[3]))))), loose[4])
        assert np.array_equal(cnt.cpu().numpy(), oc) and np.array_equal(d.cpu().numpy(), od)
        fused.append(depth_to_points_cuda(d, info['poses'][i].astype(np.float64), mvs.centre_K(info['Ks'][i])).cpu().numpy())
        ofused.append(OM.unproject(od, info['Ks'][i], info['poses'][i]))
    fused, ofused = np.concatenate(fused, 0), np.concatenate(ofused, 0)
    assert fused.shape == ofused.shape and fused.shape[0] > 100
    assert np.allclose(fused, ofused, rtol=0, atol=1e-5)       # fp64 unprojection, fp32 output of depth_to_points_cuda


def test_two_runs_identical(tiny):
    root, _, cloud, _, _ = tiny
    again, _ = _run(root, radius=2, step=1, iterations=2)
    assert torch.equal(cloud, again)


@pytest.fixture(scope='module')
def scene12(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('mvs_scene'))
    pr = OM.project(root, 12, 320, 240, seed=3)
    cloud, info = _run(root)
    return root, pr, cloud, info


def test_accuracy_on_the_synthetic_scene(scene12):
    root, pr, cloud, info = scene12
    kept = good = seen = seen_kept = 0
    for i, tr in enumerate(pr['truth']):
        if info['depth'][i] is None:
            continue
        d = info['depth'][i].cpu().numpy().astype(np.float64)
        td = tr['depth']
        k = (d > 0) & (td > 0)
        kept += int((d > 0).sum())
        good += int((np.abs(d[k] - td[k]) <= 0.01 * td[k]).sum())
        obj = tr['surface'] >= 1
        seen += int(obj.sum())
        seen_kept += int((obj & (d > 0)).sum())
    _, D, _, _ = OP.scene_scale(OP.read_colmap_model(os.path.join(root, 'sparse', '0'))[0])
    dist = OM.surface_distance(cloud.cpu().numpy())
    frac_depth, frac_pts, frac_obj = good / kept, float((dist <= 0.005 * D).mean()), seen_kept / seen
    print(f'views {info["views_used"]}, kept {kept}, within 1 % depth {frac_depth:.4f}, within 0.005 D {frac_pts:.4f}, '
          f'object pixels kept {frac_obj:.4f}')
    assert info['views_used'] == 12
    # measured on an H100: 98.47 % within 1 % of the true depth, 99.09 % of the points within 0.005 D of the surface, 59.9 %
    # of the object's pixels kept
    assert frac_depth >= 0.95 and frac_pts >= 0.95 and frac_obj >= 0.5


def test_dense_points_then_prepare_custom_object(scene12, capsys):
    root, pr, _, _ = scene12
    tool('dense_points').main(['--root', root])
    assert os.path.isfile(os.path.join(root, 'points.ply'))
    # the sphere touches the box top in one point, hidden from every camera, so box and sphere are two voxel components:
    # keep every component with at least a tenth of the largest one's points
    tool('prepare_custom_object').main(['--root', root, '--min-component', '0.1'])
    up = np.loadtxt(os.path.join(root, 'meta_info.txt'))[0]
    ang = np.degrees(np.arccos(np.clip(up @ pr['up'] / np.linalg.norm(up), -1, 1)))
    obj = read_points_ply(os.path.join(root, 'object_point_cloud.ply'))
    _, D, _, _ = OP.scene_scale(OP.read_colmap_model(os.path.join(root, 'sparse', '0'))[0])
    voxel = OP.VOXEL_FRAC * D
    lo, hi = OM.object_bbox()
    err = max(np.abs(obj.min(0) - lo).max(), np.abs(obj.max(0) - hi).max())
    print(capsys.readouterr().out)
    print(f'up error {ang:.4f} deg, bounding-box error {err:.4f} = {err / voxel:.2f} voxels, {obj.shape[0]} object points')
    assert ang <= 1.0 and err <= 2 * voxel        # measured on an H100: 0.0009 deg, 0.79 voxels
