"""GPU: mesh clean-up and surface sampling (k_meshpts.cu through nero_b200.evaluate) against the numpy oracle, bit for bit:
triangle areas, crop, component labels and areas, the kept sets, the compacted mesh and the sampled points; determinism,
independence from chunking, the accuracy of points on a marching-cubes sphere, and tools/sample_mesh_points.py end to end."""
import importlib.util
import io
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import nero_oracle_meshpts as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def blobs_mesh(res=48):
    """Marching cubes (GPU) of a field with four separate blobs of different sizes, in world coordinates."""
    from nero_b200.mesh import marching_cubes
    ax = np.linspace(-1.0, 1.0, res)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    cs = np.asarray([[-0.45, -0.4, -0.3], [0.45, 0.4, 0.3], [0.5, -0.5, 0.4], [-0.5, 0.5, -0.5]])
    rs = np.asarray([0.4, 0.3, 0.18, 0.1])
    u = np.min(np.linalg.norm(x[..., None, :] - cs, axis=-1) - rs, -1).astype(np.float32)
    v, t = marching_cubes(u, 0.0)
    return (v * (2.0 / (res - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def sphere_mesh(res=64, r=0.6):
    from nero_b200.mesh import marching_cubes
    ax = np.linspace(-1.0, 1.0, res)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    v, t = marching_cubes((np.linalg.norm(x, axis=-1) - r).astype(np.float32), 0.0)
    return (v * (2.0 / (res - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def messy_mesh(seed=8):
    """Random triangles over a vertex set with unreferenced vertices and degenerate triangles."""
    rng = np.random.RandomState(seed)
    v = rng.rand(3000, 3).astype(np.float32)
    t = rng.randint(0, 2000, (2500, 3)).astype(np.int32)       # vertices 2000.. are never used
    t[::5, 2] = t[::5, 1]
    t[1::7] = t[1::7, :1]
    return v, t


MESHES = {'floaters': O.floater_scene, 'blobs': blobs_mesh, 'messy': messy_mesh}
REGIONS = [dict(), dict(min_component=0.5), dict(sphere=(0.0, 0.0, 0.0, 1.0), min_component=0.1),
           dict(box=(-0.6, -0.7, -0.8, 0.9, 0.8, 0.7), min_component=0.02), dict(sphere=(0.1, 0.0, 0.0, 0.75), box=(-1, -1, -1, 1, 0.5, 1))]


def check_clean(v, t, **kw):
    from nero_b200 import evaluate as E
    cv, ct, info = E.clean_mesh_cuda(v, t, **kw)
    r = O.clean(v, t, **kw)
    np.testing.assert_array_equal(info['area'].cpu().numpy(), r['area'])
    np.testing.assert_array_equal(info['keep'].cpu().numpy().astype(bool), r['keep'])
    np.testing.assert_array_equal(info['label'].cpu().numpy(), r['label'])
    np.testing.assert_array_equal(info['comp_label'].cpu().numpy(), r['comp_label'])
    np.testing.assert_array_equal(info['comp_area'].cpu().numpy(), r['comp_area'])
    np.testing.assert_array_equal(info['comp_keep'].cpu().numpy(), r['comp_keep'])
    np.testing.assert_array_equal(ct.cpu().numpy(), r['tris'])
    np.testing.assert_array_equal(cv.cpu().numpy(), r['verts'])
    assert info['kept_triangles'] == r['tris'].shape[0] and info['kept_vertices'] == r['verts'].shape[0]
    return cv, ct, info, r


@pytest.mark.parametrize('name', sorted(MESHES))
@pytest.mark.parametrize('region', range(len(REGIONS)))
def test_clean_mesh_matches_the_oracle(name, region):
    v, t = MESHES[name]()
    check_clean(v, t, **REGIONS[region])


def test_floater_is_dropped():
    v, t = O.floater_scene()
    _, ct, info, _ = check_clean(v, t, min_component=0.5)
    assert info['components'] == 4 and info['kept_components'] == 1
    _, _, info, _ = check_clean(v, t, sphere=(0, 0, 0, 1.0))
    assert info['components'] == 3 and info['kept_components'] == 3


def test_long_reversed_strip_is_one_component():
    v, t = O.reversed_strip(1_000_000)
    _, ct, info, _ = check_clean(v, t)
    assert info['components'] == 1 and bool((info['label'] == 0).all())
    _, _, info, _ = check_clean(v, t, box=(-1, -1, -1, 2500, 1, 1))      # the first half of the strip along x
    assert info['components'] == 1 and 0 < info['kept_triangles'] < t.shape[0]


@pytest.mark.parametrize('n', [1, 1023, 1024, 1025, 500_000])
def test_samples_match_the_oracle(n):
    from nero_b200 import evaluate as E
    for v, t in (O.floater_scene(), blobs_mesh()):
        p = E.sample_surface(v, t, n, seed=17).cpu().numpy()
        q, _ = O.sample(v, t, n, seed=17)
        np.testing.assert_array_equal(p, q)


def test_samples_of_meshes_with_degenerate_triangles_match_the_oracle():
    from nero_b200 import evaluate as E
    v, t = messy_mesh()
    p = E.sample_surface(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda(), 100_000, seed=3).cpu().numpy()
    q, tri = O.sample(v, t, 100_000, seed=3)
    np.testing.assert_array_equal(p, q)
    assert (O.areas(v, t)[tri] > 0).all()


def test_samples_do_not_depend_on_chunking_or_the_run():
    from nero_b200 import evaluate as E
    v, t = blobs_mesh()
    full = E.sample_surface(v, t, 50_000, seed=9)
    again = E.sample_surface(v, t, 50_000, seed=9)
    assert torch.equal(full, again)
    parts = [E.sample_surface(v, t, n, seed=9, first=i0) for i0, n in ((0, 1), (1, 1023), (1024, 1025), (2049, 47_951))]
    assert torch.equal(torch.cat(parts), full)
    assert not torch.equal(E.sample_surface(v, t, 50_000, seed=10), full)


def test_sphere_samples_lie_within_the_chord_error():
    from nero_b200 import evaluate as E
    r = 0.6
    v, t = sphere_mesh(r=r)
    p = E.sample_surface(v, t, 500_000, seed=1).cpu().numpy()
    vd = v.astype(np.float64)
    err_v = np.abs(np.linalg.norm(vd, axis=1) - r).max()
    e = vd[t[:, [1, 2, 0]]] - vd[t]
    lmax = np.linalg.norm(e, axis=-1).max()
    d = np.abs(np.linalg.norm(p, axis=1) - r)
    assert d.max() <= err_v + lmax * lmax / (4 * r), (d.max(), err_v, lmax)
    # area-uniform: the octant counts are balanced
    oct_ = (p[:, 0] > 0) * 4 + (p[:, 1] > 0) * 2 + (p[:, 2] > 0)
    c = np.bincount(oct_, minlength=8)
    assert np.abs(c - 500_000 / 8).max() < 5 * np.sqrt(500_000 / 8)


def test_empty_or_arealess_meshes_are_errors():
    from nero_b200 import evaluate as E
    v = np.asarray([[0, 0, 0], [1, 0, 0], [2, 0, 0]], np.float32)
    with pytest.raises(ValueError):
        E.sample_surface(v, np.asarray([[0, 1, 2]], np.int32), 10)
    vv, tt = O.floater_scene()
    with pytest.raises(ValueError):
        E.clean_mesh(vv, tt, sphere=(10.0, 10.0, 10.0, 0.1))


def _load(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', name + '.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tool_end_to_end(tmp_path, monkeypatch):
    import nero_oracle_eval as OE
    from nero_b200 import evaluate as E
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    tool = _load('sample_mesh_points')
    # sphere + floater: --min-component 0.5 drops the floater
    v, t = O.floater_scene()
    mesh, out, kept = tmp_path / 'scene.ply', tmp_path / 'scene-pts.ply', tmp_path / 'scene-kept.ply'
    write_ply(str(mesh), v, t)
    tool.main(['--mesh', str(mesh), '--out', str(out), '--num', '4096', '--seed', '5', '--min-component', '0.5',
               '--mesh-out', str(kept)])
    r = O.clean(v, t, min_component=0.5)
    kv, kt = read_ply(str(kept))
    np.testing.assert_array_equal(kv, r['verts'])
    np.testing.assert_array_equal(kt, r['tris'])
    pts = E.read_points_ply(str(out))
    np.testing.assert_array_equal(pts, O.sample(r['verts'], r['tris'], 4096, seed=5)[0])
    np.testing.assert_array_equal(pts, E.sample_surface(r['verts'], r['tris'], 4096, seed=5).cpu().numpy())
    # a marching-cubes sphere sampled by the tool, scored against analytic sphere points by eval_real_shape.py
    sv, st = sphere_mesh(res=40)
    smesh, spts, gt = tmp_path / 'sphere.ply', tmp_path / 'sphere-nero.ply', tmp_path / 'sphere-gt.ply'
    write_ply(str(smesh), sv, st)
    tool.main(['--mesh', str(smesh), '--out', str(spts), '--num', '3000'])
    k = np.arange(3000) + 0.5
    phi, z = k * np.pi * (3.0 - np.sqrt(5.0)), 1.0 - 2.0 * k / 3000
    g = 0.6 * np.stack([np.sqrt(1 - z * z) * np.cos(phi), np.sqrt(1 - z * z) * np.sin(phi), z], 1)
    E.write_points_ply(str(gt), g)
    monkeypatch.chdir(tmp_path)
    os.makedirs('data', exist_ok=True)
    buf = io.StringIO()
    with redirect_stdout(buf):
        _load('eval_real_shape').main(['--pr', str(spts), '--gt', str(gt)])
    stem, value = buf.getvalue().split()
    oc = OE.chamfer(E.read_points_ply(str(gt)).astype(np.float32), E.read_points_ply(str(spts)).astype(np.float32))[0]
    assert stem == 'sphere-nero' and abs(float(value) - oc) <= 6e-6, (value, oc)
