"""GPU: mesh simplification (k_simplify.cu through nero_b200.simplify) against the numpy oracle, bit for bit, round by round
on small meshes and for the first round of a mesh with more than 2^24 valid edges; determinism; the input checks; the accuracy the feature is for (a simplified fine mesh against a coarse marching-cubes
mesh of the same size); and tools/extract_mesh.py --faces and tools/simplify_mesh.py end to end."""
import importlib.util
import io
import os
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mat as OM
import nero_oracle_simplify as OS
from helpers import build_params, load_golden
from test_simplify_host import blobs_mesh, cropped_mesh, sphere_mesh, target, torus_mesh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

MESHES = {'sphere32': lambda: sphere_mesh(32), 'torus48': lambda: torus_mesh(48), 'blobs': blobs_mesh, 'cropped': cropped_mesh}


@pytest.mark.parametrize('name', sorted(MESHES))
@pytest.mark.parametrize('frac', [0.1, 0.37])
def test_matches_the_oracle_round_by_round(name, frac):
    """0.37 gives an odd target that the last round reaches in the middle of its budget."""
    from nero_b200.simplify import simplify_cuda
    v, t = MESHES[name]()
    F = target(t.shape[0]) if frac == 0.1 else int(t.shape[0] * frac) | 1
    gtr, otr = [], []
    gv, gt, gst = simplify_cuda(v, t, F, trace=gtr)
    ov, ot, ost = OS.simplify(v, t, F, trace=otr)
    assert len(gtr) == len(otr) > 3
    for r, (g, o) in enumerate(zip(gtr, otr)):
        for k in ('tris', 'edges', 'key', 'selected', 'collapsed', 'x', 'cost'):
            assert np.array_equal(g[k], o[k]), f'round {r}: {k} differs from the oracle'
    np.testing.assert_array_equal(gt.cpu().numpy(), ot)
    np.testing.assert_array_equal(gv.cpu().numpy(), ov)
    assert gst == ost
    assert gst['triangles'] in (F, F + 1) if name != 'cropped' else gst['triangles'] >= F


def test_two_runs_give_the_same_bytes():
    from nero_b200.simplify import simplify_cuda
    v, t = torus_mesh(64)
    a = simplify_cuda(v, t, 3000)
    b = simplify_cuda(torch.from_numpy(v).cuda(), torch.from_numpy(t).cuda(), 3000)
    assert a[2] == b[2] and a[2]['triangles'] == 3000
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_rejections_match_the_oracle():
    from nero_b200.simplify import simplify_cuda
    v = np.random.RandomState(0).rand(6, 3).astype(np.float32)
    for t in ([[0, 1, 2], [0, 2, 6]], [[0, 1, 2], [3, 4, 3]], [[0, 1, 2], [1, 0, 3], [0, 1, 4], [2, 1, 5]],
              [[0, 1, 2], [2, 1, 3], [0, 1, 4]], [[0, 1, 2], [-1, 1, 3]]):
        t = np.asarray(t, np.int32)
        with pytest.raises(ValueError) as want:
            OS.simplify(v, t, 4)
        with pytest.raises(ValueError) as got:
            simplify_cuda(v, t, 4)
        assert str(got.value) == str(want.value)


def _analytic(kind, p):
    if kind == 'sphere':
        return np.abs(np.linalg.norm(p, axis=-1) - 0.6)
    return np.abs(np.hypot(np.hypot(p[:, 0], p[:, 1]) - 0.5, p[:, 2]) - 0.2)


def _mc(kind, res):
    from nero_b200.mesh import marching_cubes_cuda
    ax = torch.linspace(-1.0, 1.0, res, device='cuda', dtype=torch.float64)
    x, y, z = torch.meshgrid(ax, ax, ax, indexing='ij')
    u = torch.sqrt(x * x + y * y + z * z) - 0.6 if kind == 'sphere' else torch.hypot(torch.hypot(x, y) - 0.5, z) - 0.2
    v, t = marching_cubes_cuda(u.float(), 0.0)
    return v * (2.0 / (res - 1)) - 1.0, t


@pytest.mark.parametrize('kind', ['sphere', 'torus'])
def test_simplified_fine_mesh_is_closer_than_coarse_marching_cubes(kind):
    """The claim the feature rests on: 256^3 simplified to the size of the 64^3 mesh lies closer to the analytic surface."""
    from nero_b200.evaluate import sample_surface
    from nero_b200.simplify import simplify_cuda
    cv, ct = _mc(kind, 64)
    fv, ft = _mc(kind, 256)
    sv, st, stats = simplify_cuda(fv, ft, ct.shape[0])
    assert st.shape[0] == ct.shape[0]
    dc = _analytic(kind, sample_surface(cv, ct, 200000, seed=5).cpu().numpy())
    ds = _analytic(kind, sample_surface(sv, st, 200000, seed=5).cpu().numpy())
    print(f'{kind}: {ct.shape[0]} triangles; 64^3 mesh mean {dc.mean():.3e} max {dc.max():.3e}; 256^3 simplified '
          f'({ft.shape[0]} -> {st.shape[0]}, {stats["rounds"]} rounds) mean {ds.mean():.3e} max {ds.max():.3e}')
    assert ds.mean() <= dc.mean()


def _field_net():
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden('shape_materials_field')
    cfg = {'n_samples': 32, 'n_importance': 32}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(cfg, int(g['seed']), int(g['pseed'])))
    return net.cuda()


def _tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    return tool


def test_extract_mesh_faces_feeds_stage_two(tmp_path, monkeypatch):
    import yaml
    from nero_b200.material import NeROMaterialRenderer, read_ply
    net = _field_net()
    name = 'field_shape'
    os.makedirs(tmp_path / 'data' / 'model' / name)
    torch.save({'step': 77, 'network_state_dict': {k: v.cpu() for k, v in net.state_dict().items()}},
               str(tmp_path / 'data' / 'model' / name / 'model.pth'))
    cfg_path = tmp_path / 'shape.yaml'
    cfg_path.write_text(yaml.safe_dump({'name': name, 'network': 'shape', 'n_samples': 32, 'n_importance': 32}))
    monkeypatch.chdir(tmp_path)
    tool = _tool('extract_mesh')
    full = tool.main(['--cfg', str(cfg_path), '--resolution', '96', '--sparse'])
    fv, ft = read_ply(full)
    faces = 2 * (ft.shape[0] // 8)
    path = tool.main(['--cfg', str(cfg_path), '--resolution', '96', '--sparse', '--faces', str(faces)])
    assert path == full == os.path.join('data', 'meshes', f'{name}-77.ply')
    verts, tris = read_ply(path)
    assert tris.shape[0] == faces
    sv, st, _ = OS.simplify(fv, ft, faces)
    np.testing.assert_array_equal(np.asarray(tris), st)
    np.testing.assert_array_equal(np.asarray(verts, np.float32), sv)

    mat = NeROMaterialRenderer({'mesh': path, 'shader_cfg': {'human_lights': False}}, is_train=False).cuda()
    mv, mt = mat._mesh
    rays = O.synthetic_rays(4000, seed=11)
    _, _, depth, hit = mat.trace(rays['rays_o'].cuda(), rays['rays_d'].cuda())
    _, _, bdepth = OM.trace_bruteforce(mv, mt, rays['rays_o'].double(), rays['rays_d'].double(), chunk=256)
    bhit = (bdepth < OM.MISS_DEPTH).numpy()
    got = hit.reshape(-1).cpu().numpy()
    assert bhit.sum() > 500 and (got == bhit).mean() > 0.9995
    both = got & bhit
    np.testing.assert_allclose(depth.reshape(-1).cpu().numpy()[both], bdepth.numpy()[both], rtol=0, atol=1e-4)

    out = str(tmp_path / 'small.ply')
    buf = io.StringIO()
    with redirect_stdout(buf):
        _tool('simplify_mesh').main(['--mesh', path, '--out', out, '--faces', str(faces // 2)])
    assert 'rounds' in buf.getvalue()
    rv, rt = read_ply(out)
    ov, ot, _ = OS.simplify(np.asarray(verts, np.float32), np.asarray(tris, np.int32), faces // 2)
    np.testing.assert_array_equal(np.asarray(rt), ot)
    np.testing.assert_array_equal(np.asarray(rv, np.float32), ov)


def torus_grid(n=2400, R=0.5, r=0.2):
    """A closed n x n quad grid on a torus, two triangles per quad: 2 n^2 triangles and 3 n^2 edges."""
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    th, ph = 2 * np.pi * i / n, 2 * np.pi * j / n
    v = np.stack([(R + r * np.cos(ph)) * np.cos(th), (R + r * np.cos(ph)) * np.sin(th), r * np.sin(ph)], -1)
    v00, v10, v01, v11 = i * n + j, (i + 1) % n * n + j, i * n + (j + 1) % n, (i + 1) % n * n + (j + 1) % n
    t = np.concatenate([np.stack([v00, v10, v11], -1).reshape(-1, 3), np.stack([v00, v11, v01], -1).reshape(-1, 3)])
    return v.reshape(-1, 3).astype(np.float32), t.astype(np.int32)


def test_first_round_matches_the_oracle_above_2_24_valid_edges():
    """The size the 2048^3 meshes reach: 17.3 M edges, more than 2^24 of them valid, and a budget above the quarter guard,
    so the guard's rank decides which edges collapse.  Round 1 (placements, costs, keys, selected and collapsed sets) equals
    the oracle's."""
    from nero_b200.simplify import simplify_cuda
    v, t = torus_grid()
    T = t.shape[0]
    lock, pos, Q = OS.prepare(v, t)
    o = OS.one_round(pos, Q, t.astype(np.int64), lock, T)
    n1 = int(o['collapsed'].sum())
    assert int((o['key'] != OS.KEY_INF).sum()) > 2 ** 24 and n1 > 0
    trace = []
    _, _, st = simplify_cuda(v, t, T - 2 * (n1 + 10), trace=trace)       # round 1's budget n1 + 10: the guard binds
    g = trace[0]
    for k in ('tris', 'edges', 'key', 'selected', 'collapsed', 'x', 'cost'):
        assert np.array_equal(g[k], o[k]), f'round 1: {k} differs from the oracle'
    assert st['collapses'][0] == n1
