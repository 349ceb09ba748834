"""GPU: marching cubes (k_mcubes.cu through nero_b200.mesh) equals the numpy oracle exactly in connectivity and order,
NeROShapeRenderer.extract_mesh equals the oracle on extract_fields, and tools/extract_mesh.py feeds stage II."""
import os

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mat as OM
import nero_oracle_mesh as OMesh
from helpers import load_golden, build_params
from test_mcubes_host import smooth_field, assert_closed_and_oriented

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def check_against_oracle(u, iso=0.0):
    from nero_b200.mesh import marching_cubes
    v, t = marching_cubes(u, iso)
    ov, ot = OMesh.marching_cubes(u, iso)
    assert v.dtype == np.float64 and t.dtype == np.int64
    assert v.shape == ov.shape and t.shape == ot.shape, (v.shape, ov.shape, t.shape, ot.shape)
    np.testing.assert_array_equal(t, ot)
    if v.size:
        assert np.abs(v - ov).max() <= 1e-5
    return v, t


@pytest.mark.parametrize('shape,seed', [((24, 24, 24), 1), ((33, 40, 29), 2), ((17, 23, 31), 3)])
def test_random_fields_match_oracle(shape, seed):
    u = smooth_field(shape, seed)
    v, t = check_against_oracle(u)
    assert t.shape[0] > 100
    # an unstructured field too: many components, every case occurs
    rng = np.random.RandomState(seed)
    check_against_oracle(rng.randn(*shape).astype(np.float32), 0.1)


def test_nonzero_isovalue():
    u = smooth_field((30, 30, 30), 4, amp=0.6)
    for iso in (0.13, -0.05, 0.4):
        check_against_oracle(u, iso)


def test_exact_ties():
    rng = np.random.RandomState(5)
    u = rng.randint(-2, 3, size=(19, 21, 20)).astype(np.float32)
    for iso in (0.0, 1.0, -2.0):
        check_against_oracle(u, iso)


def test_empty_outputs():
    for u in (np.ones((9, 10, 11), np.float32), -np.ones((9, 10, 11), np.float32), np.zeros((5, 5, 5), np.float32)):
        v, t = check_against_oracle(u)
        assert v.shape == (0, 3) and t.shape == (0, 3)


def test_every_case_of_a_single_cube():
    """The smallest volume, 2x2x2, in all 256 corner patterns."""
    for case in range(256):
        u = np.ones((2, 2, 2), np.float32)
        for c in range(8):
            if case >> c & 1:
                u[c & 1, c >> 1 & 1, c >> 2 & 1] = -1.0 - 0.1 * c
        check_against_oracle(u)


def test_large_volume_multi_level_scan():
    """200^3: 8 M points, 7813 blocks, so the block-total scan runs over 8 chunks with a carried sum."""
    u = smooth_field((200, 200, 200), 6, amp=0.5, k=10)
    v, t = check_against_oracle(u)
    assert t.shape[0] > 100000


def test_deterministic_and_input_kinds():
    from nero_b200.mesh import marching_cubes, marching_cubes_cuda
    u = smooth_field((96, 80, 90), 8, amp=0.6)
    ud = torch.from_numpy(u).cuda()
    v1, t1 = marching_cubes_cuda(ud, 0.0)
    v2, t2 = marching_cubes_cuda(ud, 0.0)
    assert torch.equal(v1, v2) and torch.equal(t1, t2), 'two calls differ'
    a = marching_cubes(u, 0.0)
    b = marching_cubes(ud, 0.0)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])
    np.testing.assert_array_equal(a[0], v1.cpu().numpy().astype(np.float64))


def test_bad_shapes_raise():
    from nero_b200.mesh import marching_cubes
    for shape in ((8, 8), (1, 8, 8), (8, 8, 1), (2, 2, 2, 2)):
        with pytest.raises(ValueError):
            marching_cubes(torch.zeros(shape, device='cuda'), 0.0)


def _field_net():
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden('shape_materials_field')
    cfg = {'n_samples': 32, 'n_importance': 32}
    sd = build_params(cfg, int(g['seed']), int(g['pseed']))
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(sd)
    return net.cuda(), sd


def test_extract_fields_unchanged_by_slabs():
    """extract_fields fills the grid in x-slabs; the values equal one query of the whole grid, bit for bit."""
    net, _ = _field_net()
    res = 40
    axes = [torch.linspace(-1.0, 1.0, res, device='cuda') for _ in range(3)]
    pts = torch.stack(torch.meshgrid(*axes, indexing='ij'), -1).reshape(-1, 3)
    with torch.no_grad():
        val = net.engine.sdf_query(pts)[:, 0]
    val = torch.where(torch.norm(pts, dim=-1) >= 1.0, torch.full_like(val, 1.0), val)
    want = val.reshape(res, res, res).cpu().numpy()
    net.GRID_SLAB_POINTS = 3 * res * res          # 3-plane slabs, ragged last slab
    np.testing.assert_array_equal(net.extract_fields(resolution=res), want)
    del net.GRID_SLAB_POINTS
    np.testing.assert_array_equal(net.extract_fields(resolution=res), want)


@pytest.mark.parametrize('res', [64, 128])
def test_extract_mesh_matches_oracle_and_faces_inward(res):
    net, sd = _field_net()
    v, t = net.extract_mesh(resolution=res)
    u = net.extract_fields(resolution=res)
    ov, ot = OMesh.marching_cubes(u, 0.0)
    np.testing.assert_array_equal(t, ot)
    assert np.abs(v - (ov / (res - 1.0) * 2.0 - 1.0)).max() <= 1e-6
    assert t.shape[0] > 1000
    assert_closed_and_oriented(t, v.shape[0])
    # face normals point against the SDF gradient (into the solid), on a sample of faces of non-negligible area
    p0, p1, p2 = v[t[:, 0]], v[t[:, 1]], v[t[:, 2]]
    n = np.cross(p1 - p0, p2 - p0)
    area = np.linalg.norm(n, axis=-1)
    h = 2.0 / (res - 1)
    keep = np.nonzero(area > 1e-3 * h * h)[0]
    keep = np.random.RandomState(0).choice(keep, min(4000, keep.shape[0]), replace=False)
    x = torch.from_numpy((p0 + p1 + p2)[keep] / 3.0).float().requires_grad_(True)
    sdf = O.sdf_forward(sd, x)[:, 0]
    grad, = torch.autograd.grad(sdf.sum(), x)
    dots = (n[keep] * grad.double().numpy()).sum(-1)
    assert (dots < 0).mean() >= 0.999, (dots >= 0).sum()


def test_extract_mesh_tool_feeds_stage_two(tmp_path, monkeypatch):
    import importlib.util
    import yaml
    from nero_b200.material import NeROMaterialRenderer
    net, sd = _field_net()
    name = 'field_shape'
    os.makedirs(tmp_path / 'data' / 'model' / name)
    torch.save({'step': 1234, 'network_state_dict': {k: v.cpu() for k, v in net.state_dict().items()}},
               str(tmp_path / 'data' / 'model' / name / 'model.pth'))
    cfg_path = tmp_path / 'shape.yaml'
    cfg_path.write_text(yaml.safe_dump({'name': name, 'network': 'shape', 'n_samples': 32, 'n_importance': 32}))
    spec = importlib.util.spec_from_file_location('extract_mesh_tool', os.path.join(ROOT, 'tools', 'extract_mesh.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    monkeypatch.chdir(tmp_path)
    path = tool.main(['--cfg', str(cfg_path), '--resolution', '64'])
    assert path == os.path.join('data', 'meshes', f'{name}-1234.ply') and os.path.exists(path)

    mat = NeROMaterialRenderer({'mesh': path, 'shader_cfg': {'human_lights': False}}, is_train=False).cuda()
    verts, tris = mat._mesh
    rays = O.synthetic_rays(4000, seed=11)
    inters, normals, depth, hit = mat.trace(rays['rays_o'].cuda(), rays['rays_d'].cuda())
    _, _, bdepth = OM.trace_bruteforce(verts, tris, rays['rays_o'].double(), rays['rays_d'].double(), chunk=256)
    bhit = (bdepth < OM.MISS_DEPTH).numpy()
    got = hit.reshape(-1).cpu().numpy()
    assert bhit.sum() > 500
    assert (got == bhit).mean() > 0.9995, (got != bhit).sum()
    both = got & bhit
    np.testing.assert_allclose(depth.reshape(-1).cpu().numpy()[both], bdepth.numpy()[both], rtol=0, atol=1e-4)
    facing = (normals.reshape(-1, 3).cpu() * rays['rays_d']).sum(-1).numpy()[got]
    assert (facing < 0).mean() >= 0.999, (facing >= 0).sum()
