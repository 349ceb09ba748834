"""GPU: brick-wise marching cubes (k_mcsparse.cu through nero_b200.mesh.extract_sparse) equals the numpy oracle and the dense
kernels on the dense field exactly; NeROShapeRenderer.extract_mesh_sparse equals extract_mesh exactly; the tool's --sparse
PLY equals the dense tool's; a 1024^3 extraction stays below the memory of the dense field."""
import os

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mcsparse as OS
from nero_b200 import params as P
from helpers import load_golden, build_params
from test_mcubes_host import assert_closed_and_oriented
from test_mcsparse_host import CASES, TABLES, grid_axes, steep

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def on_gpu(field):
    return lambda pts: torch.from_numpy(np.asarray(field(pts.cpu().numpy()), np.float32)).cuda()


def run_case(field, axes, iso, brick, lipschitz=2.0, outside=None):
    from nero_b200.mesh import extract_sparse, marching_cubes_cuda
    v, t, stats = extract_sparse(on_gpu(field), [torch.from_numpy(a).cuda() for a in axes], iso, brick=brick, lipschitz=lipschitz,
                                 outside=outside)
    assert v.dtype == torch.float32 and t.dtype == torch.int32 and v.is_cuda and t.is_cuda
    ov, ot, ostats = OS.extract_sparse(field, axes, iso, brick, lipschitz, outside, dtype=np.float32, tables=TABLES)
    np.testing.assert_array_equal(t.cpu().numpy(), ot)
    np.testing.assert_array_equal(v.cpu().numpy(), ov)
    assert stats == ostats
    dv, dt = marching_cubes_cuda(torch.from_numpy(OS.dense_field(field, axes, outside)).cuda(), iso)
    assert torch.equal(v, dv) and torch.equal(t, dt), 'the sparse mesh differs from the dense kernels on the dense field'
    return v, t, stats


@pytest.mark.parametrize('brick', [4, 8, 16])
@pytest.mark.parametrize('case', sorted(CASES))
def test_analytic_fields_match_oracle_and_dense_kernels(case, brick):
    field, n, iso, outside = CASES[case]
    v, t, stats = run_case(field, grid_axes(n), iso, brick, outside=outside)
    assert t.shape[0] > 500


def test_growth_terminates_and_matches_the_oracle_rounds():
    v, t, stats = run_case(steep, grid_axes(65), 0.0, 8, lipschitz=1.0)
    assert stats['grow_rounds'] >= 1 and stats['bricks_added'] > 0


def test_empty_field():
    from nero_b200.mesh import extract_sparse
    axes = [torch.linspace(-1.0, 1.0, 33, device='cuda') for _ in range(3)]
    for value in (1.0, 0.01):
        v, t, stats = extract_sparse(lambda p: torch.full((p.shape[0],), value, device='cuda'), axes, 0.0)
        assert v.shape == (0, 3) and t.shape == (0, 3) and stats['triangles'] == 0
    with pytest.raises(ValueError):
        extract_sparse(lambda p: torch.zeros(p.shape[0], 1, device='cuda'), axes, 0.0)


def _field_net():
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden('shape_materials_field')
    cfg = {'n_samples': 32, 'n_importance': 32}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(cfg, int(g['seed']), int(g['pseed'])))
    return net.cuda()


@pytest.fixture(scope='module')
def field_net():
    return _field_net()


@pytest.mark.parametrize('bounds', [(-1.0, 1.0), ((-0.9, -1.0, -0.8), (1.0, 0.85, 0.9))])
@pytest.mark.parametrize('res,brick', [(128, 4), (128, 8), (256, 8), (256, 4)])
def test_extract_mesh_sparse_equals_extract_mesh(field_net, res, brick, bounds):
    v, t = field_net.extract_mesh(resolution=res, bound_min=bounds[0], bound_max=bounds[1])
    sv, st, stats = field_net.extract_mesh_sparse(resolution=res, bound_min=bounds[0], bound_max=bounds[1], brick=brick,
                                                  return_stats=True)
    assert sv.dtype == np.float64 and st.dtype == np.int64 and t.shape[0] > 1000
    np.testing.assert_array_equal(st, t)
    np.testing.assert_array_equal(sv, v)
    if res == 256:
        assert stats['points_evaluated'] < res ** 3
        assert_closed_and_oriented(st, sv.shape[0])


def test_deterministic(field_net):
    a = field_net.extract_mesh_sparse(resolution=128)
    b = field_net.extract_mesh_sparse(resolution=128)
    np.testing.assert_array_equal(a[0], b[0])
    np.testing.assert_array_equal(a[1], b[1])


def test_tool_sparse_ply_equals_dense_ply(tmp_path, monkeypatch, capsys):
    import importlib.util
    import yaml
    from nero_b200.material import read_ply
    net = _field_net()
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
    path = tool.main(['--cfg', str(cfg_path), '--resolution', '96'])
    dense = read_ply(path)
    assert 'sparse:' not in capsys.readouterr().out
    os.remove(path)
    assert tool.main(['--cfg', str(cfg_path), '--resolution', '96', '--sparse', '--brick', '4', '--lipschitz', '3']) == path
    out = capsys.readouterr().out
    assert 'sparse: coarse_points 15625' in out and 'grow_rounds' in out
    sparse = read_ply(path)
    assert dense[1].shape[0] > 1000
    np.testing.assert_array_equal(sparse[0], dense[0])
    np.testing.assert_array_equal(sparse[1], dense[1])


def test_1024_cubed_stays_below_the_dense_field():
    """The perturbed bell parameters at 1024^3: the dense field alone would take 4.3 GB.  Linear indices of the far corner
    exceed int32 by a factor of 1.5 as edge keys (3 * 1024^3), so a closed mesh here also shows the keys are 64-bit."""
    from nero_b200.renderer import NeROShapeRenderer
    cfg = {}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(O.perturb_params(P.build_shape_state_dict(cfg, seed=6033)))
    net = net.cuda()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    before = torch.cuda.memory_allocated()                  # whatever earlier tests of the process still hold
    v, t, stats = net.extract_mesh_sparse(resolution=1024, return_stats=True)
    peak = torch.cuda.max_memory_allocated() - before
    assert peak < 4 * 1024 ** 3, peak
    assert t.shape[0] > 1000000 and stats['points_evaluated'] < 1024 ** 3 // 4
    assert t.min() == 0 and t.max() == v.shape[0] - 1
    assert_closed_and_oriented(t, v.shape[0])
    assert np.abs(v).max() <= 1.0
