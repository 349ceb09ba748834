"""CPU: the brick-wise marching-cubes oracle (oracle/nero_oracle_mcsparse.py) gives exactly the arrays of the dense oracle
(nero_oracle_mesh.marching_cubes on the whole grid) on analytic fields, growth finds what seeding misses, and the argument
checks of nero_b200.mesh.extract_sparse and of include/nero_mcsparse.h run before anything touches a device.  No GPU."""
import ctypes
import os
import re

import numpy as np
import pytest

import nero_oracle_mcsparse as OS
import nero_oracle_mesh as OMesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def norm(p):
    return np.linalg.norm(p.astype(np.float64), axis=-1)


def sphere(p):
    return norm(p) - 0.55


def torus(p):
    q = p.astype(np.float64)
    return np.sqrt((np.sqrt(q[:, 0] ** 2 + q[:, 1] ** 2) - 0.5) ** 2 + q[:, 2] ** 2) - 0.2


def two_spheres(p):
    return np.minimum(norm(p - np.float32([0.45, 0.1, 0.0])) - 0.3, norm(p + np.float32([0.4, 0.2, 0.1])) - 0.25)


def cut_sphere(p):
    """negative up to the unit sphere and beyond: the override to 1.0 outside it makes part of the surface"""
    return norm(p - np.float32([0.7, 0.1, 0.0])) - 0.5


def ties(p):
    """values on a lattice of quarters, so that many grid points have u == iso exactly"""
    return np.round(4.0 * (norm(p) - 0.5)) / 4.0


def steep(p):
    return 5.0 * (norm(p) - 0.5)


def grid_axes(n, lo=-1.0, hi=1.0):
    n = (n, n, n) if np.isscalar(n) else n
    lo, hi = np.broadcast_to(lo, 3), np.broadcast_to(hi, 3)
    return [np.linspace(lo[a], hi[a], n[a]).astype(np.float32) for a in range(3)]


# name: (field, grid points, isovalue, outside); the GPU tests run the same cases
CASES = {
    'sphere': (sphere, 65, 0.0, None),
    'torus': (torus, (50, 45, 61), 0.0, None),
    'two_spheres': (two_spheres, 57, 0.0, None),
    'cut_sphere': (cut_sphere, 49, 0.0, 1.0),
    'isovalue': (torus, 41, 0.07, None),
    'ties': (ties, 33, 0.0, None),
}
TABLES = OMesh.load_tables()


def check_sparse_equals_dense(field, axes, iso, brick, lipschitz=2.0, outside=None):
    u = OS.dense_field(field, axes, outside)
    dv, dt = OMesh.marching_cubes(u, iso, TABLES)
    sv, st, stats = OS.extract_sparse(field, axes, iso, brick, lipschitz, outside, tables=TABLES)
    assert sv.dtype == np.float64 and st.dtype == np.int64
    np.testing.assert_array_equal(st, dt)
    np.testing.assert_array_equal(sv, dv)
    assert stats['vertices'] == dv.shape[0] and stats['triangles'] == dt.shape[0]
    return u, dv, dt, stats


@pytest.mark.parametrize('brick', [4, 8, 16])
@pytest.mark.parametrize('case', sorted(CASES))
def test_sparse_oracle_equals_dense_oracle(case, brick):
    field, n, iso, outside = CASES[case]
    u, dv, dt, stats = check_sparse_equals_dense(field, grid_axes(n), iso, brick, outside=outside)
    assert dt.shape[0] > 500
    assert stats['points_evaluated'] == stats['bricks'] * (brick + 1) ** 3
    if case == 'ties':
        assert (u == 0).sum() > 100
    if case == 'cut_sphere':
        x = np.stack(np.meshgrid(*grid_axes(n), indexing='ij'), -1)
        r = np.linalg.norm(x, axis=-1)
        assert (cut_sphere(x.reshape(-1, 3)).reshape(r.shape)[(r >= 1.0) & (r < 1.05)] < 0).any(), 'the field is negative at the cut'


def test_large_grid_and_anisotropic_bounds():
    check_sparse_equals_dense(sphere, grid_axes(97), 0.0, 16)
    check_sparse_equals_dense(torus, grid_axes((40, 52, 47), (-0.9, -1.0, -0.5), (0.8, 1.0, 0.6)), 0.0, 8)


def test_float32_vertices_are_the_kernels_arithmetic():
    field, n, iso, outside = CASES['torus']
    v64, t64, _ = OS.extract_sparse(field, grid_axes(n), iso, 8, tables=TABLES)
    v32, t32, _ = OS.extract_sparse(field, grid_axes(n), iso, 8, dtype=np.float32, tables=TABLES)
    assert v32.dtype == np.float32
    np.testing.assert_array_equal(t32, t64)
    assert np.abs(v32 - v64).max() <= 1e-5


def test_growth_finds_what_seeding_misses():
    """5 (|x| - 0.5) with lipschitz = 1: only bricks with a corner within 0.17 brick widths of the surface are seeds."""
    axes = grid_axes(65)
    u, dv, dt, stats = check_sparse_equals_dense(steep, axes, 0.0, 8, lipschitz=1.0)
    assert stats['seed_bricks'] > 0 and stats['grow_rounds'] >= 1 and stats['bricks_added'] > 0
    # the bricks the surface crosses outnumber the seeds: seeding alone would have lost triangles
    _, _, full = OS.extract_sparse(steep, axes, 0.0, 8, lipschitz=5.0, tables=TABLES)
    assert full['grow_rounds'] == 0 and full['seed_bricks'] >= stats['bricks'] > stats['seed_bricks']


def test_empty_field():
    for value in (1.0, -1.0):
        v, t, stats = OS.extract_sparse(lambda p: np.full(p.shape[0], value, np.float32), grid_axes(33), 0.0, 8, tables=TABLES)
        assert v.shape == (0, 3) and t.shape == (0, 3) and stats['bricks'] == 0 and stats['triangles'] == 0
    # seeds everywhere (|u - iso| is small) and still no surface
    v, t, stats = OS.extract_sparse(lambda p: np.full(p.shape[0], 0.01, np.float32), grid_axes(20), 0.0, 4, tables=TABLES)
    assert v.shape == (0, 3) and t.shape == (0, 3) and stats['bricks'] == 5 ** 3


def test_bad_arguments_raise():
    import torch
    from nero_b200.mesh import extract_sparse
    axes = grid_axes(17)
    for brick in (0, 5, 32):
        with pytest.raises(ValueError):
            OS.extract_sparse(sphere, axes, 0.0, brick)
        with pytest.raises(ValueError):
            extract_sparse(None, [torch.from_numpy(a) for a in axes], 0.0, brick=brick)
    with pytest.raises(ValueError):
        OS.extract_sparse(sphere, axes[:2], 0.0, 8)
    with pytest.raises(ValueError):
        OS.extract_sparse(sphere, [axes[0], axes[1], axes[2][:1]], 0.0, 8)
    t = [torch.from_numpy(a) for a in axes]
    for bad in (t[:2], [t[0], t[1], t[2][:1]], [t[0], t[1], t[2].reshape(1, -1)]):
        with pytest.raises(ValueError):
            extract_sparse(None, bad, 0.0)
    with pytest.raises(RuntimeError):                       # CPU tensors: there is no CPU path
        extract_sparse(None, t, 0.0)


def test_mcsparse_header_is_bound():
    """Every prototype of include/nero_mcsparse.h is exported by the library and bound with one argtype per parameter."""
    from nero_b200 import ops
    txt = re.sub(r'/\*.*?\*/', ' ', open(os.path.join(ROOT, 'include', 'nero_mcsparse.h')).read(), flags=re.S)
    protos = dict(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(([^)]*)\)', txt))
    assert len(protos) == 9 and set(protos) == set(ops.MCSPARSE_PROTOS)
    for name, params in protos.items():
        fn = getattr(ops.lib, name)
        assert fn.argtypes is not None and len(fn.argtypes) == params.count(',') + 1 and fn.restype is ctypes.c_int, name


def test_c_abi_rejects_bad_arguments_without_launching():
    from nero_b200 import ops
    lib = ops.lib
    buf = 16      # never dereferenced: the checks come first
    for grid in ((1, 9, 9, 8), (9, 9, 1, 8), (9, 9, 9, 5), (9, 9, 9, 0)):
        assert lib.nero_mcsparse_coarse_points(buf, buf, buf, *grid, 0, 8, buf, None) == 1
        assert lib.nero_mcsparse_seed(buf, None, *grid, 0.0, 0.1, buf, None) == 1
        assert lib.nero_mcsparse_brick_points(buf, buf, buf, *grid, buf, 0, 1, buf, None) == 1
        assert lib.nero_mcsparse_grow(buf, buf, 0, 1, buf, *grid, 0.0, buf, None) == 1
        assert lib.nero_mcsparse_count(buf, buf, 1, *grid, 0.0, buf, buf, buf, None) == 1
        assert lib.nero_mcsparse_emit(buf, buf, 1, *grid, 0.0, buf, buf, buf, buf, buf, None) == 1
    good = (9, 9, 9, 8)
    assert lib.nero_mcsparse_coarse_points(buf, buf, buf, *good, 0, 9, buf, None) == 1        # 8 coarse points only
    assert lib.nero_mcsparse_coarse_points(buf, buf, None, *good, 0, 8, buf, None) == 1
    assert lib.nero_mcsparse_seed(buf, None, *good, 0.0, -1.0, buf, None) == 1
    assert lib.nero_mcsparse_seed(buf, None, *good, 0.0, float('nan'), buf, None) == 1
    assert lib.nero_mcsparse_compact_count(buf, 0, buf, buf, buf, None) == 1
    assert lib.nero_mcsparse_compact_count(buf, 2 ** 31, buf, buf, buf, None) == 1
    assert lib.nero_mcsparse_compact_emit(buf, 8, buf, -1, buf, buf, None) == 1
    assert lib.nero_mcsparse_brick_points(buf, buf, buf, *good, None, 0, 1, buf, None) == 1
    assert lib.nero_mcsparse_grow(buf, buf, 0, 0, buf, *good, 0.0, buf, None) == 1
    assert lib.nero_mcsparse_count(buf, buf, 0, *good, 0.0, buf, buf, buf, None) == 1
    assert lib.nero_mcsparse_emit(buf, buf, 1, *good, 0.0, buf, None, buf, buf, buf, None) == 1
    assert lib.nero_mcsparse_lookup(buf, 0, buf, 3, buf, None) == 1
    assert lib.nero_mcsparse_lookup(buf, 2 ** 31, buf, 3, buf, None) == 1
    assert lib.nero_mcsparse_lookup(buf, 4, None, 3, buf, None) == 1
