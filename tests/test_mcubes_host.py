"""CPU: the generated marching-cubes tables (tools/gen_mc_tables.py -> nero_b200/csrc/mc_tables.cuh), the numpy oracle built on
them (closed, consistently oriented meshes; a sphere), the PLY writer, and the argument checks of the C ABI."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_mesh as OMesh

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _generator():
    spec = importlib.util.spec_from_file_location('gen_mc_tables', os.path.join(ROOT, 'tools', 'gen_mc_tables.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_generator_reproduces_committed_header():
    with open(OMesh.TABLES) as f:
        assert f.read() == _generator().render()


def _case_tris(ntri, tri, case):
    return [tuple(int(e) for e in tri[case, 3 * i:3 * i + 3]) for i in range(ntri[case])]


def test_table_uses_exactly_the_sign_change_edges():
    edge_corner, ntri, tri = OMesh.load_tables()
    for case in range(256):
        cut = {e for e in range(12) if (case >> edge_corner[e, 0] & 1) != (case >> edge_corner[e, 1] & 1)}
        used = {e for t in _case_tris(ntri, tri, case) for e in t}
        assert used == cut, case
        assert (tri[case, 3 * ntri[case]:] == -1).all()


def test_table_orientation_is_consistent_within_each_case():
    _, ntri, tri = OMesh.load_tables()
    for case in range(256):
        directed = []
        for t in _case_tris(ntri, tri, case):
            assert len(set(t)) == 3, (case, t)
            directed += [(t[0], t[1]), (t[1], t[2]), (t[2], t[0])]
        assert len(set(directed)) == len(directed), case           # no directed edge twice
        for a, b in directed:
            if sum(1 for d in directed if set(d) == {a, b}) == 2:
                assert (b, a) in directed, case


def _directed_edges(tris):
    return np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])


def assert_closed_and_oriented(tris, n_verts):
    d = _directed_edges(np.asarray(tris, np.int64))
    key = d[:, 0] * n_verts + d[:, 1]
    rev = d[:, 1] * n_verts + d[:, 0]
    assert np.unique(key).shape[0] == key.shape[0], 'a directed edge is used twice'
    assert np.isin(rev, key).all(), 'an edge is used by one triangle only'


def smooth_field(shape, seed, amp=0.4, k=6):
    """|x| - 0.7 + amp * noise(x) * (1 - |x|^2) on [-1,1]^3: smooth, with its zero set inside the grid (positive for |x| >= 1)."""
    rng = np.random.RandomState(seed)
    axes = [np.linspace(-1.0, 1.0, n) for n in shape]
    x = np.stack(np.meshgrid(*axes, indexing='ij'), -1)
    r = np.linalg.norm(x, axis=-1)
    w = rng.randn(k, 3) * 4.0
    ph = rng.rand(k) * 2 * np.pi
    noise = sum(np.sin(x @ w[i] + ph[i]) for i in range(k)) / k
    return (r - 0.7 + amp * noise * (1.0 - r * r)).astype(np.float32)


@pytest.mark.parametrize('shape,seed', [((20, 20, 20), 1), ((24, 31, 17), 2), ((33, 33, 33), 3), ((16, 40, 28), 4)])
def test_oracle_meshes_of_smooth_fields_are_closed(shape, seed):
    u = smooth_field(shape, seed)
    assert (u != 0).all()
    v, t = OMesh.marching_cubes(u, 0.0)
    assert t.shape[0] > 100
    assert_closed_and_oriented(t, v.shape[0])
    assert np.unique(t).shape[0] == v.shape[0], 'every vertex is used'


@pytest.mark.parametrize('res', [16, 24, 40])
def test_oracle_sphere(res):
    r = 0.55
    ax = np.linspace(-1.0, 1.0, res)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    u = (np.linalg.norm(x, axis=-1) - r).astype(np.float32)
    assert (u != 0).all()
    v, t = OMesh.marching_cubes(u, 0.0)
    assert_closed_and_oriented(t, v.shape[0])
    d = _directed_edges(t)
    n_edges = np.unique(np.sort(d, 1), axis=0).shape[0]
    assert v.shape[0] - n_edges + t.shape[0] == 2, 'Euler characteristic of a sphere'
    h = 2.0 / (res - 1)
    w = v * h - 1.0
    assert np.abs(np.linalg.norm(w, axis=-1) - r).max() < h * h
    p0, p1, p2 = w[t[:, 0]], w[t[:, 1]], w[t[:, 2]]
    n = np.cross(p1 - p0, p2 - p0)
    c = (p0 + p1 + p2) / 3.0
    assert (np.linalg.norm(n, axis=-1) > 0).all()
    assert ((n * c).sum(-1) < 0).all(), 'face normals point to the inside (the below side)'


def test_oracle_order_and_vertex_positions():
    """Canonical order on a small field, checked independently of the oracle's vectorised construction."""
    u = smooth_field((7, 6, 5), 9, amp=0.8)
    iso = np.float32(0.05)
    v, t = OMesh.marching_cubes(u, iso)
    want = []
    for L in range(u.size):
        p = np.unravel_index(L, u.shape)
        for a in range(3):
            q = list(p)
            q[a] += 1
            if q[a] < u.shape[a] and (u[p] <= iso) != (u[tuple(q)] <= iso):
                tt = (np.float64(iso) - np.float64(u[p])) / (np.float64(u[tuple(q)]) - np.float64(u[p]))
                want.append([p[i] + (tt if i == a else 0.0) for i in range(3)])
    np.testing.assert_array_equal(v, np.array(want))
    assert t.shape[0] > 0


def test_write_ply_round_trips_through_read_ply(tmp_path):
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    u = smooth_field((18, 18, 18), 5)
    v, t = OMesh.marching_cubes(u, 0.0)
    v = v / 17.0 * 2.0 - 1.0
    path = str(tmp_path / 'm.ply')
    write_ply(path, v, t)
    rv, rt = read_ply(path)
    np.testing.assert_array_equal(rv, v.astype(np.float32))
    np.testing.assert_array_equal(rt, t)
    write_ply(path, np.zeros((0, 3)), np.zeros((0, 3), np.int64))
    rv, rt = read_ply(path)
    assert rv.shape == (0, 3) and rt.shape == (0, 3)
    with pytest.raises(ValueError):
        write_ply(path, v, t + v.shape[0])


def test_c_abi_rejects_bad_arguments_without_launching():
    from nero_b200 import ops
    lib = ops.lib
    buf = 16      # never dereferenced: the checks come first
    for dims in ((1, 4, 4), (4, 1, 4), (4, 4, 1), (0, 4, 4)):
        assert lib.nero_mcubes_count(buf, *dims, 0.0, buf, buf, buf, None) == 1
        assert lib.nero_mcubes_emit(buf, *dims, 0.0, buf, 0, 0, buf, buf, buf, None) == 1
    big = 2 ** 31
    assert lib.nero_mcubes_emit(buf, 4, 4, 4, 0.0, buf, big, 1, buf, buf, buf, None) == 1
    assert lib.nero_mcubes_emit(buf, 4, 4, 4, 0.0, buf, 8, big, buf, buf, buf, None) == 1
    assert lib.nero_mcubes_count(None, 4, 4, 4, 0.0, buf, buf, buf, None) == 1


def test_marching_cubes_rejects_bad_shapes_before_touching_the_device():
    from nero_b200.mesh import marching_cubes
    for shape in ((4, 4), (4, 4, 4, 4), (1, 5, 5), (5, 5, 1)):
        with pytest.raises(ValueError):
            marching_cubes(np.zeros(shape, np.float32), 0.0)


def test_matches_pymcubes_when_available():
    mcubes = pytest.importorskip('mcubes')
    from scipy.spatial import cKDTree
    u = smooth_field((30, 26, 34), 7)
    v, t = OMesh.marching_cubes(u, 0.0)
    mv, mt = mcubes.marching_cubes(u, 0.0)
    assert cKDTree(mv).query(v)[0].max() < 1e-6 and cKDTree(v).query(mv)[0].max() < 1e-6

    def area(vv, tt):
        return 0.5 * np.linalg.norm(np.cross(vv[tt[:, 1]] - vv[tt[:, 0]], vv[tt[:, 2]] - vv[tt[:, 0]]), axis=-1).sum()
    assert abs(area(v, t) - area(mv, mt)) <= 1e-3 * area(mv, mt)
