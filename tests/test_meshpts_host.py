"""CPU: the mesh clean-up and sampling oracle (components against scipy, points on their triangles, area-proportional
triangle counts, zero-area triangles never chosen, the blocked prefix), the argument checks of nero_b200.evaluate, of the C ABI
(include/nero_meshpts.h) and of tools/sample_mesh_points.py."""
import importlib.util
import os

import numpy as np
import pytest

import nero_oracle_meshpts as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def scipy_labels(tris, keep, V):
    """Triangle labels from scipy's connected components, relabelled to the smallest vertex index of each component."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = np.asarray(tris, np.int64)[keep]
    a = np.concatenate([t[:, 0], t[:, 1]])
    b = np.concatenate([t[:, 1], t[:, 2]])
    g = coo_matrix((np.ones(a.shape[0]), (a, b)), shape=(V, V))
    _, lab = connected_components(g, directed=False)
    first = np.full(lab.max() + 1, V, np.int64)
    np.minimum.at(first, lab, np.arange(V))
    out = np.full(np.asarray(tris).shape[0], V, np.int64)
    out[keep] = first[lab[t[:, 0]]]
    return out


def random_mesh(rng, V, T):
    v = rng.rand(V, 3).astype(np.float32)
    t = rng.randint(0, V, (T, 3)).astype(np.int32)
    return v, t


@pytest.mark.parametrize('V,T,seed', [(50, 20, 0), (400, 150, 1), (2000, 1200, 2), (3000, 5000, 3)])
def test_components_match_scipy_on_random_meshes(V, T, seed):
    rng = np.random.RandomState(seed)
    v, t = random_mesh(rng, V, T)
    keep = rng.rand(T) < 0.8
    lab = O.components(t, keep, V)
    np.testing.assert_array_equal(lab, scipy_labels(t, keep, V))
    assert (lab[~keep] == V).all()


def test_components_of_a_long_reversed_strip():
    v, t = O.reversed_strip(200_000)
    keep = np.ones(t.shape[0], bool)
    lab = O.components(t, keep, v.shape[0])
    assert (lab == 0).all()
    keep[100_000:100_002] = False    # two consecutive triangles out: the pieces share no vertex
    lab = O.components(t, keep, v.shape[0])
    np.testing.assert_array_equal(lab, scipy_labels(t, keep, v.shape[0]))
    assert np.unique(lab[keep]).tolist() == [0, t.shape[0] - 100_000]   # the far piece holds vertex 0


def test_floater_scene_components_and_selection():
    v, t = O.floater_scene()
    r = O.clean(v, t, min_component=0.5)
    np.testing.assert_array_equal(r['label'], scipy_labels(t, np.ones(t.shape[0], bool), v.shape[0]))
    assert r['comp_label'].shape[0] == 4 and r['comp_keep'].tolist() == [True, False, False, False]
    assert r['verts'].shape[0] == (r['label'] == 0).sum() // 2 + 2     # a closed sphere: V = T / 2 + 2
    r = O.clean(v, t, sphere=(0, 0, 0, 1.0))
    assert r['keep'].sum() == t.shape[0] - 2                            # the far quad is cropped
    r = O.clean(v, t, box=(-1, -1, -1, 1, 1, 1), min_component=0.0)
    assert r['comp_keep'].all() and r['comp_label'].shape[0] == 3


def test_component_areas_are_sequential_sums_in_triangle_order():
    rng = np.random.RandomState(4)
    v, t = random_mesh(rng, 300, 400)
    r = O.clean(v, t)
    for lab, s in zip(r['comp_label'], r['comp_area']):
        acc = 0.0
        for a in r['area'][r['label'] == lab]:
            acc += a
        assert acc == s


def test_compaction_keeps_order_and_geometry():
    v, t = O.floater_scene()
    r = O.clean(v, t, sphere=(0, 0, 0, 1.0), min_component=0.1)
    kept = np.asarray(t)[r['tri_keep']]
    np.testing.assert_array_equal(r['verts'][r['tris']], v[kept])
    used = np.unique(kept)
    np.testing.assert_array_equal(r['verts'], v[used])


def test_cdf_is_the_blocked_prefix():
    rng = np.random.RandomState(5)
    a = rng.rand(1000) * (rng.rand(1000) < 0.9)
    c = O.cdf(a)
    assert (np.diff(c) >= 0).all()
    ref = np.concatenate([np.cumsum(a[:256]), np.cumsum(a[256:512]), np.cumsum(a[512:768]), np.cumsum(a[768:])])
    off = np.cumsum([0.0, ref[255], ref[511], ref[767]])
    np.testing.assert_array_equal(c[:256], ref[:256])
    np.testing.assert_array_equal(c[256:512], off[1] + ref[256:512])
    assert abs(c[-1] - a.sum()) <= 1e-12 * a.sum()


def test_sample_points_lie_on_their_triangles():
    v, t = O.floater_scene()
    p, tri = O.sample(v, t, 20_000, seed=7)
    q = v.astype(np.float64)[t[tri]]
    e1, e2, d = q[:, 1] - q[:, 0], q[:, 2] - q[:, 0], p - q[:, 0]
    g = np.stack([np.einsum('ij,ij->i', e1, e1), np.einsum('ij,ij->i', e1, e2), np.einsum('ij,ij->i', e2, e2)], 1)
    rhs = np.stack([np.einsum('ij,ij->i', d, e1), np.einsum('ij,ij->i', d, e2)], 1)
    det = g[:, 0] * g[:, 2] - g[:, 1] ** 2
    b1 = (rhs[:, 0] * g[:, 2] - rhs[:, 1] * g[:, 1]) / det
    b2 = (rhs[:, 1] * g[:, 0] - rhs[:, 0] * g[:, 1]) / det
    b = np.stack([1 - b1 - b2, b1, b2], 1)
    assert (b >= -1e-12).all() and (b <= 1 + 1e-12).all()
    np.testing.assert_allclose(q[:, 0] + b1[:, None] * e1 + b2[:, None] * e2, p, atol=1e-12)


def test_triangle_counts_follow_the_areas():
    """Ten triangles with areas 1 : 2 : ... : 10 (and a zero-area one) get counts a chi-square test accepts."""
    from scipy.stats import chi2
    k = np.arange(1, 11, dtype=np.float32)
    verts, tris = [], []
    for i, s in enumerate(k):
        base = np.float32(3 * i)
        verts += [[base, 0, 0], [base + 2 * s / 10, 0, 0], [base, 1, 0]]
        tris.append([3 * i, 3 * i + 1, 3 * i + 2])
    verts += [[0, 5, 0], [1, 5, 0], [2, 5, 0]]                          # collinear: zero area
    tris.insert(4, [30, 31, 32])
    v, t = np.asarray(verts, np.float32), np.asarray(tris, np.int32)
    n = 200_000
    _, tri = O.sample(v, t, n, seed=11)
    counts = np.bincount(tri, minlength=11)
    assert counts[4] == 0
    obs = np.delete(counts, 4)
    exp = n * k / k.sum()
    stat = ((obs - exp) ** 2 / exp).sum()
    assert stat < chi2.ppf(0.999, 9), (obs, exp, stat)


def test_zero_area_triangles_are_never_chosen():
    rng = np.random.RandomState(8)
    v, t = random_mesh(rng, 40, 300)
    t[::3, 2] = t[::3, 1]                                                # a third of the triangles are degenerate
    t[0] = t[-1] = [5, 5, 5]
    a = O.areas(v, t)
    assert (a[::3] == 0).all()
    _, tri = O.sample(v, t, 100_000, seed=2)
    assert (a[tri] > 0).all()


def test_samples_do_not_depend_on_chunking_and_depend_on_the_seed():
    v, t = O.floater_scene()
    p, _ = O.sample(v, t, 3000, seed=5)
    parts = [O.sample(v, t, n, seed=5, i0=i0)[0] for i0, n in ((0, 1000), (1000, 1), (1001, 1999))]
    np.testing.assert_array_equal(np.concatenate(parts), p)
    assert not np.array_equal(O.sample(v, t, 3000, seed=6)[0], p)


def test_hash_is_the_relight_mix():
    import nero_oracle_relight as ORl
    x = np.random.RandomState(0).randint(0, 2 ** 32, 1000, dtype=np.uint64)
    np.testing.assert_array_equal(O._mix(x.astype(np.uint32)), ORl._mix(x).astype(np.uint32))


@pytest.mark.parametrize('kw', [dict(min_component=1.5), dict(min_component=-0.1), dict(sphere=(0, 0, 0, 0)),
                                dict(sphere=(0, 0, 0, -1)), dict(sphere=(0, 0, 0)), dict(box=(1, 0, 0, 0, 1, 1)),
                                dict(box=(0, 0, 0, 1, 1, np.nan))])
def test_clean_mesh_rejects_bad_regions_on_the_host(kw):
    from nero_b200 import evaluate as E
    v, t = O.floater_scene()
    with pytest.raises(ValueError):
        E.clean_mesh(v, t, **kw)


def test_bad_meshes_and_counts_are_rejected_on_the_host():
    from nero_b200 import evaluate as E
    v, t = O.floater_scene()
    for fn in (E.clean_mesh, lambda a, b: E.sample_surface(a, b, 10)):
        with pytest.raises(ValueError):
            fn(v, t + 1000)
        with pytest.raises(ValueError):
            fn(v, t - 1)
        with pytest.raises(ValueError):
            fn(v, t[:0])
        with pytest.raises(ValueError):
            fn(v[:, :2], t)
        bad = v.copy()
        bad[3, 1] = np.inf
        with pytest.raises(ValueError):
            fn(bad, t)
    for kw in (dict(n=0), dict(n=-5), dict(n=10, seed=-1), dict(n=10, seed=2 ** 32), dict(n=10, first=-1)):
        with pytest.raises(ValueError):
            E.sample_surface(v, t, **kw)


def test_c_abi_rejects_bad_arguments_without_launching():
    from nero_b200 import ops
    lib = ops.lib
    buf = 16      # never dereferenced: the checks come first
    good_s = np.asarray([0, 0, 0, 1.0])
    assert lib.nero_meshpts_areas(buf, 0, buf, 4, None, None, buf, buf, None) == 1
    assert lib.nero_meshpts_areas(buf, 4, buf, 0, None, None, buf, buf, None) == 1
    assert lib.nero_meshpts_areas(None, 4, buf, 4, None, None, buf, buf, None) == 1
    assert lib.nero_meshpts_areas(buf, 4, buf, 4, np.asarray([0, 0, 0, 0.0]), None, buf, buf, None) == 1
    assert lib.nero_meshpts_areas(buf, 4, buf, 4, np.asarray([0, 0, np.nan, 1.0]), None, buf, buf, None) == 1
    assert lib.nero_meshpts_areas(buf, 4, buf, 4, None, np.asarray([0, 0, 1, 1, 1, 0.0]), buf, buf, None) == 1
    assert lib.nero_meshpts_areas(buf, 4, buf, 4, good_s, None, buf, None, None) == 1     # a crop needs keep
    assert lib.nero_meshpts_components(buf, 4, buf, 0, buf, buf, None) == 1
    assert lib.nero_meshpts_components(buf, 0, buf, 4, buf, buf, None) == 1
    assert lib.nero_meshpts_components(buf, 4, None, 4, buf, buf, None) == 1
    for frac in (-0.5, 1.5, float('nan')):
        assert lib.nero_meshpts_component_areas(buf, buf, buf, buf, 3, frac, buf, buf, None) == 1
    assert lib.nero_meshpts_component_areas(buf, buf, buf, buf, 0, 0.5, buf, buf, None) == 1
    assert lib.nero_meshpts_compact_count(buf, 4, buf, buf, buf, 0, buf, buf, buf, buf, buf, None) == 1
    assert lib.nero_meshpts_compact_count(buf, 4, buf, buf, None, 4, buf, buf, buf, buf, buf, None) == 1
    assert lib.nero_meshpts_compact_emit(buf, 4, buf, 4, buf, buf, buf, 5, 1, buf, buf, buf, None) == 1
    assert lib.nero_meshpts_compact_emit(buf, 4, buf, 4, buf, buf, buf, 1, 5, buf, buf, buf, None) == 1
    assert lib.nero_meshpts_compact_emit(buf, 4, buf, 4, buf, buf, buf, 1, 1, buf, None, buf, None) == 1
    assert lib.nero_meshpts_cdf(buf, 0, buf, buf, None) == 1
    assert lib.nero_meshpts_cdf(buf, 4, None, buf, None) == 1
    assert lib.nero_meshpts_sample(buf, 4, buf, 4, buf, 0, 0, 0, buf, None) == 1
    assert lib.nero_meshpts_sample(buf, 4, buf, 4, buf, 0, -1, 10, buf, None) == 1
    assert lib.nero_meshpts_sample(buf, 4, buf, 4, None, 0, 0, 10, buf, None) == 1
    assert lib.nero_meshpts_sample(buf, 4, buf, 4, buf, 0, 0, 2 ** 40, buf, None) == 1


def _tool():
    spec = importlib.util.spec_from_file_location('sample_mesh_points', os.path.join(ROOT, 'tools', 'sample_mesh_points.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_tool_argument_errors(tmp_path):
    tool = _tool()
    mesh = tmp_path / 'm.ply'
    mesh.write_bytes(b'ply\n')
    base = ['--mesh', str(mesh), '--out', str(tmp_path / 'p.ply')]
    f = tool.parse_args(base + ['--num', '1000', '--crop-sphere', '0', '0', '0', '1', '--crop-box', '-1', '-1', '-1', '1', '1', '1',
                                '--min-component', '0.5', '--seed', '3'])
    assert f.num == 1000 and f.crop_sphere == [0, 0, 0, 1] and f.crop_box == [-1, -1, -1, 1, 1, 1] and f.min_component == 0.5
    assert tool.parse_args(base).num == 500_000 and tool.parse_args(base).min_component == 0.0
    for extra in (['--num', '0'], ['--min-component', '1.5'], ['--min-component', '-1'], ['--crop-sphere', '0', '0', '0', '0'],
                  ['--crop-sphere', '0', '0', '1'], ['--crop-box', '1', '0', '0', '0', '1', '1'], ['--seed', '-1']):
        with pytest.raises(SystemExit):
            tool.parse_args(base + extra)
    with pytest.raises(SystemExit):
        tool.parse_args(['--mesh', str(tmp_path / 'missing.ply'), '--out', str(tmp_path / 'p.ply')])
    with pytest.raises(SystemExit):
        tool.parse_args(['--mesh', str(mesh)])
