"""CPU: the mesh simplification oracle (oracle/nero_oracle_simplify.py): rejections of malformed meshes, topology kept on
marching-cubes meshes of a sphere, a torus and four blobs, independent selected sets on every round, planes kept planar,
locked boundaries kept bit for bit; the argument checks of the C ABI (include/nero_simplify.h); and the per-round torch
plumbing of nero_b200.simplify (threshold, edges, CSRs) against the oracle above 2^24 edges and valid keys."""
import ctypes

import numpy as np
import pytest

import nero_oracle_mesh as OMesh
import nero_oracle_simplify as O


def _world(u, res):
    v, t = OMesh.marching_cubes(u.astype(np.float32), 0.0)
    return (v * (2.0 / (res - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def _grid(res):
    ax = np.linspace(-1.0, 1.0, res)
    return np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)


def sphere_mesh(res=32, r=0.6):
    x = _grid(res)
    return _world(np.linalg.norm(x, axis=-1) - r + 0.05 * np.sin(5 * x[..., 0]) * np.cos(4 * x[..., 1] + x[..., 2]), res)


def torus_mesh(res=40, R=0.5, r=0.2):
    x = _grid(res)
    return _world(np.hypot(np.hypot(x[..., 0], x[..., 1]) - R, x[..., 2]) - r, res)


def blobs_mesh(res=40):
    """Four separate blobs of different sizes (the blobs of tests/test_meshpts_gpu.py)."""
    x = _grid(res)
    cs = np.asarray([[-0.45, -0.4, -0.3], [0.45, 0.4, 0.3], [0.5, -0.5, 0.4], [-0.5, 0.5, -0.5]])
    rs = np.asarray([0.4, 0.3, 0.18, 0.1])
    return _world(np.min(np.linalg.norm(x[..., None, :] - cs, axis=-1) - rs, -1), res)


def cropped_mesh():
    """The sphere cut open by z < 0.2: the triangles with all three vertices below, and the vertices they use."""
    v, t = sphere_mesh()
    t = t[(v[t][..., 2] < 0.2).all(1)]
    used = np.unique(t)
    new = np.full(v.shape[0], -1, np.int64)
    new[used] = np.arange(used.shape[0])
    return v[used], new[t].astype(np.int32)


MESHES = {'sphere': sphere_mesh, 'torus': torus_mesh, 'blobs': blobs_mesh}
EULER = {'sphere': [2], 'torus': [0], 'blobs': [2, 2, 2, 2]}


def components(tris, V):
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import connected_components
    t = np.asarray(tris, np.int64)
    a, b = np.concatenate([t[:, 0], t[:, 1]]), np.concatenate([t[:, 1], t[:, 2]])
    _, lab = connected_components(coo_matrix((np.ones(a.shape[0]), (a, b)), shape=(V, V)), directed=False)
    return lab


def euler(tris, V):
    """Euler characteristic of each component, ordered by the component's smallest vertex."""
    lab = components(tris, V)
    t = np.asarray(tris, np.int64)
    e = np.unique(np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), 1), axis=0)
    out = []
    for c in np.unique(lab):
        nv = int((lab == c).sum())
        out.append(nv - int((lab[e[:, 0]] == c).sum()) + int((lab[t[:, 0]] == c).sum()))
    return out


def zero_area(v, t):
    return int((O._cross(*(v.astype(np.float64)[t[:, c]] for c in range(3))) == 0).all(1).sum())


def target(T, frac=0.1):
    return 2 * int(round(T * frac / 2))


@pytest.mark.parametrize('name', sorted(MESHES))
def test_topology_is_kept(name):
    v, t = MESHES[name]()
    F = target(t.shape[0])
    trace = []
    ov, ot, st = O.simplify(v, t, F, trace=trace)
    assert ot.shape[0] == F and st['triangles'] == F and st['rounds'] == len(st['collapses']) > 0
    assert st['locked'] == 0
    twin = O.check(ov, ot)                               # indices, repeats, edges in > 2 triangles, winding
    assert (twin >= 0).all(), 'the output has a boundary edge'
    assert np.array_equal(np.unique(ot), np.arange(ov.shape[0])), 'unreferenced or missing vertices'
    assert zero_area(ov, ot) <= zero_area(v, t)
    assert euler(ot, ov.shape[0]) == euler(t, v.shape[0]) == EULER[name]
    assert sum(st['collapses']) * 2 == t.shape[0] - F
    assert [int(r['collapsed'].sum()) for r in trace if r['collapsed'].any()] == st['collapses']


@pytest.mark.parametrize('name', sorted(MESHES))
def test_selected_edges_have_disjoint_neighbourhoods(name):
    """On every round: no endpoint of a selected edge lies in the closed 1-ring of an endpoint of another selected edge, so
    no triangle touches two of them."""
    v, t = MESHES[name]()
    trace = []
    O.simplify(v, t, target(t.shape[0]), trace=trace)
    V = v.shape[0]
    assert len(trace) > 3
    for r in trace:
        tris = r['tris']
        sel = r['edges'][r['selected']]
        assert sel.shape[0] > 0
        assert (r['key'][r['collapsed']] != O.KEY_INF).all() and not (r['collapsed'] & ~r['selected']).any()
        adj = np.zeros((V, V), bool)
        for i, j in ((0, 1), (1, 2), (2, 0)):
            adj[tris[:, i], tris[:, j]] = adj[tris[:, j], tris[:, i]] = True
        adj[np.arange(V), np.arange(V)] = True
        ring = adj[sel[:, 0]] | adj[sel[:, 1]]           # closed 1-ring of each selected edge's endpoints
        cover = ring.sum(0)
        assert (cover[sel[:, 0]] == 1).all() and (cover[sel[:, 1]] == 1).all()
        owner = np.full(V, -1)
        owner[sel[:, 0]] = owner[sel[:, 1]] = np.arange(sel.shape[0])
        o = owner[tris]
        o0 = np.where(o[:, 0] >= 0, o[:, 0], np.where(o[:, 1] >= 0, o[:, 1], o[:, 2]))
        assert ((o == -1) | (o == o0[:, None])).all(), 'a triangle touches two selected edges'


def test_planes_stay_planar():
    """A jittered planar grid on z = (x + y) / 4 with dyadic coordinates: every output vertex is on the plane."""
    n = 24
    rng = np.random.RandomState(3)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    x = (i * 8 + rng.randint(-2, 3, i.shape)) / 64.0
    y = (j * 8 + rng.randint(-2, 3, j.shape)) / 64.0
    v = np.stack([x, y, (x + y) / 4], -1).reshape(-1, 3).astype(np.float32)
    q = (i[:-1, :-1] * n + j[:-1, :-1]).reshape(-1)
    t = np.concatenate([np.stack([q, q + n, q + n + 1], 1), np.stack([q, q + n + 1, q + 1], 1)]).astype(np.int32)
    ov, ot, st = O.simplify(v, t, 400)
    assert st['rounds'] > 0 and ot.shape[0] < t.shape[0] and st['locked'] == 4 * (n - 1)
    p = ov.astype(np.float64)
    assert np.abs(p[:, 2] - (p[:, 0] + p[:, 1]) / 4).max() <= 1e-12
    n_out = O._cross(*(p[ot[:, c]] for c in range(3)))
    assert (n_out[:, 2] > 0).all(), 'a triangle flipped'


def test_boundaries_are_locked():
    v, t = cropped_mesh()
    twin = O.check(v, t)
    src, dst = t.reshape(-1), t[:, [1, 2, 0]].reshape(-1)
    bnd = np.unique(np.concatenate([src[twin < 0], dst[twin < 0]]))
    assert bnd.shape[0] > 20
    ov, ot, st = O.simplify(v, t, target(t.shape[0], 0.2))
    assert st['locked'] >= bnd.shape[0] and ot.shape[0] < t.shape[0] // 2
    otw = O.check(ov, ot)
    osrc, odst = ot.reshape(-1), ot[:, [1, 2, 0]].reshape(-1)
    edges_in = {(tuple(v[a]), tuple(v[b])) for a, b in zip(src[twin < 0], dst[twin < 0])}
    edges_out = {(tuple(ov[a]), tuple(ov[b])) for a, b in zip(osrc[otw < 0], odst[otw < 0])}
    assert edges_in == edges_out, 'the boundary changed'


def test_rejections():
    v = np.random.RandomState(0).rand(6, 3).astype(np.float32)
    cases = [(np.array([[0, 1, 2], [0, 2, 6]]), r'triangle 1 has an index outside \[0, 6\): \(0, 2, 6\)'),
             (np.array([[0, 1, 2], [3, 4, 3]]), r'triangle 1 repeats an index: \(3, 4, 3\)'),
             (np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [2, 1, 5]]), r'edge \(0, 1\) is used by more than two triangles'),
             (np.array([[0, 1, 2], [2, 1, 3], [0, 1, 4]]), r'edge \(0, 1\) is used twice in the same direction')]
    for t, msg in cases:
        with pytest.raises(ValueError, match=msg):
            O.simplify(v, t.astype(np.int32), 4)
    with pytest.raises(ValueError, match='face count'):
        O.simplify(v, np.array([[0, 1, 2]], np.int32), 3)


def test_zero_area_triangles_are_accepted():
    """Marching cubes makes zero-area triangles where a grid value equals the isovalue: accepted, never a collapse that
    leaves a triangle with a zero normal."""
    res = 24
    x = _grid(res)
    u = np.round((np.linalg.norm(x, axis=-1) - 0.55) * 8) / 8               # many grid values exactly at the isovalue
    v, t = _world(u, res)
    assert zero_area(v, t) > 0
    trace = []
    ov, ot, _ = O.simplify(v, t, target(t.shape[0], 0.3), trace=trace)
    assert zero_area(ov, ot) <= zero_area(v, t)
    O.check(ov, ot)


def test_c_abi_refuses_bad_arguments():
    from nero_b200 import ops
    buf = (ctypes.c_byte * 4096)()
    p = ctypes.addressof(buf)
    assert ops.lib.nero_simplify_check_tris(p, 0, 3, p, None) == 1
    assert ops.lib.nero_simplify_check_edges(p, p, 2, p, p, None) == 1
    assert ops.lib.nero_simplify_edges(p, p, p, 3, p, 1, p, p, p, p, p, p, 0, p, p, p, None) == 1
    assert ops.lib.nero_simplify_select(p, p, 1, p, p, p, 0, p, p, p, None) == 1
    assert ops.lib.nero_simplify_collapse(p, p, 1, p, p, None, p, 3, p, p, p, p, None) == 1
    assert ops.lib.nero_simplify_rewrite_emit(p, 2, p, p, 3, p, None) == 1
    assert ops.lib.nero_simplify_output_emit(p, 3, p, 1, p, p, 4, p, p, p, None) == 1


# ------------------------------------------------------------------------------------------------ plumbing at full size
# The per-round plumbing of nero_b200/simplify.py (torch on any device) against the oracle at sizes the 2048^3 meshes
# reach: more than 2^24 edges and valid keys, where a float32 rank or index would round.

@pytest.mark.parametrize('nvalid', [2 ** 24 + 1, 21000001])
def test_threshold_is_exact_above_2_24_valid_keys(nvalid):
    import torch
    from nero_b200.simplify import _threshold
    rng = np.random.RandomState(nvalid % 1000)
    E = nvalid + 4099
    ids = np.arange(E, dtype=np.int64)
    key = (rng.randint(0, 1 << 30, E).astype(np.int64) << 32) | ids
    key[rng.permutation(E)[:E - nvalid]] = O.KEY_INF
    sel = (rng.rand(E) < 0.05) & (key != O.KEY_INF)
    exact = np.sort(key)[-(-nvalid // 4) - 1]                 # ceil(nvalid / 4)-th smallest valid key, in integers
    for budget in (E, 1000):
        want = O.threshold(key, sel, budget)
        got = int(_threshold(torch.from_numpy(key), torch.from_numpy(sel.astype(np.uint8)), budget)[0])
        assert got == want
        if budget == E:
            assert want == exact


def test_edges_and_vertex_triangles_above_2_24_edges():
    """A closed 2400 x 2400 torus grid: 11.5 M triangles, 17.3 M edges, the adjacency and triangle CSRs equal the oracle's."""
    import torch
    from nero_b200.simplify import _edges, _vertex_triangles
    n = 2400
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    v00, v10, v01, v11 = i * n + j, (i + 1) % n * n + j, i * n + (j + 1) % n, (i + 1) % n * n + (j + 1) % n
    tris = np.concatenate([np.stack([v00, v10, v11], -1).reshape(-1, 3), np.stack([v00, v11, v01], -1).reshape(-1, 3)])
    tris = tris.astype(np.int32)
    V = n * n
    ea, eb, ptr, nbr, _ = O.edges(tris.astype(np.int64), V)
    assert ea.shape[0] == 3 * V > 2 ** 24
    t = torch.from_numpy(tris)
    gea, geb, gptr, gnbr = _edges(t, V)
    assert np.array_equal(gea.numpy(), ea) and np.array_equal(geb.numpy(), eb)
    assert np.array_equal(gptr.numpy(), ptr) and np.array_equal(gnbr.numpy(), nbr)
    del gea, geb, gptr, gnbr, ea, eb, nbr
    vptr, vt = O.vertex_triangles(tris.astype(np.int64), V)
    gptr, gvt = _vertex_triangles(t, V)
    assert np.array_equal(gptr.numpy(), vptr) and np.array_equal(gvt.numpy(), vt)
