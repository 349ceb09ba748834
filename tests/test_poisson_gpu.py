"""Screened Poisson reconstruction on the GPU: every kernel of k_poisson.cu and the first PCG iterates against
oracle/nero_oracle_poisson.py bit for bit, the converged solution against scipy's direct solve, the geometry of spheres,
tori, noisy and half-sampled clouds, run-to-run identity, argument checks before any launch, and dense_points.py --normals
-> poisson_mesh.py -> compare_meshes.py end to end on the synthetic table / box / sphere project."""
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

import nero_oracle_mvs as OM
import nero_oracle_poisson as OP
from nero_b200 import ops, poisson as P
from nero_b200.evaluate import nearest_dist_cuda, read_oriented_points_ply, read_points_ply
from nero_b200.mesh import marching_cubes_cuda

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def host(t):
    return t.cpu().numpy()


def grid_cloud(N, kind, seed):
    """Samples in grid units (origin 0, h 1): random or clustered, with points on cell faces, edges and corners, on the grid
    boundary and outside it (clamped)."""
    rng = np.random.RandomState(seed)
    if kind == 'random':
        p = rng.uniform(0, N - 1, (3000, 3))
    else:
        c = rng.uniform(2, N - 3, (6, 3))
        p = c[rng.randint(0, 6, 3000)] + rng.randn(3000, 3) * 0.7
    faces = rng.uniform(0, N - 1, (200, 3))
    faces[:, 0] = np.round(faces[:, 0])                       # on x faces
    faces[100:, 1] = np.round(faces[100:, 1])                 # on edges
    corners = rng.randint(0, N, (40, 3)).astype(np.float64)   # on nodes, the grid boundary included
    border = rng.uniform(0, N - 1, (60, 3))
    border[:20, 0], border[20:40, 1], border[40:, 2] = 0.0, N - 1.0, -0.3    # on the boundary faces and just outside
    p = np.concatenate([p, faces, corners, border])
    nrm = rng.randn(p.shape[0], 3)
    return p, (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize('N', [17, 33])
@pytest.mark.parametrize('kind', ['random', 'clustered'])
def test_kernels_match_oracle_bit_for_bit(N, kind):
    p, nrm = grid_cloud(N, kind, N)
    n = p.shape[0]
    q = torch.empty(n, 3, dtype=torch.float32, device='cuda')
    keys = torch.empty(n, dtype=torch.int32, device='cuda')
    ops.K('nero_poisson_keys', cuda(p), n, 0.0, 0.0, 0.0, 1.0, N, q, keys)
    oq, okeys = OP.keys(p, np.zeros(3), 1.0, N)
    assert np.array_equal(host(q), oq) and np.array_equal(host(keys), okeys)
    sk, order = torch.sort(keys, stable=True)
    oorder = np.argsort(okeys, kind='stable')
    assert np.array_equal(host(order), oorder)
    q, g_nrm = q[order].contiguous(), cuda(nrm)[order].contiguous()
    oq, onrm = oq[oorder], nrm[oorder]
    cells = (N - 1) ** 3
    start = torch.empty(cells + 1, dtype=torch.int32, device='cuda')
    ops.K('nero_poisson_cell_starts', sk, n, cells, start)
    ostart = OP.cell_starts(okeys[oorder], cells)
    assert np.array_equal(host(start), ostart)
    sigma = np.float32(2.75)
    E = (N - 1) * N * N
    v = [torch.empty(E, dtype=torch.float32, device='cuda') for _ in range(3)]
    ops.K('nero_poisson_edge_splat', q, g_nrm, n, start, N, float(sigma), *v)
    ov = OP.edge_splat(oq, onrm, ostart, N, sigma)
    for a in range(3):
        assert np.array_equal(host(v[a]), ov[a]), f'edge lattice {a}'
    b = torch.empty(N ** 3, dtype=torch.float32, device='cuda')
    ops.K('nero_poisson_rhs', *v, N, b)
    assert np.array_equal(host(b), OP.rhs(*ov, N))
    dens, diag = torch.empty_like(b), torch.empty_like(b)
    ops.K('nero_poisson_node_splat', q, n, start, N, dens, diag)
    od, odiag = OP.node_splat(oq, ostart, N)
    assert np.array_equal(host(dens), od) and np.array_equal(host(diag), odiag)
    rng = np.random.RandomState(7)
    x = rng.randn(N ** 3).astype(np.float32)
    y, sx = torch.empty_like(b), torch.empty(n, dtype=torch.float32, device='cuda')
    ws = np.float32(0.37)
    ops.K('nero_poisson_matvec', cuda(x), N, q, n, start, float(ws), sx, y)
    assert np.array_equal(host(sx), OP.interp(x, N, oq)) and np.array_equal(host(y), OP.matvec(x, N, oq, ostart, ws))
    bb = rng.randn(N ** 3).astype(np.float32)
    d = np.abs(rng.randn(N ** 3)).astype(np.float32)
    for colour in (0, 1):
        for s in (1.0, 4.0):
            gx = cuda(x)
            ops.K('nero_poisson_smooth', gx, cuda(bb), cuda(d), N, s, colour)
            assert np.array_equal(host(gx), OP.smooth(x, bb, d, N, s, colour)), f'colour {colour}, s {s}'
    r = torch.empty_like(b)
    ops.K('nero_poisson_residual', cuda(x), cuda(bb), cuda(d), N, 2.0, r)
    assert np.array_equal(host(r), OP.residual(x, bb, d, N, 2.0))
    Nc = (N - 1) // 2 + 1
    c = torch.empty(Nc ** 3, dtype=torch.float32, device='cuda')
    ops.K('nero_poisson_restrict', cuda(x), N, c)
    assert np.array_equal(host(c), OP.restrict(x, N))
    xc = rng.randn(Nc ** 3).astype(np.float32)
    f = cuda(bb)
    ops.K('nero_poisson_prolong', cuda(xc), Nc, f)
    assert np.array_equal(host(f), OP.prolong(xc, Nc, bb))
    be = P._Cuda(N, q, start, ws)
    assert be.total(cuda(x), cuda(bb)) == OP.total(x, bb) and be.total(cuda(x)) == OP.total(x)
    blocks = ops.ceil_div(N ** 3, 256)
    part = torch.empty(blocks, dtype=torch.float64, device='cuda')
    ops.K('nero_poisson_dot', cuda(x), cuda(bb), N ** 3, part)
    assert np.array_equal(host(part), OP.OA.block_partials((x.astype(np.float64) * bb.astype(np.float64))[:, None])[:, 0])
    gx, gr = cuda(x), cuda(bb)
    ops.K('nero_poisson_update', gx, gr, cuda(d), cuda(xc[:1].repeat(N ** 3)), 0.3, N ** 3)
    assert np.array_equal(host(gx), x + np.float32(0.3) * d) and np.array_equal(host(gr), bb - np.float32(0.3) * xc[0])
    ops.K('nero_poisson_direction', gx, cuda(d), -1.7, N ** 3)
    assert np.array_equal(host(gx), d + np.float32(-1.7) * (x + np.float32(0.3) * d))


def sphere(n, r=0.35, seed=0):
    rng = np.random.RandomState(seed)
    d = rng.randn(n, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * r, d


def torus(n, R=0.3, r=0.12, seed=0):
    """Area-uniform samples of a torus about z and their outward normals."""
    rng = np.random.RandomState(seed)
    u = rng.uniform(0, 2 * np.pi, 4 * n)
    v = rng.uniform(0, 2 * np.pi, 4 * n)
    keep = rng.uniform(0, 1, 4 * n) < (R + r * np.cos(v)) / (R + r)
    u, v = u[keep][:n], v[keep][:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    return np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], 1), nrm


@pytest.mark.parametrize('kind', ['sphere', 'clustered'])
def test_setup_and_first_pcg_iterates_match_oracle(kind):
    if kind == 'sphere':
        p, nrm = sphere(4000)
    else:
        p, nrm = grid_cloud(33, 'clustered', 1)
        p = p * 0.01
    p, nrm = P.check_inputs(p, nrm, 33)
    S = P.setup(p, nrm, 33)
    O = OP.setup(p, nrm, 33)
    for k in ('q', 'nrm', 'keys', 'start', 'b', 'density', 'diag'):
        assert np.array_equal(host(S[k]), O[k]), k
    assert S['occupied'] == O['occupied'] and S['ws'] == O['ws'] and S['sigma32'] == O['sigma32']
    for a in range(3):
        assert np.array_equal(host(S['v'][a]), O['v'][a])
    be = P._Cuda(33, S['q'], S['start'], S['ws'])
    L = P.hierarchy(be, 33, S['diag'], S['ws'])
    OL = OP.hierarchy(33, O['diag'], O['ws'])
    for lv, olv in zip(L, OL):
        assert lv['N'] == olv['N'] and np.array_equal(host(lv['d']), olv['d'])
    gtr, otr = [], []
    P.pcg(be, L, S['b'], 1e-30, 3, gtr)
    OP.solve(O, 33, 1e-30, 3, otr)
    assert len(gtr) == len(otr) == 3
    for g, o in zip(gtr, otr):
        for k in ('x', 'r', 'p'):
            assert np.array_equal(g[k], o[k]), k
        for k in ('alpha', 'beta', 'rz', 'pap'):
            assert g[k] == o[k], k


def test_converged_solution_matches_scipy():
    p, nrm = sphere(20000, seed=1)
    trace = {}
    P.reconstruct(p, nrm, 33, tol=1e-6, max_iters=100, trace=trace)
    Sh = {k: (host(v) if torch.is_tensor(v) else v) for k, v in trace.items() if k in ('q', 'ws', 'v')}
    Sh['v'] = [host(a) for a in trace['v']]
    chi = OP.exact(Sh, 33)
    err = np.abs(host(trace['chi']).astype(np.float64) - chi).max() / np.abs(chi).max()
    print(f'max |chi - exact| / max |exact| = {err:.2e}')
    assert err <= 1e-4


def topology(verts, tris):
    """(components, every edge in exactly two triangles, Euler characteristic)."""
    t = np.asarray(tris, np.int64)
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    import scipy.sparse as sp
    import scipy.sparse.csgraph as cg
    V = verts.shape[0]
    A = sp.coo_matrix((np.ones(e.shape[0]), (e[:, 0], e[:, 1])), shape=(V, V))
    ncomp = cg.connected_components(A, directed=False)[0] - (V - np.unique(t).size)
    return ncomp, bool((cnt == 2).all()), V - cnt.size + t.shape[0]


def outward(verts, tris):
    """(centroids, outward unit face normals) for the project's winding (cross(e1, e2) points inside)."""
    v = np.asarray(verts, np.float64)[np.asarray(tris, np.int64)]
    c = -np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    return v.mean(1), c / np.linalg.norm(c, axis=1, keepdims=True)


def test_sphere_is_closed_and_accurate():
    p, nrm = sphere(100000, seed=2)
    v, t, info = P.reconstruct(p, nrm, 65)
    v, t = host(v), host(t)
    comps, manifold, euler = topology(v, t)
    d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.35) / info['h']
    print(f'{info["iterations"]} iterations, residual {info["history"][-1]:.2e}, {t.shape[0]} triangles, '
          f'mean |d| {d.mean():.4f} h, max {d.max():.4f} h')
    assert comps == 1 and manifold and euler == 2 and d.max() <= 0.25
    c, n = outward(v, t)
    assert (n * c / np.linalg.norm(c, axis=1, keepdims=True)).sum(1).mean() > 0.9
    ax = torch.linspace(-1, 1, 33, device='cuda')
    g = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), -1)
    sv, st = marching_cubes_cuda(torch.linalg.norm(g, dim=-1) - 0.6, 0.0)
    sc, sn = outward(host(sv) - 16.0, host(st))
    assert (sn * sc).sum(1).mean() > 0             # the SDF mesh is wound the same way


def test_torus_has_euler_characteristic_zero():
    p, nrm = torus(100000, seed=3)
    v, t, info = P.reconstruct(p, nrm, 65)
    comps, manifold, euler = topology(host(v), host(t))
    assert comps == 1 and manifold and euler == 0


def test_noisy_samples_stay_closed():
    p, nrm = sphere(100000, seed=4)
    h = 1.1 * 0.7 / 64
    rng = np.random.RandomState(5)
    pj = p + rng.randn(*p.shape) * 0.2 * h
    nj = nrm + rng.randn(*nrm.shape) * 0.2
    v, t, info = P.reconstruct(pj, nj, 65)
    v, t = host(v), host(t)
    comps, manifold, euler = topology(v, t)
    d = np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - 0.35) / info['h']
    print(f'noisy: mean |d| {d.mean():.4f} h, max {d.max():.4f} h')
    assert comps == 1 and manifold and euler == 2 and d.mean() <= 0.5


def area(v, t):
    x = np.asarray(v, np.float64)[np.asarray(t, np.int64)]
    return 0.5 * np.linalg.norm(np.cross(x[:, 1] - x[:, 0], x[:, 2] - x[:, 0]), axis=1)


def test_trim_removes_the_unsampled_cap():
    p, nrm = sphere(120000, seed=6)
    keep = p[:, 2] >= 0
    p, nrm = p[keep], nrm[keep]
    # the surface closing an open cloud bulges past it: a grid twice the bounding cube leaves it room
    v0, t0, i0 = P.reconstruct(p, nrm, 65, scale=2.0)
    comps, manifold, euler = topology(host(v0), host(t0))
    assert manifold and euler == 2
    v1, t1, i1 = P.reconstruct(p, nrm, 65, scale=2.0, trim=0.1)
    h = i1['h']
    samples = cuda(p.astype(np.float32))
    c1, _ = outward(host(v1), host(t1))
    d1 = host(nearest_dist_cuda(cuda(c1.astype(np.float32)), samples))
    c0, _ = outward(host(v0), host(t0))
    d0 = host(nearest_dist_cuda(cuda(c0.astype(np.float32)), samples))
    a0, a1 = area(host(v0), host(t0)), area(host(v1), host(t1))
    near0, near1 = a0[d0 <= h].sum(), a1[d1 <= h].sum()
    print(f'trim 0.1: {i1["triangles_before"]} -> {i1["triangles_after"]} triangles, farthest centroid {d1.max() / h:.3f} h, '
          f'area within h kept {near1 / near0:.4f}')
    assert i1['triangles_after'] < i1['triangles_before'] and i1['density'].shape[0] == v1.shape[0]
    # measured on an H100: the farthest kept centroid lies 3.31 h from a sample (the density is restricted to 4h, so it fades
    # over a few h past the rim), and all of the area within h of the samples is kept
    assert d1.max() <= 4 * h and near1 >= 0.99 * near0


def test_two_runs_are_identical():
    p, nrm = torus(30000, seed=7)
    a = P.reconstruct(p, nrm, 65, trim=0.05)
    b = P.reconstruct(p, nrm, 65, trim=0.05)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2]['history'] == b[2]['history']


def test_bad_inputs_raise_before_any_launch():
    p, nrm = sphere(100)
    cases = [(np.where(np.arange(300).reshape(100, 3) == 7, np.nan, p), nrm, 33), (p, np.where(np.arange(100)[:, None] == 3, 0.0, nrm), 33),
             (p[:15], nrm[:15], 33), (p, nrm, 64), (p, nrm[:50], 33)]
    for pp, nn, N in cases:
        before = ops.launch_count
        with pytest.raises(ValueError):
            P.reconstruct(pp, nn, N)
        assert ops.launch_count == before


@pytest.fixture(scope='module')
def scene(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('poisson_scene'))
    pr = OM.project(root, 8, 160, 120, seed=3)
    return root, pr


def test_dense_points_normals_then_poisson_mesh(scene, capsys):
    root, pr = scene
    plain, oriented = os.path.join(root, 'plain.ply'), os.path.join(root, 'oriented.ply')
    tool('dense_points').main(['--root', root, '--output', plain])
    tool('dense_points').main(['--root', root, '--output', oriented, '--normals'])
    pts = read_points_ply(plain)
    # the layout without --normals: Open3D's `double x y z`, byte for byte
    header = (f'ply\nformat binary_little_endian 1.0\ncomment Created by nero_b200\nelement vertex {pts.shape[0]}\n'
              'property double x\nproperty double y\nproperty double z\nend_header\n').encode('ascii')
    assert open(plain, 'rb').read() == header + np.ascontiguousarray(pts, '<f8').tobytes()
    opts, onrm = read_oriented_points_ply(oriented)
    assert np.array_equal(opts, pts) and np.abs(np.linalg.norm(onrm, axis=1) - 1).max() < 1e-6
    lo, hi = OM.object_bbox()
    pad = 0.02 * (hi - lo).max()
    mesh_out = os.path.join(root, 'mvs_mesh.ply')
    tool('poisson_mesh').main(['--points', oriented, '--out', mesh_out, '--resolution', '129', '--trim', '0.2',
                               '--crop-box', *map(str, np.concatenate([lo - pad, hi + pad]))])
    from nero_b200.material import read_ply
    v, t = read_ply(mesh_out)
    dist = OM.surface_distance(v)
    D = float(np.linalg.norm(hi - lo))
    print(capsys.readouterr().out)
    print(f'{t.shape[0]} triangles, vertex distance to the scene: median {np.median(dist) / D:.5f} D, '
          f'90th percentile {np.percentile(dist, 90) / D:.5f} D')
    assert t.shape[0] > 1000 and np.median(dist) <= 0.01 * D and np.percentile(dist, 90) <= 0.03 * D
    js = os.path.join(root, 'cmp.json')
    tool('compare_meshes').main(['--pr', mesh_out, '--gt', mesh_out, '--samples', '20000', '--json', js])
    m = json.load(open(js))
    assert isinstance(m, dict) and m
