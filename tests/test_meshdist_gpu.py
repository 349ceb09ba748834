"""GPU: nero_meshdist_query against oracle/nero_oracle_meshdist.py bit for bit (dist, tri, closest point) on marching-cubes
meshes, a mesh seeded with degenerate triangles and a 1 M-triangle torus, with and without max_dist; closed-form cases
(a cube against its 1.01 scaling, a plane); properties (vertex bound, self distance, triangle order, determinism); compare()
and tools/compare_meshes.py end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_mesh as OMesh
import nero_oracle_meshdist as OD
from nero_b200 import evaluate as E
from nero_b200 import meshdist as MD
from nero_b200 import ops

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _mc(field, n=24):
    ax = np.linspace(-1.0, 1.0, n)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    v, t = OMesh.marching_cubes(field(x).astype(np.float32), 0.0)
    return (v * (2.0 / (n - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def sphere():
    return _mc(lambda x: np.linalg.norm(x, axis=-1) - 0.6 + 0.05 * np.sin(6 * x[..., 0]))


def torus():
    return _mc(lambda x: np.hypot(np.hypot(x[..., 0], x[..., 1]) - 0.55, x[..., 2]) - 0.22, 28)


def degenerate():
    """The sphere plus zero-area triangles: repeated indices, exactly and nearly collinear vertices and vertices repeated at
    one position."""
    v, t = sphere()
    V = v.shape[0]
    rng = np.random.RandomState(4)
    i = rng.randint(0, V, (40, 2))
    line = np.concatenate([v[:20], v[:20] + 0.25 * (v[20:40] - v[:20]), v[:20] + 0.5 * (v[20:40] - v[:20])]).astype(np.float32)
    dup = v[40:60].copy()
    x = rng.randint(-8, 8, (10, 1)) / 16.0
    axis = np.concatenate([np.concatenate([x + 0.25 * k, np.zeros((10, 1)), x / 2], 1) for k in range(3)]).astype(np.float32)
    W = V + 80
    extra = np.concatenate([np.stack([W + np.arange(10), W + 20 + np.arange(10), W + 10 + np.arange(10)], 1),
                            np.stack([i[:, 0], i[:, 0], i[:, 1]], 1), np.stack([i[:, 0], i[:, 1], i[:, 0]], 1),
                            np.stack([V + np.arange(20), V + 20 + np.arange(20), V + 40 + np.arange(20)], 1),
                            np.stack([40 + np.arange(20), V + 60 + np.arange(20), 41 + np.arange(20)], 1)])
    vv = np.concatenate([v, line, dup, axis]).astype(np.float32)
    tt = np.concatenate([t, extra]).astype(np.int32)
    perm = rng.permutation(tt.shape[0])                 # spread the degenerate triangles over the BVH
    return vv, tt[perm]


def torus_grid(n, R=0.5, r=0.2):
    u = np.arange(n) * (2 * np.pi / n)
    U, W = np.meshgrid(u, u, indexing='ij')
    v = np.stack([(R + r * np.cos(W)) * np.cos(U), (R + r * np.cos(W)) * np.sin(U), r * np.sin(W)], -1).reshape(-1, 3).astype(np.float32)
    i, j = np.meshgrid(np.arange(n), np.arange(n), indexing='ij')
    a, b, c, d = i * n + j, ((i + 1) % n) * n + j, ((i + 1) % n) * n + (j + 1) % n, i * n + (j + 1) % n
    t = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    return v, t


def queries(v, t, n_random, seed, far=8, vertices=64, edges=64, centroids=64, faces=64):
    """Random points in twice the bounding box, vertices, edge midpoints, centroids, points 10^3 away and points exactly
    on faces of BVH node boxes."""
    rng = np.random.RandomState(seed)
    lo, hi = v.min(0).astype(np.float64), v.max(0).astype(np.float64)
    mid, half = (lo + hi) / 2, (hi - lo) / 2
    vd = v.astype(np.float64)
    tt = t[rng.randint(0, t.shape[0], max(edges, centroids))]
    parts = [mid + (rng.rand(n_random, 3) * 2 - 1) * 2 * half, vd[rng.randint(0, v.shape[0], vertices)],
             (vd[tt[:edges, 0]] + vd[tt[:edges, 1]]) / 2, (vd[tt[:centroids, 0]] + vd[tt[:centroids, 1]] + vd[tt[:centroids, 2]]) / 3]
    d = rng.randn(far, 3)
    parts.append(mid + 1e3 * d / np.linalg.norm(d, axis=1, keepdims=True))
    nodes = ops.bvh_build(v, t)[0].view(np.float32).reshape(-1, 8)
    nd = nodes[rng.randint(0, nodes.shape[0], faces)].astype(np.float64)
    p = nd[:, :3] + rng.rand(faces, 3) * (nd[:, 4:7] - nd[:, :3])
    ax = rng.randint(0, 3, faces)
    side = rng.randint(0, 2, faces)
    p[np.arange(faces), ax] = np.where(side == 0, nd[np.arange(faces), ax], nd[np.arange(faces), 4 + ax])
    parts.append(p)
    return np.concatenate(parts)


def check_oracle(v, t, p, max_dist=np.inf):
    md = MD.MeshDistance(v, t)
    d, tri, q = (x.cpu().numpy() for x in md.query(p, max_dist=max_dist, closest=True))
    od, otri, oq = OD.query(p, v, t, max_dist)
    assert np.array_equal(tri, otri), np.flatnonzero(tri != otri)[:10]
    assert np.array_equal(d, od)
    assert np.array_equal(q, oq, equal_nan=True)
    return d, tri


@pytest.mark.parametrize('mesh', [sphere, torus, degenerate])
def test_bit_exact_against_the_oracle(mesh):
    v, t = mesh()
    p = queries(v, t, 512, seed=1)
    d, tri = check_oracle(v, t, p)
    assert (tri >= 0).all() and np.isfinite(d).all()
    md = float(np.median(d))
    d2, tri2 = check_oracle(v, t, p, max_dist=md)
    assert ((tri2 == -1) == (d > md)).all() and (d2[tri2 >= 0] == d[tri2 >= 0]).all() and (d2[tri2 < 0] == np.inf).all()


def test_bit_exact_on_equidistant_ties():
    """Vertices of a grid shared by six triangles each (exact ties, resolved to the lowest index), and points half way
    between two nested copies of the grid."""
    v, t = torus_grid(24)
    v2 = np.concatenate([v, v * np.float32(1.25)])
    t2 = np.concatenate([t, t + v.shape[0]])
    p = v.astype(np.float64) * 1.125
    check_oracle(v2, t2, np.concatenate([p, v.astype(np.float64)]))


def test_bit_exact_on_a_million_triangles():
    v, t = torus_grid(708)
    assert t.shape[0] > 1_000_000
    rng = np.random.RandomState(3)
    near = E.sample_surface(v, t, 160, seed=5).cpu().numpy() + rng.randn(160, 3) * 0.01
    p = np.concatenate([near, queries(v, t, 8, seed=2, far=2, vertices=8, edges=8, centroids=8, faces=8)])
    check_oracle(v, t, p)
    check_oracle(v, t, p[:64], max_dist=0.004)


def cube(s=1.0):
    c = np.asarray([[x, y, z] for x in (-s, s) for y in (-s, s) for z in (-s, s)], np.float32)
    f = []
    for ax in range(3):
        for sign in (0, 1):
            idx = [i for i in range(8) if ((i >> (2 - ax)) & 1) == sign]
            a, b, cc, d = idx[0], idx[1], idx[3], idx[2]
            f += [[a, b, cc], [a, cc, d]]
    return c, np.asarray(f, np.int32)


def test_cube_against_its_scaling_in_closed_form():
    v, t = cube(1.0)
    sv, st = cube(1.01)
    p = E.sample_surface(sv, st, 200000, seed=3)
    d = MD.MeshDistance(v, t).query(p)[0].cpu().numpy()
    pn = p.cpu().numpy()
    exact = np.linalg.norm(np.maximum(np.abs(pn) - 1.0, 0.0), axis=1)       # face, edge and corner regions
    assert np.abs(d - exact).max() <= 1e-12
    assert (np.abs(pn).max(1) - 1.0 > 0.0099).all()
    g = E.sample_surface(v, t, 100000, seed=4)
    dg = MD.MeshDistance(sv, st).query(g)[0].cpu().numpy()
    assert np.abs(dg - (np.float32(1.01) - 1.0)).max() <= 1e-12


def test_plane_distance_is_the_height():
    n = 65
    ax = np.linspace(-1, 1, n, dtype=np.float32)
    X, Y = np.meshgrid(ax, ax, indexing='ij')
    v = np.stack([X, Y, np.zeros_like(X)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing='ij')
    a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
    t = np.concatenate([np.stack([a, b, c], -1).reshape(-1, 3), np.stack([a, c, d], -1).reshape(-1, 3)]).astype(np.int32)
    rng = np.random.RandomState(8)
    p = np.concatenate([rng.uniform(-0.99, 0.99, (20000, 2)), rng.randn(20000, 1)], 1)
    dist, tri, q = (x.cpu().numpy() for x in MD.MeshDistance(v, t).query(p, closest=True))
    assert np.abs(dist - np.abs(p[:, 2])).max() <= 1e-15
    assert np.abs(q[:, :2] - p[:, :2]).max() <= 1e-15 and (q[:, 2] == 0).all()


@pytest.mark.parametrize('mesh', [sphere, degenerate])
def test_properties(mesh):
    v, t = mesh()
    md = MD.MeshDistance(v, t)
    p = queries(v, t, 4096, seed=9)
    pt = torch.from_numpy(p).cuda()
    d, tri = md.query(pt)
    used = torch.from_numpy(np.unique(t)).cuda().long()
    vd = E.nearest_dist_cuda(pt, md.verts[used]).double()
    assert bool((d <= vd * (1 + 1e-6) + 1e-7).all())                      # a vertex is a point of the mesh
    s = E.sample_surface(v, t, 20000, seed=2)
    assert float(md.query(s)[0].max()) <= 1e-12                            # samples of the mesh lie on it
    rng = np.random.RandomState(1)
    perm = rng.permutation(t.shape[0])
    d1, tri1 = md.query(pt)
    d2, tri2 = MD.MeshDistance(v, t[perm]).query(pt)
    assert torch.equal(d1, d2)
    tri1, back = tri1.cpu().numpy(), perm[tri2.cpu().numpy()]
    # the ids agree after remapping, except on ties (a closest point on a shared vertex or edge), where each order keeps
    # its own lowest index of equally distant triangles
    tie = np.flatnonzero(tri1 != back)
    vd64 = v.astype(np.float64)
    d2_of = lambda ids: OD.triangle_d2(p[tie], *(vd64[t[ids, k]] for k in range(3)))
    assert np.array_equal(d2_of(tri1[tie]), d2_of(back[tie])) and (tri1[tie] < back[tie]).all()
    assert tie.size < p.shape[0] // 2
    a, b = md.query(pt, closest=True), md.query(pt, closest=True)
    assert all(x.cpu().numpy().tobytes() == y.cpu().numpy().tobytes() for x, y in zip(a, b))


def test_query_argument_errors():
    v, t = sphere()
    md = MD.MeshDistance(v, t)
    with pytest.raises(ValueError, match='max_dist'):
        md.query(np.zeros((2, 3)), max_dist=-1.0)
    with pytest.raises(ValueError, match='max_dist'):
        md.query(np.zeros((2, 3)), max_dist=float('nan'))
    with pytest.raises(ValueError, match=r'\[n,3\]'):
        md.query(np.zeros((2, 2)))
    with pytest.raises(ValueError, match='finite'):
        md.query(np.asarray([[0.0, np.nan, 0.0]]))
    d, tri = md.query(np.zeros((0, 3)))
    assert d.shape == (0,) and tri.shape == (0,)


def test_compare_a_mesh_with_itself_and_the_cube_pair():
    v, t = sphere()
    m = MD.compare(v, t, v, t, samples=20000, seed=3)
    assert all(r['fscore'] == 1.0 for r in m['thresholds'])
    assert m['hausdorff'] <= 1e-12 and m['samples'] == 20000 and m['seed'] == 3
    cv, ct = cube(1.0)
    sv, st = cube(1.01)
    N = 200000
    taus = (0.0099, 0.01 + 1e-9, 0.02)
    m = MD.compare(sv, st, cv, ct, samples=N, seed=0, thresholds=taus)
    p0, p1, p2 = (r['precision'] for r in m['thresholds'])
    r0, r1, r2 = (r['recall'] for r in m['thresholds'])
    share = (1 / 1.01) ** 2                        # points of the larger cube's faces that project inside a face of the cube
    assert p0 == 0.0 and p2 == 1.0 and abs(p1 - share) <= 4 * np.sqrt(share * (1 - share) / N) + 1e-5
    assert (r0, r1, r2) == (0.0, 1.0, 1.0)
    assert abs(m['completeness']['mean'] - (np.float32(1.01) - 1.0)) <= 1e-12 and m['completeness']['max'] - m['completeness']['median'] <= 1e-12


def test_tool_end_to_end(tmp_path):
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    v, t = sphere()
    gv, gt = torus()
    pr, gtp = str(tmp_path / 'a.ply'), str(tmp_path / 'b.ply')
    write_ply(pr, v, t)
    write_ply(gtp, gv, gt)
    e, js = str(tmp_path / 'e.ply'), str(tmp_path / 'm.json')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compare_meshes.py'), '--pr', pr, '--gt', gtp, '--samples', '5000',
                        '--threshold', '0.05', '0.1', '--errors', e, '--json', js], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    printed = dict(ln.split(' ', 1) for ln in r.stdout.splitlines())
    m = json.load(open(js))
    ref = MD.compare(v, t, gv, gt, samples=5000, seed=0, thresholds=(0.05, 0.1))
    for k in ('chamfer', 'hausdorff', 'accuracy', 'completeness', 'thresholds'):
        assert m[k] == ref[k], k
    assert float(printed['chamfer']) == ref['chamfer'] and float(printed['fscore@0.05']) == ref['thresholds'][0]['fscore']
    ev, et = read_ply(e)
    assert np.array_equal(ev, v) and np.array_equal(et, t)
    d = MD.MeshDistance(gv, gt).query(v.astype(np.float64))[0].cpu().numpy()
    raw = open(e, 'rb').read().split(b'end_header\n', 1)[1]
    dt = np.dtype([('p', '<f4', (3,)), ('c', 'u1', (3,)), ('q', '<f4')])
    rec = np.frombuffer(raw[:dt.itemsize * v.shape[0]], dt)
    assert np.array_equal(rec['c'], MD.error_colors(d, 0.05)) and np.array_equal(rec['q'], d.astype(np.float32))
    s = np.minimum(d / 0.05, 1.0)
    assert np.array_equal(rec['c'][:, 0], np.floor(255 * s + 0.5).astype(np.uint8)) and (rec['c'][:, 1] == 0).all()
