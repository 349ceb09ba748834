"""CPU: the point-to-triangle convention of include/nero_meshdist.h in oracle/nero_oracle_meshdist.py (hand-derived closest
points in the seven Voronoi regions and on degenerate triangles, the tie rule, max_dist), the metric reduction, the
error-map colours, write_ply with colours and quality, argument errors and the header's exports."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_meshdist as OD
from nero_b200 import meshdist as MD

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

A, B, C = (0.0, 0.0, 0.0), (1.0, 0.0, 0.0), (0.0, 1.0, 0.0)


@pytest.mark.parametrize('p, q, region', [
    ((-1.0, -1.0, 0.5), A, 0),
    ((2.0, -0.5, 1.0), B, 1),
    ((-0.5, 2.0, 0.0), C, 2),
    ((0.5, -1.0, 2.0), (0.5, 0.0, 0.0), 3),
    ((-1.0, 0.25, -3.0), (0.0, 0.25, 0.0), 4),
    ((1.0, 1.0, 0.5), (0.5, 0.5, 0.0), 5),
    ((0.25, 0.25, 3.0), (0.25, 0.25, 0.0), 6),
])
def test_each_voronoi_region_gives_its_hand_derived_closest_point(p, q, region):
    got, reg = OD.closest_points(np.asarray([p]), np.asarray([A]), np.asarray([B]), np.asarray([C]))
    assert reg[0] == region
    assert np.array_equal(got[0], np.asarray(q))
    assert OD.triangle_d2(np.asarray([p]), np.asarray([A]), np.asarray([B]), np.asarray([C]))[0] == sum((x - y) ** 2 for x, y in zip(p, q))


@pytest.mark.parametrize('tri, p, q', [
    (((0, 0, 0), (0, 0, 0), (1, 0, 0)), (0.5, 1.0, 0.0), (0.5, 0.0, 0.0)),          # repeated vertex (zero-length edge)
    (((0, 0, 0), (1, 0, 0), (0, 0, 0)), (2.0, 0.0, 1.0), (1.0, 0.0, 0.0)),
    (((0, 0, 0), (1, 0, 0), (2, 0, 0)), (1.5, 1.0, 0.0), (1.5, 0.0, 0.0)),          # collinear, the middle vertex first
    (((2, 0, 0), (0, 0, 0), (1, 0, 0)), (-1.0, 0.0, 0.0), (0.0, 0.0, 0.0)),         # collinear, the middle vertex last
    (((1, 2, 3), (1, 2, 3), (1, 2, 3)), (0.0, 0.0, 0.0), (1.0, 2.0, 3.0)),          # all three vertices the same
    (((0, 0, 0), (0.5, 0.5, 0.5), (1, 1, 1)), (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)),    # collinear, the point on it
])
def test_degenerate_triangles_are_their_edge_segments(tri, p, q):
    a, b, c = (np.asarray([v], np.float64) for v in tri)
    got, reg = OD.closest_points(np.asarray([p]), a, b, c)
    assert reg[0] == 7 and np.array_equal(got[0], np.asarray(q))


def test_no_nan_on_random_degenerate_triangles():
    rng = np.random.RandomState(5)
    a = rng.randint(-3, 4, (4000, 3)).astype(np.float32).astype(np.float64)
    d = rng.randint(-2, 3, (4000, 3)).astype(np.float64)
    b, c = a + d, a + 2 * d * rng.randint(0, 3, (4000, 1))                  # collinear or repeated vertices
    p = rng.randn(4000, 3) * 3
    q, reg = OD.closest_points(p, a, b, c)
    assert np.isfinite(q).all() and (reg == 7).all()
    seg = np.stack([np.linalg.norm(p - x, axis=1) for x in (a, b, c)], 1).min(1)
    assert (np.sqrt(OD.triangle_d2(p, a, b, c)) <= seg * (1 + 1e-12)).all()


def test_random_points_match_an_independent_projection():
    """Away from degeneracy the routine is the exact closest point: compare with scipy's constrained least squares."""
    from scipy.optimize import lsq_linear
    rng = np.random.RandomState(11)
    for _ in range(200):
        a, b, c = rng.randn(3, 3)
        p = rng.randn(3) * 2
        q, _ = OD.closest_points(p[None], a[None], b[None], c[None])
        # the interior least-squares point when it lies in the triangle, else the best of the three clamped edge projections
        M = np.stack([b - a, c - a], 1)
        sol = lsq_linear(M, p - a, bounds=([0, 0], [1, 1]))
        cands = [a + M @ sol.x] if sol.x.sum() <= 1 else []
        for x, y in ((a, b), (a, c), (b, c)):
            e = y - x
            tt = np.clip(np.dot(p - x, e) / np.dot(e, e), 0, 1)
            cands.append(x + tt * e)
        best = min(cands, key=lambda r: np.linalg.norm(r - p))
        assert abs(np.linalg.norm(q[0] - p) - np.linalg.norm(best - p)) <= 1e-9


def test_query_takes_the_lowest_index_on_ties_and_honours_max_dist():
    v = np.asarray([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 2], [1, 0, 2], [0, 1, 2]], np.float32)
    t = np.asarray([[3, 4, 5], [0, 1, 2], [0, 2, 1]], np.int32)
    p = np.asarray([[0.25, 0.25, 1.0], [0.25, 0.25, 0.5], [0.25, 0.25, -4.0]])
    d, tri, q = OD.query(p, v, t)
    assert tri.tolist() == [0, 1, 1] and d.tolist() == [1.0, 0.5, 4.0]
    assert np.array_equal(q, [[0.25, 0.25, 2.0], [0.25, 0.25, 0.0], [0.25, 0.25, 0.0]])
    d, tri, q = OD.query(p, v, t, max_dist=1.0)
    assert tri.tolist() == [0, 1, -1] and d[2] == np.inf and np.isnan(q[2]).all()


def test_metrics_reduce_the_two_distance_arrays():
    rng = np.random.RandomState(2)
    acc, comp = rng.exponential(0.002, 10001), rng.exponential(0.003, 7777)
    m = MD.metrics(acc, comp, (0.001, 0.004))
    for name, d in (('accuracy', acc), ('completeness', comp)):
        s = m[name]
        assert s['mean'] == np.mean(d) and s['median'] == np.median(d) and s['max'] == d.max()
        assert s['rms'] == np.sqrt(np.mean(d * d))
        assert [s['p90'], s['p95'], s['p99']] == list(np.percentile(d, [90, 95, 99]))
    assert m['chamfer'] == (np.mean(acc) + np.mean(comp)) / 2 and m['hausdorff'] == max(acc.max(), comp.max())
    for row, t in zip(m['thresholds'], (0.001, 0.004)):
        P, R = (acc < t).sum() / acc.size, (comp < t).sum() / comp.size
        assert row['threshold'] == t and row['precision'] == P and row['recall'] == R
        assert abs(row['fscore'] - 2 * P * R / (P + R)) <= 1e-15
    zero = MD.metrics([1.0, 2.0], [3.0], (0.5,))['thresholds'][0]
    assert zero == {'threshold': 0.5, 'precision': 0.0, 'recall': 0.0, 'fscore': 0.0}
    exact = MD.metrics([0.0, 0.0, 1.0, 1.0], [0.0, 1.0], (0.5,))
    assert exact['thresholds'][0]['precision'] == 0.5 and exact['thresholds'][0]['recall'] == 0.5
    assert exact['thresholds'][0]['fscore'] == 0.5 and exact['accuracy']['p90'] == 1.0 and exact['accuracy']['median'] == 0.5


def test_error_colour_ramp():
    t = 0.004
    d = np.asarray([0.0, t / 2, t, 2 * t, np.inf, t / 255, 3 * t / 4])
    got = MD.error_colors(d, t)
    assert got.dtype == np.uint8
    assert got.tolist() == [[0, 0, 255], [128, 0, 128], [255, 0, 0], [255, 0, 0], [255, 0, 0], [1, 0, 254], [191, 0, 64]]


def test_write_ply_with_colours_and_quality_reads_back(tmp_path):
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    rng = np.random.RandomState(1)
    v = rng.randn(50, 3).astype(np.float32)
    t = rng.randint(0, 50, (70, 3)).astype(np.int32)
    plain = str(tmp_path / 'plain.ply')
    write_ply(plain, v, t)
    face = np.empty(70, dtype=[('n', 'u1'), ('v', '<i4', (3,))])
    face['n'], face['v'] = 3, t
    header = ('ply\nformat binary_little_endian 1.0\nelement vertex 50\nproperty float x\nproperty float y\nproperty float z\n'
              'element face 70\nproperty list uchar int vertex_indices\nend_header\n').encode('ascii')
    assert open(plain, 'rb').read() == header + v.tobytes() + face.tobytes()
    col = rng.randint(0, 256, (50, 3)).astype(np.uint8)
    q = rng.rand(50)
    for kw in ({'colors': col}, {'quality': q}, {'colors': col, 'quality': q}):
        path = str(tmp_path / f'{"_".join(kw)}.ply')
        write_ply(path, v, t, **kw)
        rv, rt = read_ply(path)
        assert np.array_equal(rv, v) and np.array_equal(rt, t)
        raw = open(path, 'rb').read()
        head, body = raw.split(b'end_header\n', 1)
        props = [ln.split()[-1] for ln in head.decode().splitlines() if ln.startswith('property') and 'list' not in ln]
        assert props == ['x', 'y', 'z'] + (['red', 'green', 'blue'] if 'colors' in kw else []) + (['quality'] if 'quality' in kw else [])
        dt = np.dtype([('p', '<f4', (3,))] + ([('c', 'u1', (3,))] if 'colors' in kw else []) + ([('q', '<f4')] if 'quality' in kw else []))
        rec = np.frombuffer(body[:dt.itemsize * 50], dt)
        assert np.array_equal(rec['p'], v)
        if 'colors' in kw:
            assert np.array_equal(rec['c'], col)
        if 'quality' in kw:
            assert np.array_equal(rec['q'], q.astype(np.float32))
    with pytest.raises(ValueError, match='colors'):
        write_ply(plain, v, t, colors=col.astype(np.int32))
    with pytest.raises(ValueError, match='quality'):
        write_ply(plain, v, t, quality=q[:10])


def test_argument_errors():
    with pytest.raises(ValueError, match='non-empty'):
        MD.metrics([], [1.0])
    with pytest.raises(ValueError, match='thresholds'):
        MD.metrics([1.0], [1.0], (0.0,))
    with pytest.raises(ValueError, match='threshold'):
        MD.error_colors([1.0], float('nan'))
    with pytest.raises(ValueError, match='MeshDistance'):
        MD.MeshDistance(np.zeros((4, 3), np.float32), np.zeros((2, 4), np.int32))
    with pytest.raises(ValueError, match='out of range'):
        MD.MeshDistance(np.zeros((4, 3), np.float32), np.asarray([[0, 1, 4]], np.int32))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    tool = os.path.join(ROOT, 'tools', 'compare_meshes.py')
    r = subprocess.run([sys.executable, tool, '--pr', '/nonexistent/a.ply', '--gt', '/nonexistent/b.ply'], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and 'does not exist' in r.stderr
    r = subprocess.run([sys.executable, tool, '--help'], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'not tuned' in r.stdout


def test_library_exports_every_symbol_of_the_meshdist_header():
    import __graft_entry__ as g
    lib = ctypes.CDLL(g.build())
    txt = open(os.path.join(ROOT, 'include', 'nero_meshdist.h')).read()
    syms = sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))
    assert syms == ['nero_meshdist_query']
    assert hasattr(lib, syms[0])
    from nero_b200 import ops
    fn = ops.lib.nero_meshdist_query
    assert len(fn.argtypes) == len(ops.MESHDIST_PROTOS['nero_meshdist_query']) == 12
    buf = ctypes.c_void_p(16)
    assert fn(buf, -1, buf, buf, buf, buf, 1.0, buf, buf, None, buf, None) == 1                 # n < 0
    assert fn(buf, 4, buf, buf, buf, buf, float('nan'), buf, buf, None, buf, None) == 1         # max_dist NaN
    assert fn(buf, 4, buf, buf, buf, buf, -1.0, buf, buf, None, buf, None) == 1                 # max_dist < 0
    assert fn(buf, 4, None, buf, buf, buf, 1.0, buf, buf, None, buf, None) == 1                 # no nodes
    assert fn(buf, 4, buf, buf, buf, buf, 1.0, buf, buf, None, None, None) == 1                 # no status word
    assert fn(None, 0, None, None, None, None, float('inf'), None, None, None, None, None) == 0  # nothing to do
