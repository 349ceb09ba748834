"""CPU: the registration convention of include/nero_align.h and nero_b200/align.py in oracle/nero_oracle_align.py -- recovery
of a known similarity, the principal-axis start, rigid mode, undetermined rotations of a sphere and a torus, the pairwise
tree against an independent pairwise sum, degenerate triangles -- and argument errors, the header's exports and
tools/align_meshes.py's argument parsing."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_align as OA
import nero_oracle_mesh as OMesh
import nero_oracle_meshpts as OMp
from nero_b200 import align as A

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def mc(field, n):
    ax = np.linspace(-1.0, 1.0, n)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    v, t = OMesh.marching_cubes(field(x).astype(np.float32), 0.0)
    return (v * (2.0 / (n - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def blob_field(x):
    """Three unequal spheres and an ellipsoid: no symmetry, so every degree of freedom is determined."""
    sd = lambda c, r: np.linalg.norm(x - np.asarray(c), axis=-1) - r
    ell = (np.linalg.norm(x / np.asarray([0.55, 0.25, 0.3]), axis=-1) - 1.0) * 0.25
    return np.minimum.reduce([sd((0.35, 0.1, 0.0), 0.3), sd((-0.3, 0.25, 0.1), 0.22), sd((0.0, -0.3, 0.25), 0.18), ell])


def blob(n=32):
    return mc(blob_field, n)


def sphere(n=24):
    return mc(lambda x: np.linalg.norm(x, axis=-1) - 0.6, n)


def torus(n=28):
    return mc(lambda x: np.hypot(np.hypot(x[..., 0], x[..., 1]) - 0.55, x[..., 2]) - 0.22, n)


def similarity(s, axis, degrees, t):
    a = np.asarray(axis, np.float64)
    return A.matrix(s, A.rodrigues(a / np.linalg.norm(a) * np.radians(degrees)), np.asarray(t, np.float64))


def moved(v, T):
    """The vertices v mapped by the inverse of T, in float32: registering them to v must give T."""
    return OA.transform(v.astype(np.float64), A.inverse(T)[:3]).astype(np.float32)


def errors(M, T):
    """(rotation angle between the two, relative scale error, translation error) of two similarities."""
    s1, R1, t1 = A.decompose(M)
    s2, R2, t2 = A.decompose(T)
    c = np.clip((np.trace(R1.T @ R2) - 1) / 2, -1.0, 1.0)
    return float(np.arccos(c)), abs(s1 / s2 - 1), float(np.abs(t1 - t2).max())


def run(src_v, t, v, n=1024, **kw):
    pts = OMp.sample(src_v, t, n, seed=0)[0]
    tgt = OMp.sample(v, t, n, seed=1)[0]
    return OA.align(pts, v, t, tgt, **kw)


def test_oracle_recovers_a_known_similarity():
    v, t = blob()
    T = similarity(1.3, (1, 2, 3), 8.0, (0.05, -0.03, 0.02))
    res, b = run(moved(v, T), t, v, max_iters=30)
    rot, sc, tr = errors(res['matrix'], T)
    assert res['converged'] and rot < 1e-6 and sc < 1e-6 and tr < 1e-6
    assert res['undetermined'] == [] and len(res['tau']) == res['iterations'] == len(b.trace)
    assert all(b <= a for a, b in zip(res['tau'], res['tau'][1:])) and res['rms'][-1] < 1e-6
    assert res['tau'][-1] == A.TAU_MIN * res['length']


def test_auto_start_finds_a_quarter_and_a_half_turn():
    v, t = blob()
    T = similarity(2.5, (0, 0, 1), 90.0, (0.1, 0.2, -0.1)) @ similarity(1.0, (1, 0, 0), 180.0, (0, 0, 0))
    res, _ = run(moved(v, T), t, v, init='auto', max_iters=30, coarse=512)
    assert len(res['coarse_scores']) == 24 and res['coarse_best'] == int(np.argmin(res['coarse_scores']))
    rot, sc, tr = errors(res['matrix'], T)
    assert res['converged'] and rot < 1e-6 and sc < 1e-6 and tr < 1e-6
    res_id, _ = run(moved(v, T), t, v, max_distance=2.0, max_iters=5)
    assert errors(res_id['matrix'], T)[0] > 0.1                # the identity start is nowhere near


def test_rigid_mode_keeps_the_scale_exactly_one():
    v, t = blob()
    T = similarity(1.0, (2, -1, 1), 6.0, (0.03, 0.0, -0.02))
    res, _ = run(moved(v, T), t, v, rigid=True, max_iters=30)
    assert res['scale'] == 1.0 and res['matrix'][3, 3] == 1.0
    rot, _, tr = errors(res['matrix'], T)
    assert res['converged'] and rot < 1e-6 and tr < 1e-6
    res, _ = run(moved(v, similarity(1.1, (0, 0, 1), 2.0, (0, 0, 0))), t, v, rigid=True, init=np.diag([1.2, 1.2, 1.2, 1.0]), max_iters=3)
    assert res['scale'] == 1.0                                  # a user start's scale is dropped too


def test_a_sphere_leaves_three_rotations_and_a_torus_one_undetermined():
    v, t = sphere()
    T = similarity(1.05, (1, 1, 0), 0.0, (0.02, -0.01, 0.0))
    res, _ = run(moved(v, T), t, v, max_distance=0.3, max_iters=40)
    assert [u['kind'] for u in res['undetermined']] == ['rotation'] * 3
    assert np.isfinite(res['matrix']).all() and abs(res['scale'] / 1.05 - 1) < 2e-3
    centre = A.inverse(T)[:3, 3]                                # the source sphere's centre, mapped by the result
    assert np.abs(res['matrix'][:3, :3] @ centre + res['matrix'][:3, 3]).max() < 2e-3
    v, t = torus()
    T = similarity(1.1, (1, 0, 0), 5.0, (0.02, 0.0, 0.01))
    res, _ = run(moved(v, T), t, v, max_distance=0.3, max_iters=40)
    assert [u['kind'] for u in res['undetermined']] == ['rotation']
    axis = res['undetermined'][0]['vector'][:3]
    assert abs(abs(axis[2]) - 1) < 1e-2                         # free: the rotation about the torus' own axis
    s, R, _ = A.decompose(res['matrix'])
    s0, R0, _ = A.decompose(T)
    assert np.isfinite(res['matrix']).all() and abs(s / s0 - 1) < 2e-3 and np.abs(R[:, 2] - R0[:, 2]).max() < 2e-3
    assert np.abs(res['matrix'][:3, :3] @ A.inverse(T)[:3, 3] + res['matrix'][:3, 3]).max() < 2e-3


def pairwise(x):
    """An independent pairwise sum: the two halves summed recursively, then added."""
    if x.shape[0] == 1:
        return x[0]
    h = x.shape[0] // 2
    return pairwise(x[:h]) + pairwise(x[h:])


@pytest.mark.parametrize('n', [1, 255, 256, 1000, 70000])
def test_tree_reduction_equals_an_independent_pairwise_sum(n):
    rng = np.random.RandomState(n)
    x = rng.randn(n, 3) * np.exp(rng.randn(n, 1) * 8)         # wide dynamic range: the order shows in the last bits
    P = 1 << max(0, (n - 1).bit_length())
    pad = np.zeros((P, 3))
    pad[:n] = x
    got = OA.reduce(OA.block_partials(x)[None])[0]
    assert np.array_equal(got, pairwise(pad))
    assert np.array_equal(OA.block_partials(x)[0], pairwise(pad[:256]) if n >= 256 else pairwise(np.concatenate([x, np.zeros((256 - n, 3))])))
    k = 3
    d = np.abs(rng.randn(k * n)) * np.where(rng.rand(k * n) < 0.1, np.inf, 1.0)
    s = OA.reduce(OA.score_partials(d, k, 0.7)[:, :, None])[:, 0]
    for j in range(k):
        v = np.minimum(d[j * n:(j + 1) * n], 0.7)
        pj = np.zeros(max(P, 256))
        pj[:n] = v * v
        assert s[j] == pairwise(pj)


def test_degenerate_triangles_are_skipped_and_counted():
    v = np.asarray([[0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0]], np.float32)
    t = np.asarray([[0, 1, 2], [0, 0, 1], [0, 1, 3], [2, 2, 2]], np.int32)
    y = np.asarray([[0.2, 0.2, 0.5], [0.5, 0.0, 0.1], [1.5, 0.0, 0.0], [0.0, 1.0, 0.0], [9.0, 9.0, 9.0]])
    q = np.asarray([[0.2, 0.2, 0.0], [0.5, 0.0, 0.0], [1.5, 0.0, 0.0], [0.0, 1.0, 0.0], [np.nan] * 3])
    tri = np.asarray([0, 1, 2, 3, -1])
    val = OA.terms_values(y, tri, q, v, t, np.zeros(3))
    expect = np.zeros((4, 38))
    expect[:3, 37] = 1.0                                        # repeated vertex, collinear, one point: counted only
    assert np.array_equal(val[1:], expect)                      # and the point with no triangle within tau: zeros
    J = np.asarray([0.2, -0.2, 0.0, 0.0, 0.0, 1.0, 0.5])      # (y x n, n, n . y) with n = +z
    assert np.array_equal(val[0], np.concatenate([[J[i] * J[j] for i in range(7) for j in range(i, 7)], J * 0.5, [0.25, 1.0, 0.0]]))
    sums = OA.reduce(OA.block_partials(val)[None])[0]
    assert sums[36] == 1.0 and sums[37] == 3.0


def test_host_pieces():
    assert len(A.GROUP) == 24 and len({G.tobytes() for G in A.GROUP}) == 24
    assert all(np.linalg.det(G) > 0 for G in A.GROUP) and np.array_equal(A.GROUP[0], np.eye(3))
    w = np.asarray([0.3, -0.2, 0.5])
    R = A.rodrigues(w)
    assert np.allclose(R @ R.T, np.eye(3), atol=1e-15) and np.allclose(R @ w, w, atol=1e-15)
    assert np.allclose(A.rodrigues(w * 1e-6), np.eye(3) - np.cross(np.eye(3), w * 1e-6).T, atol=1e-12)
    T = similarity(1.7, (1, 2, 3), 20.0, (0.3, -0.1, 0.2))
    assert np.allclose(A.inverse(T) @ T, np.eye(4), atol=1e-14)
    s, R, t = A.decompose(T)
    assert abs(s - 1.7) < 1e-14 and np.allclose(A.matrix(s, R, t), T, atol=1e-14)
    c = np.asarray([0.1, 0.2, 0.3])
    s2, R2, t2 = A.compose(1.0, np.eye(3), np.zeros(3), np.asarray([0, 0, 0, 0.1, 0, 0, np.log(2.0)]), c)
    assert s2 == 2.0 and np.array_equal(R2, np.eye(3)) and np.allclose(t2, -c + [0.1, 0, 0], atol=1e-16)


def test_argument_errors():
    with pytest.raises(ValueError, match='init'):
        A.check_args('nearest', 1000, 0, None, 10)
    with pytest.raises(ValueError, match='det'):
        A.check_args(np.diag([1.0, 1.0, -1.0, 1.0]), 1000, 0, None, 10)
    with pytest.raises(ValueError, match='4 x 4'):
        A.check_args(np.eye(3), 1000, 0, None, 10)
    with pytest.raises(ValueError, match='samples'):
        A.check_args('auto', 100, 0, None, 10)
    with pytest.raises(ValueError, match='seed'):
        A.check_args('auto', 1000, -1, None, 10)
    with pytest.raises(ValueError, match='max_distance'):
        A.check_args('auto', 1000, 0, 0.0, 10)
    with pytest.raises(ValueError, match='max_iters'):
        A.check_args('auto', 1000, 0, None, 0)
    v, t = blob(20)
    with pytest.raises(RuntimeError, match='too few'):
        run(v + np.float32(5.0), t, v, n=256, max_iters=2)


def test_library_exports_every_symbol_of_the_align_header():
    import __graft_entry__ as g
    lib = ctypes.CDLL(g.build())
    txt = open(os.path.join(ROOT, 'include', 'nero_align.h')).read()
    syms = sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))
    assert syms == ['nero_align_moments', 'nero_align_reduce', 'nero_align_score', 'nero_align_terms', 'nero_align_transform']
    assert all(hasattr(lib, s) for s in syms)
    from nero_b200 import ops
    assert sorted(ops.ALIGN_PROTOS) == syms
    f = {s: getattr(ops.lib, s) for s in syms}
    buf = ctypes.c_void_p(16)
    assert f['nero_align_transform'](buf, -1, buf, 1, buf, None) == 1
    assert f['nero_align_transform'](buf, 4, buf, 0, buf, None) == 1
    assert f['nero_align_transform'](None, 0, None, 1, None, None) == 0
    assert f['nero_align_terms'](buf, 4, buf, None, buf, buf, 0.0, 0.0, 0.0, buf, None) == 1
    assert f['nero_align_moments'](buf, 4, 0.0, 0.0, 0.0, None, None) == 1
    assert f['nero_align_score'](buf, 0, 1, 1.0, buf, None) == 1
    assert f['nero_align_score'](buf, 4, 1, float('nan'), buf, None) == 1
    assert f['nero_align_reduce'](buf, 1, 1, 65, buf, None) == 1
    assert f['nero_align_reduce'](buf, 0, 1, 1, buf, None) == 1


def test_align_meshes_argument_parsing(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    tool = os.path.join(ROOT, 'tools', 'align_meshes.py')
    r = subprocess.run([sys.executable, tool, '--help'], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and '--rigid' in r.stdout and 'not tuned' in r.stdout
    r = subprocess.run([sys.executable, tool, '--src', '/nonexistent/a.ply', '--dst', '/nonexistent/b.ply'], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and 'does not exist' in r.stderr
    bad = tmp_path / 'm.txt'
    bad.write_text('1 0 0\n0 1 0\n')
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    try:
        import align_meshes
    finally:
        sys.path.pop(0)
    with pytest.raises(SystemExit, match='4 lines'):
        align_meshes.read_matrix(str(bad))
    M = similarity(1.7, (1, 2, 3), 20.0, (0.3, -0.1, 0.2))
    good = str(tmp_path / 'good.txt')
    align_meshes.write_matrix(good, M)
    assert np.array_equal(align_meshes.read_matrix(good), M)
    assert align_meshes.parse(['--src', 'a', '--dst', 'b']).init == 'identity'
    f = align_meshes.parse(['--src', 'a', '--dst', 'b', '--init', 'auto', '--rigid', '--samples', '5000', '--iterations', '7'])
    assert (f.init, f.rigid, f.samples, f.iterations) == ('auto', True, 5000, 7)
