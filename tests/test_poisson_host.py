"""CPU: the screened Poisson discretisation of include/nero_poisson.h in oracle/nero_oracle_poisson.py -- the matrix-free
operator and right-hand side against the assembled scipy system, the exact surfaces of a sphere and a torus, the multigrid
preconditioned CG converging on the oracle kernels -- the oriented PLY reader and writer, argument checks, the header's
exports and tools/poisson_mesh.py's argument parsing."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_poisson as OP
from nero_b200 import poisson as P
from nero_b200.evaluate import read_oriented_points_ply, read_points_ply, write_points_ply

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def sphere(n, r=0.35, seed=0):
    rng = np.random.RandomState(seed)
    d = rng.randn(n, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * r, d


def torus(n, R=0.3, r=0.12, seed=0):
    rng = np.random.RandomState(seed)
    u, v = rng.uniform(0, 2 * np.pi, 4 * n), rng.uniform(0, 2 * np.pi, 4 * n)
    keep = rng.uniform(0, 1, 4 * n) < (R + r * np.cos(v)) / (R + r)
    u, v = u[keep][:n], v[keep][:n]
    nrm = np.stack([np.cos(v) * np.cos(u), np.cos(v) * np.sin(u), np.sin(v)], 1)
    return np.stack([(R + r * np.cos(v)) * np.cos(u), (R + r * np.cos(v)) * np.sin(u), r * np.sin(v)], 1), nrm


def euler(v, t):
    e = np.sort(np.concatenate([t[:, [0, 1]], t[:, [1, 2]], t[:, [2, 0]]]), axis=1)
    u, cnt = np.unique(e, axis=0, return_counts=True)
    return v.shape[0] - u.shape[0] + t.shape[0], bool((cnt == 2).all())


def test_matrix_free_operator_equals_assembled_matrix():
    p, nrm = P.check_inputs(*sphere(3000))
    S = OP.setup(p, nrm, 17)
    G, Sm = OP.assemble(S['q'], float(S['ws']), 17)
    v = np.concatenate([a.astype(np.float64) for a in S['v']])
    b = G.T @ v
    assert np.abs(S['b'] - b).max() <= 1e-6 * np.abs(b).max()
    A = G.T @ G + float(S['ws']) * (Sm.T @ Sm)
    x = np.random.RandomState(1).randn(17 ** 3).astype(np.float32)
    y = OP.matvec(x, 17, S['q'], S['start'], S['ws'])
    ref = A @ x.astype(np.float64)
    assert np.abs(y - ref).max() <= 1e-5 * np.abs(ref).max()
    assert np.abs(S['diag'] - (Sm.multiply(Sm)).sum(0).A1).max() <= 1e-5
    assert np.abs(S['density'] - Sm.sum(0).A1).max() <= 1e-5
    # G^T G is the 7-point Laplacian with Neumann boundary: L 1 = 0
    assert np.abs(OP.stencil(np.ones(17 ** 3, np.float32), 17)[1]).max() == 0


@pytest.mark.slow
def test_oracle_sphere_and_torus_geometry():
    p, nrm = P.check_inputs(*sphere(50000), 33)
    v, t, chi, iso, S = OP.mesh(p, nrm, 33)
    d = np.abs(np.linalg.norm(v, axis=1) - 0.35) / S['h']
    e, closed = euler(v, t)
    assert closed and e == 2 and d.mean() <= 0.03 and d.max() <= 0.1      # fp64 prototype: 0.022 h and 0.085 h
    assert chi.reshape(33, 33, 33)[16, 16, 16] < iso                      # chi is below the iso value inside
    p, nrm = P.check_inputs(*torus(60000), 33)
    v, t, chi, iso, S = OP.mesh(p, nrm, 33)
    e, closed = euler(v, t)
    assert closed and e == 0


def test_oracle_pcg_converges_to_the_exact_solution():
    p, nrm = P.check_inputs(*sphere(5000, seed=3))
    S = OP.setup(p, nrm, 17)
    x, hist, it = OP.solve(S, 17, tol=1e-6, max_iters=60)
    chi = OP.exact(S, 17)
    assert hist[-1] <= 1e-6 and it < 30
    assert all(np.isfinite(hist)) and np.abs(x - chi).max() <= 1e-4 * np.abs(chi).max()
    assert P.levels(513) == [513, 257, 129, 65, 33, 17, 9, 5] and P.levels(33) == [33, 17, 9, 5]


def test_multigrid_transfers_are_transposes():
    rng = np.random.RandomState(2)
    f, c = rng.randn(17 ** 3).astype(np.float32), rng.randn(9 ** 3).astype(np.float32)
    lhs = float(OP.restrict(f, 17).astype(np.float64) @ c)
    rhs = float(f.astype(np.float64) @ OP.prolong(c, 9, np.zeros(17 ** 3, np.float32)))
    assert abs(lhs - rhs) <= 1e-4 * abs(lhs)


def test_oriented_ply_round_trip(tmp_path):
    rng = np.random.RandomState(0)
    p, n = rng.randn(50, 3), rng.randn(50, 3)
    path = str(tmp_path / 'o.ply')
    write_points_ply(path, p, n)
    rp, rn = read_oriented_points_ply(path)
    assert np.array_equal(rp, p) and np.array_equal(rn, n) and np.array_equal(read_points_ply(path), p)
    plain = str(tmp_path / 'p.ply')
    write_points_ply(plain, p)
    head = (b'ply\nformat binary_little_endian 1.0\ncomment Created by nero_b200\nelement vertex 50\n'
            b'property double x\nproperty double y\nproperty double z\nend_header\n')
    assert open(plain, 'rb').read() == head + p.astype('<f8').tobytes()
    with pytest.raises(ValueError, match='nx'):
        read_oriented_points_ply(plain)
    # COLMAP's fused.ply: float x y z nx ny nz, uchar red green blue
    dt = np.dtype([(c, '<f4') for c in ('x', 'y', 'z', 'nx', 'ny', 'nz')] + [(c, 'u1') for c in ('red', 'green', 'blue')])
    rec = np.zeros(50, dt)
    for i, c in enumerate('xyz'):
        rec[c], rec['n' + c] = p[:, i], n[:, i]
    rec['red'] = 200
    fused = str(tmp_path / 'fused.ply')
    with open(fused, 'wb') as f:
        f.write(b'ply\nformat binary_little_endian 1.0\nelement vertex 50\n' + b''.join(
            f'property float {c}\n'.encode() for c in ('x', 'y', 'z', 'nx', 'ny', 'nz')) +
            b'property uchar red\nproperty uchar green\nproperty uchar blue\nend_header\n' + rec.tobytes())
    rp, rn = read_oriented_points_ply(fused)
    assert np.array_equal(rp, p.astype(np.float32).astype(np.float64)) and np.array_equal(rn, n.astype(np.float32).astype(np.float64))


def test_argument_errors():
    p, n = sphere(100)
    with pytest.raises(ValueError, match='finite'):
        P.check_inputs(np.where(np.arange(300).reshape(100, 3) == 5, np.inf, p), n)
    with pytest.raises(ValueError, match='zero'):
        P.check_inputs(p, np.where(np.arange(100)[:, None] == 3, 0.0, n))
    with pytest.raises(ValueError, match='at least'):
        P.check_inputs(p[:15], n[:15])
    with pytest.raises(ValueError, match='resolution'):
        P.check_inputs(p, n, 100)
    with pytest.raises(ValueError, match='screen'):
        P.check_inputs(p, n, screen=0.0)
    with pytest.raises(ValueError, match='coincide'):
        P.check_inputs(np.ones((20, 3)), n[:20])
    q, m = P.check_inputs(p, n * 3.0)
    assert q.dtype == np.float64 and m.dtype == np.float32 and np.abs(np.linalg.norm(m, axis=1) - 1).max() < 1e-6


def test_library_exports_every_symbol_of_the_poisson_header():
    import __graft_entry__ as g
    lib = ctypes.CDLL(g.build())
    txt = open(os.path.join(ROOT, 'include', 'nero_poisson.h')).read()
    syms = sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))
    assert len(syms) == 15 and all(hasattr(lib, s) for s in syms)
    from nero_b200 import ops
    assert sorted(ops.POISSON_PROTOS) == syms
    f = {s: getattr(ops.lib, s) for s in syms}
    buf = ctypes.c_void_p(16)
    assert f['nero_poisson_keys'](buf, 0, 0.0, 0.0, 0.0, 1.0, 33, buf, buf, None) == 1
    assert f['nero_poisson_keys'](buf, 4, 0.0, 0.0, 0.0, 0.0, 33, buf, buf, None) == 1
    assert f['nero_poisson_keys'](buf, 4, 0.0, 0.0, 0.0, 1.0, 2, buf, buf, None) == 1
    assert f['nero_poisson_cell_starts'](buf, 4, 0, buf, None) == 1
    assert f['nero_poisson_edge_splat'](buf, buf, 4, buf, 33, 0.0, buf, buf, buf, None) == 1
    assert f['nero_poisson_node_splat'](buf, 4, None, 33, buf, buf, None) == 1
    assert f['nero_poisson_rhs'](buf, buf, None, 33, buf, None) == 1
    assert f['nero_poisson_interp'](buf, 33, buf, 0, buf, None) == 1
    assert f['nero_poisson_matvec'](buf, 1026, buf, 4, buf, 1.0, buf, buf, None) == 1
    assert f['nero_poisson_smooth'](buf, buf, buf, 33, 1.0, 2, None) == 1
    assert f['nero_poisson_smooth'](buf, buf, buf, 33, 0.0, 0, None) == 1
    assert f['nero_poisson_residual'](buf, buf, buf, 33, -1.0, buf, None) == 1
    assert f['nero_poisson_restrict'](buf, 32, buf, None) == 1
    assert f['nero_poisson_prolong'](buf, 1, buf, None) == 1
    assert f['nero_poisson_dot'](None, None, 4, buf, None) == 1
    assert f['nero_poisson_update'](buf, buf, buf, buf, 1.0, 0, None) == 1
    assert f['nero_poisson_direction'](buf, None, 1.0, 4, None) == 1
    assert f['nero_poisson_trim'](buf, 3, buf, 0, 0.1, buf, None) == 1


def test_poisson_mesh_argument_parsing(tmp_path):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    tool = os.path.join(ROOT, 'tools', 'poisson_mesh.py')
    r = subprocess.run([sys.executable, tool, '--help'], env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and '--trim' in r.stdout and '--custom-frame' in r.stdout
    r = subprocess.run([sys.executable, tool, '--points', '/nonexistent/a.ply', '--out', str(tmp_path / 'm.ply')], env=env,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and 'does not exist' in r.stderr
    pts = str(tmp_path / 'p.ply')
    write_points_ply(pts, *sphere(100))
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    try:
        import poisson_mesh
    finally:
        sys.path.pop(0)
    assert poisson_mesh.RESOLUTIONS == P.RESOLUTIONS
    f = poisson_mesh.parse(['--points', pts, '--out', str(tmp_path / 'm.ply'), '--resolution', '129', '--trim', '0.2'])
    assert (f.resolution, f.trim, f.screen, f.min_component) == (129, 0.2, 4.0, 0.0)
    with pytest.raises(SystemExit):
        poisson_mesh.parse(['--points', pts, '--out', str(tmp_path / 'm.ply'), '--resolution', '100'])
    with pytest.raises(SystemExit):
        poisson_mesh.parse(['--points', pts, '--out', str(tmp_path / 'm.ply'), '--custom-frame', str(tmp_path)])
