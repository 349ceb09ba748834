"""GPU: the registration kernels (transform, terms, moments, score, reduce) against oracle/nero_oracle_align.py bit for bit,
the first ICP iterates and the coarse scores bit for bit, recovery of known similarities (same and different
tessellation, a source with an outlier plate), determinism, and tools/compare_meshes.py --align / tools/align_meshes.py
end to end."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_align as OA
from nero_b200 import align as A
from nero_b200 import evaluate as E
from nero_b200 import meshdist as MD
from test_align_host import blob, errors, mc, moved, similarity
from test_meshdist_gpu import degenerate

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def bumpy():
    """The smoke test's bumpy marching-cubes sphere."""
    return mc(lambda x: np.linalg.norm(x, axis=-1) - 0.6 + 0.1 * np.sin(5 * x[..., 0]) * np.cos(4 * x[..., 1] + x[..., 2]), 32)


def blob_cuda(n):
    """The blob of test_align_host at n^3 through the GPU marching cubes, in [-1, 1]^3."""
    from nero_b200.mesh import marching_cubes_cuda
    ax = torch.linspace(-1.0, 1.0, n, dtype=torch.float64, device='cuda')
    x = torch.stack(torch.meshgrid(ax, ax, ax, indexing='ij'), -1)
    sd = lambda c, r: torch.linalg.norm(x - torch.tensor(c, dtype=torch.float64, device='cuda'), dim=-1) - r
    ell = (torch.linalg.norm(x / torch.tensor([0.55, 0.25, 0.3], dtype=torch.float64, device='cuda'), dim=-1) - 1.0) * 0.25
    f = torch.minimum(torch.minimum(sd((0.35, 0.1, 0.0), 0.3), sd((-0.3, 0.25, 0.1), 0.22)), torch.minimum(sd((0.0, -0.3, 0.25), 0.18), ell))
    v, t = marching_cubes_cuda(f.float(), 0.0)
    return (v.double() * (2.0 / (n - 1)) - 1.0).float().cpu().numpy(), t.cpu().numpy()


@pytest.mark.parametrize('mesh', [bumpy, degenerate])
def test_kernels_bit_exact_against_the_oracle(mesh):
    v, t = mesh()
    md = MD.MeshDistance(v, t)
    rng = np.random.RandomState(2)
    p = np.concatenate([E.sample_surface(v, t, 3000, seed=4).cpu().numpy() + rng.randn(3000, 3) * 0.02, v.astype(np.float64)])
    M = similarity(1.1, (1, -2, 0.5), 4.0, (0.01, 0.02, -0.03))[:3]
    y = A.transform(p, M)
    oy = OA.transform(p, M)
    assert np.array_equal(y.cpu().numpy(), oy)
    center = np.asarray([0.01, -0.02, 0.03])
    for tau in (0.03, np.inf):
        d, tri, q = md.query(y, max_dist=tau, closest=True)
        part = A.terms(y, tri, q, md, center)
        opart = OA.block_partials(OA.terms_values(oy, tri.cpu().numpy(), q.cpu().numpy(), v, t, center))
        assert np.array_equal(part.cpu().numpy(), opart)
        sums = A.reduce(part, 1, A.TERMS).cpu().numpy()
        assert np.array_equal(sums, OA.reduce(opart[None]))
        assert sums[0, 36] > 0 and (sums[0, 36] + sums[0, 37] == (tri >= 0).sum().item())
        if mesh is degenerate and tau == np.inf:
            assert sums[0, 37] > 0                                   # some closest triangles have no normal
    origin = A.bbox_center(y)
    part = A.moments(y, origin)
    opart = OA.block_partials(OA.moments_values(oy, origin))
    assert np.array_equal(part.cpu().numpy(), opart)
    assert np.array_equal(A.reduce(part, 1, A.MOMENTS).cpu().numpy(), OA.reduce(opart[None]))


def test_coarse_candidates_bit_exact_against_the_oracle():
    v, t = blob()
    md = MD.MeshDistance(v, t)
    src = moved(v, similarity(1.7, (1, 2, 3), 70.0, (0.3, 0.1, -0.2)))
    pts = E.sample_surface(src, t, 4096, seed=0)
    tgt = E.sample_surface(v, t, 4096, seed=1)
    b = A._Gpu(pts, md, tgt)
    stats = [A.moment_stats(b.moments(w), o) for w, o in (('src', b.src_origin), ('dst', b.dst_origin))]
    ob = OA.Backend(pts.cpu().numpy(), v, t, tgt.cpu().numpy())
    for w, g in (('src', b.moments('src')), ('dst', b.moments('dst'))):
        assert np.array_equal(g, ob.moments(w))
    mats = np.stack([A.matrix(*c)[:3] for c in A.candidates(*stats, False)])
    tau = 0.05
    y = A.transform(b.sub, mats)
    assert np.array_equal(y.cpu().numpy(), OA.transform(b.sub.cpu().numpy(), mats))
    d = md.query(y, max_dist=tau)[0]
    part = A.score(d, 24, tau)
    opart = OA.score_partials(d.cpu().numpy(), 24, tau)
    assert part.shape == (24, 16) and np.array_equal(part.cpu().numpy(), opart)
    assert np.array_equal(A.reduce(part, 24, 1).cpu().numpy()[:, 0], OA.reduce(opart[:, :, None])[:, 0])


@pytest.mark.parametrize('init', ['identity', 'auto'])
def test_first_iterates_bit_exact_against_the_oracle(init):
    v, t = blob()
    T = similarity(1.2, (1, 2, 3), 8.0 if init == 'identity' else 120.0, (0.05, -0.03, 0.02))
    src = moved(v, T)
    md = MD.MeshDistance(v, t)
    iters = 4 if init == 'identity' else 2
    res = A.align((src, t), md, init=init, samples=1024, seed=3, max_iters=iters)
    ores, _ = OA.align(E.sample_surface(src, t, 1024, seed=3).cpu().numpy(), v, t, E.sample_surface(v, t, 1024, seed=4).cpu().numpy(),
                       init=init, max_iters=iters)
    assert res['matrix'].tobytes() == ores['matrix'].tobytes()
    for k in ('tau', 'inliers', 'rms', 'degenerate', 'coarse_scores', 'coarse_best'):
        assert res.get(k) == ores.get(k), k


def assert_recovered(res, T, extent, rot, scale, trans):
    r, s, tr = errors(res['matrix'], T)
    assert res['converged'] and r < rot and s < scale and tr < trans * extent, (r, s, tr / extent, res['iterations'])


BIG = similarity(1.7, (1, 2, 3), 20.0, (0.3, -0.2, 0.1))


def test_recovers_a_similarity_on_the_same_tessellation():
    """A float32 copy of a ~300 k-triangle mesh mapped by BIG: only the vertex rounding separates the two."""
    v, t = blob_cuda(384)
    assert 250_000 < t.shape[0] < 400_000
    res = A.align((moved(v, BIG), t), MD.MeshDistance(v, t), init='auto')
    assert res['undetermined'] == []
    assert_recovered(res, BIG, 2.0, 2e-6, 2e-6, 2e-6)


def test_recovers_a_similarity_across_tessellations():
    """128^3 against 192^3 marching cubes of one field: the surfaces differ by the discretisation, O(h^2) with h = 2 / 127,
    so the bound is 1e-3 in rotation (rad), relative scale and translation over the extent."""
    v1, t1 = blob_cuda(128)
    v2, t2 = blob_cuda(192)
    res = A.align((moved(v1, BIG), t1), MD.MeshDistance(v2, t2), init='auto')
    assert_recovered(res, BIG, 2.0, 1e-3, 1e-3, 1e-3)


def plate(v, t, share, gap):
    """A square plate under the mesh (z = min z - gap) with `share` of the mesh's area, as two triangles per grid cell."""
    a = v[t].astype(np.float64)
    area = 0.5 * np.linalg.norm(np.cross(a[:, 1] - a[:, 0], a[:, 2] - a[:, 0]), axis=1).sum()
    side = np.sqrt(share * area)
    n = 64
    g = np.linspace(-side / 2, side / 2, n)
    X, Y = np.meshgrid(g, g, indexing='ij')
    c = (v.min(0) + v.max(0)) / 2
    pv = np.stack([X + c[0], Y + c[1], np.full_like(X, v[:, 2].min() - gap)], -1).reshape(-1, 3)
    i, j = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing='ij')
    q = [i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1]
    pt = np.concatenate([np.stack([q[0], q[1], q[2]], -1).reshape(-1, 3), np.stack([q[0], q[2], q[3]], -1).reshape(-1, 3)])
    return np.concatenate([v, pv.astype(np.float32)]), np.concatenate([t, pt + v.shape[0]]).astype(np.int32)


def test_an_outlier_plate_does_not_move_the_result():
    """The source carries a plate of 30 % of its area, 0.15 below it (farther than the first inlier distance, 0.1 of the
    target's RMS radius): the plate never becomes inlier and the transform is recovered as without it."""
    v, t = blob_cuda(128)
    T = similarity(1.02, (1, 1, 0), 3.0, (0.01, 0.0, -0.01))
    sv, st = plate(moved(v, T), t, 0.3, 0.15)
    res = A.align((sv, st), MD.MeshDistance(v, t))
    assert abs(res['inliers'][-1] / 200_000 - 1 / 1.3) < 0.01    # the plate's samples (0.3 / 1.3 of them) are not inliers
    assert_recovered(res, T, 2.0, 2e-6, 2e-6, 2e-6)


def test_two_runs_give_the_same_bytes():
    v, t = blob_cuda(128)
    md = MD.MeshDistance(v, t)
    a = A.align((moved(v, BIG), t), md, init='auto')
    b = A.align((moved(v, BIG), t), md, init='auto')
    assert a['matrix'].tobytes() == b['matrix'].tobytes() and a['rms'] == b['rms'] and a['coarse_scores'] == b['coarse_scores']


def test_point_cloud_source_and_apply():
    v, t = blob()
    T = similarity(0.9, (0, 1, 1), 5.0, (0.02, 0.01, 0.0))
    pts = A.apply(A.inverse(T), E.sample_surface(v, t, 20000, seed=7))
    res = A.align(pts.cpu().numpy(), MD.MeshDistance(v, t))
    assert_recovered(res, T, 2.0, 1e-5, 1e-5, 1e-5)
    with pytest.raises(TypeError, match='MeshDistance'):
        A.align(pts, (v, t))


def test_compare_meshes_align_end_to_end(tmp_path):
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    v, t = blob_cuda(96)
    T = similarity(1.03, (1, -1, 2), 3.0, (0.02, -0.01, 0.01))
    pr, gt = str(tmp_path / 'pr.ply'), str(tmp_path / 'gt.ply')
    write_ply(pr, moved(v, T), t)
    write_ply(gt, v, t)
    js, e = str(tmp_path / 'm.json'), str(tmp_path / 'e.ply')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'compare_meshes.py'), '--pr', pr, '--gt', gt, '--samples', '100000',
                        '--align', 'icp', '--json', js, '--errors', e], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    out = r.stdout.splitlines()
    assert out[0].startswith('align.matrix.0 ') and 'align.undetermined none' in out
    m = json.load(open(js))
    assert all(row['fscore'] == 1.0 for row in m['thresholds'])
    ref = MD.compare(v, t, v, t, samples=100000, seed=0)        # the untransformed pair
    for side in ('accuracy', 'completeness'):
        for k in ('mean', 'max', 'p99'):
            assert abs(m[side][k] - ref[side][k]) <= 1e-6, (side, k)
    assert_recovered({'matrix': np.asarray(m['align']['matrix']), 'converged': m['align']['converged']}, T, 2.0, 2e-6, 2e-6, 2e-6)
    ev, et = read_ply(e)
    assert np.array_equal(et, t) and np.abs(ev - v).max() < 1e-5


def test_align_meshes_end_to_end(tmp_path):
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    v, t = blob_cuda(96)
    src, dst = str(tmp_path / 'src.ply'), str(tmp_path / 'dst.ply')
    write_ply(src, moved(v, BIG), t)
    write_ply(dst, v, t)
    out, mat, cloud = str(tmp_path / 'out.ply'), str(tmp_path / 'm.txt'), str(tmp_path / 'cloud.ply')
    tool = os.path.join(ROOT, 'tools', 'align_meshes.py')
    r = subprocess.run([sys.executable, tool, '--src', src, '--dst', dst, '--init', 'auto', '--out', out, '--matrix', mat],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    M = np.loadtxt(mat)
    assert_recovered({'matrix': M, 'converged': True}, BIG, 2.0, 2e-6, 2e-6, 2e-6)
    ov, ot = read_ply(out)
    assert np.array_equal(ot, t) and np.abs(ov - v).max() < 1e-5
    E.write_points_ply(cloud, A.apply(A.inverse(BIG), E.sample_surface(v, t, 20000, seed=9)).cpu().numpy())
    r = subprocess.run([sys.executable, tool, '--src', cloud, '--dst', dst, '--init', mat, '--iterations', '3'],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr
    assert abs(float(dict(ln.split(' ', 1) for ln in r.stdout.splitlines())['scale']) / 1.7 - 1) < 1e-5
