"""Mesh registration on one H100: the perturbed-bell meshes of tools/bench_meshdist.py.  The source is the 2048^3 mesh
simplified to 300 000 triangles, mapped by a known similarity (s = 1.7, 20 degrees about the axis (1, 2, 3), a translation
of length 0.3); the targets are the same mesh simplified to 888 056 triangles and the 14.25 M-triangle mesh itself.

    python tools/bench_align.py [--samples 200000] [--repeats 9] [--out DIR]

Per target: the card's name, power limit and max SM clock read in the same run; the host BVH build with the upload; the
whole align(init='auto') call, the coarse search alone and, at the final transform, one iteration's kernels between CUDA
events (transform, BVH query, terms + reduce; median and range of --repeats after a warm call); iterations to convergence
and the error of the recovered transform.  Then the convergence basin of init='identity' on the 888 056-triangle target:
rotation offsets of 10, 20, 40 and 60 degrees about the axis (1, -1, 2) through the target's centroid, and whether each
run converges to the known transform (rotation error below 1e-4 rad).
Prints one JSON line per measurement (and writes them to DIR/bench_align.json with --out).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np
import torch

from bench_mesh import card
from bench_mesh_sparse import clocked, spread
from bench_normalmap import events


def similarity(A, s, axis, degrees, t):
    a = np.asarray(axis, np.float64)
    return A.matrix(s, A.rodrigues(a / np.linalg.norm(a) * np.radians(degrees)), np.asarray(t, np.float64))


def errors(A, M, T):
    """(rotation angle, relative scale error, translation error) between two similarities."""
    s1, R1, t1 = A.decompose(M)
    s2, R2, t2 = A.decompose(T)
    c = np.clip((np.trace(R1.T @ R2) - 1) / 2, -1.0, 1.0)
    return float(np.arccos(c)), float(abs(s1 / s2 - 1)), float(np.abs(t1 - t2).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=200_000)
    ap.add_argument('--repeats', type=int, default=9)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_align: needs a CUDA device')
    from nero_b200 import align as A, evaluate as E, params as P, synthetic
    from nero_b200.meshdist import MeshDistance
    from nero_b200.renderer import NeROShapeRenderer
    from nero_b200.simplify import simplify_cuda
    dev = torch.device('cuda', 0)
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    net = net.to(dev)
    gpu = card()
    lines = []

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    fv, ft = net.extract_mesh_sparse(resolution=2048)
    fv, ft = torch.from_numpy(fv).float().to(dev), torch.from_numpy(ft).int().to(dev)
    targets = {}
    sv, st, _ = simplify_cuda(fv, ft, 300000)
    v, t, _ = simplify_cuda(fv, ft, 888056)
    targets['sparse_2048_simplified_888056'] = (v, t)
    targets['sparse_2048'] = (fv, ft)
    truth = similarity(A, 1.7, (1, 2, 3), 20.0, 0.3 * np.asarray([1.0, -1.0, 1.0]) / np.sqrt(3.0))
    src = A.apply(A.inverse(truth), sv).float()

    index = {}
    for name, (v, t) in targets.items():
        build_s, md = clocked(lambda: MeshDistance(v, t))
        index[name] = md
        total_s, res = clocked(lambda: A.align((src, st), md, init='auto', samples=args.samples))
        rot, sc, tr = errors(A, res['matrix'], truth)
        pts = E.sample_surface(src, st, args.samples, 0)
        b = A._Gpu(pts, md, E.sample_surface(md.verts, md.tris, args.samples, 1))
        center, C = A.moment_stats(b.moments('dst'), b.dst_origin)
        L = float(np.sqrt(np.trace(C)))
        cands = A.candidates(A.moment_stats(b.moments('src'), b.src_origin), (center, C), False)
        mats = np.stack([A.matrix(*c)[:3] for c in cands])
        coarse = []
        for _ in range(args.repeats):
            coarse.append(clocked(lambda: b.score(mats, A.COARSE_TAU * L))[0])
        M = res['matrix'][:3]
        tau = res['tau'][-1]
        n = pts.shape[0]
        y = A.transform(pts, M)
        t_tr = events(lambda: A.transform(pts, M), args.repeats)
        t_q = events(lambda: b._query(y, tau, b.dist, b.tri, b.closest), args.repeats)
        t_terms = events(lambda: A.reduce(A.terms(y, b.tri, b.closest, md, center), 1, A.TERMS), args.repeats)
        assert int(b.status.item()) == 0
        med = lambda ts: sorted(ts)[len(ts) // 2]
        emit({'metric': 'align', 'gpu': gpu, 'target': name, 'target_triangles': int(t.shape[0]), 'source_triangles': int(st.shape[0]),
              'samples': n, 'bvh_build_host_s': round(build_s, 3), 'align_auto_s': round(total_s, 3),
              'coarse_search_ms': spread(coarse), 'iteration_ms': {'transform': spread(t_tr), 'query': spread(t_q),
                                                                   'terms_reduce': spread(t_terms)},
              'iteration_kernels_ms_median': round((med(t_tr) + med(t_q) + med(t_terms)) * 1e3, 3),
              'iterations': res['iterations'], 'converged': res['converged'], 'coarse_best': res['coarse_best'],
              'rms_final': res['rms'][-1], 'rotation_error_rad': rot, 'scale_error_rel': sc, 'translation_error': tr,
              'translation_error_over_L': tr / L, 'L': L, 'undetermined': [u['kind'] for u in res['undetermined']]})

    name = 'sparse_2048_simplified_888056'
    md = index[name]
    b0 = A._Gpu(src, md, E.sample_surface(md.verts, md.tris, args.samples, 1))
    centroid = A.moment_stats(b0.moments('dst'), b0.dst_origin)[0]
    for deg in (10.0, 20.0, 40.0, 60.0):
        R = similarity(A, 1.0, (1, -1, 2), deg, (0, 0, 0))
        T = A.matrix(1.0, R[:3, :3], centroid - R[:3, :3] @ centroid)
        s_v = A.apply(A.inverse(T), sv).float()
        try:
            secs, res = clocked(lambda: A.align((s_v, st), md, init='identity', samples=args.samples))
            rot, sc, tr = errors(A, res['matrix'], T)
            row = {'iterations': res['iterations'], 'converged': res['converged'], 'rotation_error_rad': rot, 'scale_error_rel': sc,
                   'translation_error': tr, 'recovered': bool(res['converged'] and rot < 1e-4), 'align_s': round(secs, 3)}
        except RuntimeError as e:
            row = {'recovered': False, 'error': str(e)}
        emit({'metric': 'align_basin', 'gpu': gpu, 'target': name, 'init': 'identity', 'rotation_offset_deg': deg, **row})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_align.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
