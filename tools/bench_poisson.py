"""Screened Poisson reconstruction on one H100: about 5 M oriented samples of the 888 056-triangle perturbed-bell mesh of
tools/bench_meshdist.py (512^3 dense marching cubes), each with the outward normal of the triangle MeshDistance.query
returns for it.

    python tools/bench_poisson.py [--samples 5000000] [--resolutions 257 513] [--repeats 5] [--out DIR]

Per resolution: the card's name, power limit and max SM clock read in the same run; binning plus splats (setup()), one
matvec, one V-cycle (CUDA events, median and range of --repeats after a warm call), the whole PCG solve and its iteration
count, extraction plus a 0.1 trim, peak device memory of the whole reconstruct(), and accuracy / completeness of the
untrimmed surface against the source mesh with an F-score at h (meshdist.compare, 1 M samples).  Prints one JSON line per
resolution (and writes them to DIR/bench_poisson.json with --out).
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=5_000_000)
    ap.add_argument('--resolutions', type=int, nargs='+', default=[257, 513])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_poisson: needs a CUDA device')
    from nero_b200 import evaluate as E, params as Pm, poisson as P, synthetic
    from nero_b200.meshdist import MeshDistance, compare
    from nero_b200.renderer import NeROShapeRenderer
    dev = torch.device('cuda', 0)
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(Pm.build_shape_state_dict({}, seed=6033)))
    net = net.to(dev)
    gpu = card()
    cv, ct = net.extract_mesh(resolution=512)
    gv, gt = torch.from_numpy(cv).float().to(dev), torch.from_numpy(ct).int().to(dev)
    pts = E.sample_surface(gv, gt, args.samples, 0)
    _, tri = MeshDistance(gv, gt).query(pts)
    tv = gv.double()[gt.long()[tri.long()]]
    nrm = -torch.linalg.cross(tv[:, 1] - tv[:, 0], tv[:, 2] - tv[:, 0])        # outward: the project's winding points inside
    nrm = nrm / torch.linalg.norm(nrm, dim=1, keepdim=True)
    p, n = P.check_inputs(pts, nrm, 513)
    lines = []
    for N in args.resolutions:
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        setup_s, S = clocked(lambda: P.setup(p, n, N))
        be = P._Cuda(N, S['q'], S['start'], S['ws'])
        L = P.hierarchy(be, N, S['diag'], S['ws'])
        x, y, z = be.vec(), be.vec(), be.vec()
        x.copy_(S['b'])
        t_mv = events(lambda: be.matvec(x, y), args.repeats)
        t_vc = events(lambda: P.vcycle(be, L, x, z), args.repeats)
        solve_s, (chi, hist, it) = clocked(lambda: P.pcg(be, L, S['b']))
        ext_s, (wv, wt, dens, iso, T0) = clocked(lambda: P.extract(be, S, L, chi, 0.1))
        peak_pipeline = torch.cuda.max_memory_allocated()
        del x, y, z, L, be, S, chi, wv, wt, dens
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        total_s, (v, t, info) = clocked(lambda: P.reconstruct(p, n, N))
        peak = torch.cuda.max_memory_allocated()
        m = compare(v, t, gv, gt, samples=1_000_000, thresholds=(info['h'],))
        line = {'metric': 'poisson', 'gpu': gpu, 'resolution': N, 'samples': int(p.shape[0]), 'source_triangles': int(gt.shape[0]),
                'occupied_cells': info['occupied'], 'sigma': info['sigma'], 'h': info['h'],
                'setup_binning_splat_ms': round(setup_s * 1e3, 3), 'matvec_ms': spread(t_mv), 'vcycle_ms': spread(t_vc),
                'solve_ms': round(solve_s * 1e3, 3), 'iterations': it, 'residual': hist[-1],
                'extract_trim_ms': round(ext_s * 1e3, 3), 'triangles': T0, 'reconstruct_total_ms': round(total_s * 1e3, 3),
                'peak_memory_gib': round(peak / 2 ** 30, 3), 'peak_memory_pipeline_gib': round(peak_pipeline / 2 ** 30, 3),
                'accuracy_mean_over_h': m['accuracy']['mean'] / info['h'], 'completeness_mean_over_h': m['completeness']['mean'] / info['h'],
                'accuracy_p99_over_h': m['accuracy']['p99'] / info['h'], 'fscore_at_h': m['thresholds'][0]['fscore']}
        print(json.dumps(line), flush=True)
        lines.append(line)
        del v, t, info
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_poisson.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
