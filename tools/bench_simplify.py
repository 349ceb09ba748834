"""Mesh simplification on one H100: the perturbed-bell narrow-band meshes (the network tools/bench_mesh_sparse.py uses) at
1024^3 and 2048^3 reduced to 888 056 and to 300 000 triangles.

    python tools/bench_simplify.py [--resolutions 1024 2048] [--faces 888056 300000] [--repeats 2] [--samples 2000000] [--out DIR]

Per line: the card's name and power limit read in the same run; end-to-end milliseconds of simplify_cuda (host clock around
a synchronised call, warm; median and range); rounds and the other statistics; the split into check / prepare / edges /
cost / select / collapse / output from a separate profiled call (each phase ended by a device synchronise, so their sum
exceeds the unprofiled time a little).  Then the reasons to simplify, measured once each:
  * the host BVH build (nero_bvh_build_host) and the texture-atlas unwrapper (nero_uv_atlas_host) on the finest mesh and on
    its simplification to the first --faces count;
  * Chamfer distance and one-sided maximum distances, against the finest mesh, of the 512^3 marching-cubes mesh and of
    the finest mesh simplified to the 512^3 mesh's own triangle count.  Distances are exact nearest distances between
    --samples area-uniform surface samples of each mesh (evaluate.sample_surface, nero_nearest_dist); Chamfer = the mean
    of the two directions' means.  The finest mesh's own samples under another seed give the floor those distances
    cannot go below at this sample count.
Prints one JSON line per measurement (and writes them to DIR/bench_simplify.json with --out).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch

from bench_mesh import card
from bench_mesh_sparse import clocked, spread


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--resolutions', type=int, nargs='*', default=[1024, 2048])
    ap.add_argument('--faces', type=int, nargs='*', default=[888056, 300000])
    ap.add_argument('--repeats', type=int, default=2)
    ap.add_argument('--samples', type=int, default=2000000)
    ap.add_argument('--compare', type=int, default=512, help='marching-cubes resolution of the same-size comparison (0: skip)')
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_simplify: needs a CUDA device')
    from nero_b200 import evaluate as E, ops, params as P, synthetic
    from nero_b200.renderer import NeROShapeRenderer
    from nero_b200.simplify import simplify_cuda
    from nero_b200.texmap import uv_atlas
    dev = torch.device('cuda', 0)
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    net = net.to(dev)
    gpu = card()
    lines = []

    def emit(line):
        print(json.dumps(line), flush=True)
        lines.append(line)

    meshes = {}
    for res in args.resolutions:
        v, t, _ = net.extract_mesh_sparse(resolution=res, return_stats=True)
        meshes[res] = (torch.from_numpy(v).float().to(dev), torch.from_numpy(t).int().to(dev))
        for F in args.faces:
            run = lambda: simplify_cuda(*meshes[res], F)
            run()                                            # warm
            ts = []
            for _ in range(args.repeats):
                t_, (_, _, stats) = clocked(run)
                ts.append(t_)
            ms = simplify_cuda(*meshes[res], F, profile=True)[2]['ms']
            emit({'metric': 'simplify', 'gpu': gpu, 'resolution': res, 'triangles_in': int(meshes[res][1].shape[0]),
                  'vertices_in': int(meshes[res][0].shape[0]), 'faces': F, 'simplify_ms': spread(ts),
                  'phases_ms': {k: round(x, 3) for k, x in ms.items()}, **stats})

    fine = max(args.resolutions)
    fv, ft = meshes[fine]
    sv, st, _ = simplify_cuda(fv, ft, args.faces[0])
    host = {}
    for tag, (v, t) in (('fine', (fv, ft)), ('simplified', (sv, st))):
        vn, tn = v.cpu().numpy(), t.cpu().numpy()
        t0 = time.perf_counter()
        ops.bvh_build(vn, tn)
        t1 = time.perf_counter()
        uv_atlas(vn, tn, 4096, 4096, 2)
        t2 = time.perf_counter()
        host[tag] = {'triangles': int(tn.shape[0]), 'bvh_build_host_s': round(t1 - t0, 3), 'uv_atlas_host_s': round(t2 - t1, 3)}
    emit({'metric': 'simplify_host_consumers', 'gpu': gpu, 'resolution': fine, **host})

    if args.compare:
        cv, ct = net.extract_mesh(resolution=args.compare)
        cv, ct = torch.from_numpy(cv).float().to(dev), torch.from_numpy(ct).int().to(dev)
        n = int(ct.shape[0])
        qv, qt, qstats = simplify_cuda(fv, ft, n)
        ref = E.sample_surface(fv, ft, args.samples, seed=1)

        def dists(v, t):
            p = E.sample_surface(v, t, args.samples, seed=2)
            d_pr = E.nearest_dist_cuda(p, ref).double()
            d_gt = E.nearest_dist_cuda(ref, p).double()
            return {'chamfer': 0.5 * float(d_pr.mean() + d_gt.mean()), 'to_fine_mean': float(d_pr.mean()),
                    'to_fine_max': float(d_pr.max()), 'from_fine_max': float(d_gt.max())}

        emit({'metric': 'simplify_accuracy', 'gpu': gpu, 'reference': f'{fine}^3 sparse marching cubes ({int(ft.shape[0])} triangles)',
              'samples': args.samples, 'triangles': n, f'marching_cubes_{args.compare}': dists(cv, ct),
              f'simplified_{fine}': {**dists(qv, qt), 'triangles': int(qt.shape[0]), 'rounds': qstats['rounds']},
              f'sampling_floor_{fine}': dists(fv, ft)})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_simplify.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
