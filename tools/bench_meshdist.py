"""Point-to-mesh distance on one H100: the perturbed-bell meshes of tools/bench_simplify.py -- 512^3 dense marching cubes,
the 2048^3 narrow-band mesh and that mesh simplified to 888 056 and to 300 000 triangles -- indexed once each and queried
with 1 M float64 surface samples of the 2048^3 mesh.

    python tools/bench_meshdist.py [--samples 1000000] [--repeats 5] [--out DIR]

Per mesh: the card's name and power limit read in the same run; the host BVH build with the upload (MeshDistance); the
query kernel between CUDA events (median and range of --repeats, after a warm call), in the samples' own random order and
sorted by a 30-bit Morton key of the point, with queries/s.  Then the metrics of meshdist.compare for each coarse mesh
against the 2048^3 mesh (--samples per side, seed 0).
Prints one JSON line per measurement (and writes them to DIR/bench_meshdist.json with --out).
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
from bench_mesh_sparse import spread
from bench_normalmap import events


def morton_order(p):
    """Permutation sorting points [n,3] by the Morton key of their 10-bit cell in the cloud's bounding box (torch plumbing)."""
    lo, hi = p.amin(0), p.amax(0)
    cell = ((p - lo) / (hi - lo).clamp_min(1e-30) * 1023).long().clamp(0, 1023)
    key = torch.zeros(p.shape[0], dtype=torch.int64, device=p.device)
    for bit in range(10):
        for axis in range(3):
            key |= ((cell[:, axis] >> bit) & 1) << (3 * bit + axis)
    return torch.argsort(key)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=1_000_000)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_meshdist: needs a CUDA device')
    from nero_b200 import evaluate as E, ops, params as P, synthetic
    from nero_b200.meshdist import MeshDistance, compare_index
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
    cv, ct = net.extract_mesh(resolution=512)
    meshes = {'dense_512': (torch.from_numpy(cv).float().to(dev), torch.from_numpy(ct).int().to(dev))}
    for F in (888056, 300000):
        v, t, _ = simplify_cuda(fv, ft, F)
        meshes[f'sparse_2048_simplified_{F}'] = (v, t)
    meshes['sparse_2048'] = (fv, ft)

    queries = E.sample_surface(fv, ft, args.samples, seed=1)
    order = morton_order(queries)
    sorted_q = queries[order].contiguous()
    index = {}
    for name, (v, t) in meshes.items():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        md = MeshDistance(v, t)
        torch.cuda.synchronize()
        build_s = time.perf_counter() - t0
        index[name] = md
        n = queries.shape[0]
        dist = torch.empty(n, dtype=torch.float64, device=dev)
        tri = torch.empty(n, dtype=torch.int32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        run = lambda q: ops.K('nero_meshdist_query', q, n, md.nodes, md.tri_ids, md.verts, md.tris, float('inf'), dist, tri, None, status)
        t_rand = events(lambda: run(queries), args.repeats)
        d_rand = dist.clone()
        t_sort = events(lambda: run(sorted_q), args.repeats)
        assert int(status.item()) == 0
        assert torch.equal(dist[torch.argsort(order)], d_rand), 'sorted and unsorted queries give different distances'
        med = lambda ts: sorted(ts)[len(ts) // 2]
        emit({'metric': 'meshdist_query', 'gpu': gpu, 'mesh': name, 'triangles': int(t.shape[0]), 'queries': n,
              'bvh_build_host_s': round(build_s, 3), 'query_ms_random_order': spread(t_rand),
              'queries_per_s_random_order': round(n / med(t_rand), 1), 'query_ms_morton_order': spread(t_sort),
              'queries_per_s_morton_order': round(n / med(t_sort), 1), 'mean_dist': float(d_rand.mean()), 'max_dist': float(d_rand.max())})

    gt = index['sparse_2048']
    for name in ('dense_512', 'sparse_2048_simplified_888056', 'sparse_2048_simplified_300000'):
        t0 = time.perf_counter()
        m = compare_index(index[name], gt, args.samples, 0)
        emit({'metric': 'meshdist_compare', 'gpu': gpu, 'pr': name, 'gt': f'sparse_2048 ({int(ft.shape[0])} triangles)',
              'triangles': int(meshes[name][1].shape[0]), 'compare_s': round(time.perf_counter() - t0, 3), **m})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_meshdist.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
