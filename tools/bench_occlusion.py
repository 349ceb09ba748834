"""Ambient-occlusion bake on one H100: the perturbed-bell 2048^3 narrow-band mesh of tools/bench_normalmap.py simplified to
300 000 and 50 000 triangles, unwrapped at 1024^2 with ssaa 2 (a 2048^2 atlas), baked from the low mesh itself and from the
2048^3 mesh through the cage ray, at 64 and 256 rays per texel.

    python tools/bench_occlusion.py [--resolution 2048] [--faces 300000 50000] [--size 1024] [--rays 64 256] [--repeats 5] \\
        [--distance 0.25] [--out DIR]

Per line: the card's name and power limit read in the same run, then the counting kernel (CUDA events, median of --repeats;
rays/s = covered texels x rays / time, over every texel including cage misses that cast nothing), the texel prep kernel, the
inpaint and the 2x down-sample, the host BVH build of the occluder mesh (once per mesh), the covered texels, cage hits and
misses and the mean unoccluded fraction.
Prints one JSON line per measurement (and writes them to DIR/bench_occlusion.json with --out).
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

import numpy as np
import torch

from bench_mesh import card
from bench_mesh_sparse import spread
from bench_normalmap import events


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--resolution', type=int, default=2048)
    ap.add_argument('--faces', type=int, nargs='*', default=[300000, 50000])
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--rays', type=int, nargs='*', default=[64, 256])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--distance', type=float, default=0.25)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_occlusion: needs a CUDA device')
    from nero_b200 import occlusion as OC, ops, params as P, synthetic
    from nero_b200 import texmap as TX
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

    fv, ft = net.extract_mesh_sparse(resolution=args.resolution)
    fv, ft = np.ascontiguousarray(fv, np.float32), np.ascontiguousarray(ft, np.int32)
    fv_d, ft_d = torch.from_numpy(fv).to(dev), torch.from_numpy(ft).to(dev)
    t0 = time.perf_counter()
    detail_bvh = OC._bvh_cuda(fv, ft)
    torch.cuda.synchronize()
    detail_bvh_s = time.perf_counter() - t0
    n = args.size
    for F in args.faces:
        lv, lt, _ = simplify_cuda(fv_d, ft_d, F)
        lv, lt = lv.cpu().numpy(), lt.cpu().numpy()
        vt, ftx = TX.uv_atlas(lv, lt, 2 * n, 2 * n, 4)
        for source in ('self', 'detail'):
            prof = {}
            det = (fv, ft) if source == 'detail' else (None, None)
            b = OC.bake_cuda(lv, lt, vt, ftx, n, *det, ssaa=2, rays=args.rays[0], distance=args.distance, profile=prof)
            cov = int(b['hit'].shape[0])
            hits = int(b['hit'].sum())
            prep = spread(events(lambda: ops.K('nero_occlusion_texels', *b['texel_args']), args.repeats))
            inp = events(lambda: TX.inpaint(b['img'], b['raster']['owner']), args.repeats)
            filled = TX.inpaint(b['img'], b['raster']['owner'])[0]
            down = events(lambda: TX.downsample(filled), args.repeats)
            bvh_s = detail_bvh_s if source == 'detail' else prof['bvh'] * 1e-3
            for R in args.rays:
                a = list(b['args'])
                a[6] = int(R)
                count_t = events(lambda: ops.K('nero_occlusion_points', *a), args.repeats)
                med = sorted(count_t)[len(count_t) // 2]
                mean = float(a[9].sum().item()) / (cov * R)
                emit({'metric': 'occlusion_bake', 'gpu': gpu, 'source': source, 'low_triangles': int(lt.shape[0]),
                      'occluder_triangles': int(ft.shape[0] if source == 'detail' else lt.shape[0]), 'atlas': 2 * n, 'map': n,
                      'rays': R, 'distance': args.distance, 'covered': cov, 'hits': hits, 'misses': cov - hits,
                      'mean_unoccluded': round(mean, 5), 'count_kernel_ms': spread(count_t), 'rays_per_s': round(cov * R / med, 1),
                      'texel_prep_ms': prep, 'inpaint_ms': spread(inp), 'downsample_ms': spread(down),
                      'bvh_build_host_s': round(bvh_s, 3)})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_occlusion.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
