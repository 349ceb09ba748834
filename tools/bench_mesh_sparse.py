"""Narrow-band mesh extraction on one H100: NeROShapeRenderer.extract_mesh_sparse against extract_mesh on the perturbed bell
parameters (the network tools/bench_mesh.py uses).

    python tools/bench_mesh_sparse.py [--compare 512] [--sparse 1024 2048] [--repeats 5] [--brick 8] [--out DIR]

At the --compare resolution the dense and the sparse path are timed alternately in one process, after torch.equal has shown
that both return the same vertex and triangle arrays at that size.  At the --sparse resolutions only the sparse path runs (the
dense field of 1024^3 takes 4.3 GB and 18 s by extrapolation, that of 2048^3 does not fit the card).  Per line: the card's name
and power limit read in the same run; end-to-end milliseconds (host clock around a synchronised call, warm; median and range);
the split into coarse pass / fill / grow / cube kernels / sort from a separate profiled call (each phase ended by a device
synchronise, so their sum exceeds the unprofiled time a little); extract_sparse's statistics; the peak of
torch.cuda.max_memory_allocated over a call; and the fill's algorithmic TFLOP/s (524 544 MAC per evaluated point over the fill
time of the profiled call).  Prints one JSON line per measurement (and writes them to DIR/bench_mesh_sparse.json with --out).
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

from bench_mesh import SDF_MAC_PER_POINT, card


def spread(ts):
    ts = sorted(ts)
    return {'median': round(ts[len(ts) // 2] * 1e3, 3), 'min': round(ts[0] * 1e3, 3), 'max': round(ts[-1] * 1e3, 3)}


def clocked(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--compare', type=int, default=512)
    ap.add_argument('--sparse', type=int, nargs='*', default=[1024, 2048])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--brick', type=int, default=8)
    ap.add_argument('--lipschitz', type=float, default=2.0)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mesh_sparse: needs a CUDA device')
    from nero_b200 import mesh, params as P, synthetic
    from nero_b200.renderer import NeROShapeRenderer
    dev = torch.device('cuda', 0)
    cfg = {}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict(cfg, seed=6033)))
    net = net.to(dev)
    gpu = card()
    lines = []

    def sparse_line(res, repeats):
        run = lambda: net.extract_mesh_sparse(resolution=res, brick=args.brick, lipschitz=args.lipschitz, return_stats=True)
        run()                                                # warm
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ts = []
        for _ in range(repeats):
            t, (v, tri, stats) = clocked(run)
            ts.append(t)
        peak = torch.cuda.max_memory_allocated()
        # the phase split: the same call on the same axes with a synchronise after every phase
        axes = [torch.linspace(-1.0, 1.0, res, device=dev) for _ in range(3)]

        def query(pts):
            with torch.no_grad():
                return net.engine.sdf_query(pts)[:, 0]
        ms = mesh.extract_sparse(query, axes, 0.0, brick=args.brick, lipschitz=args.lipschitz, outside=1.0, profile=True)[2]['ms']
        return {'metric': 'extract_mesh_sparse', 'resolution': res, 'brick': args.brick, 'lipschitz': args.lipschitz, 'gpu': gpu,
                'extract_mesh_sparse_ms': spread(ts), 'phases_ms': {k: round(x, 3) for k, x in ms.items()}, **stats,
                'grid_points': res ** 3, 'peak_allocated_bytes': peak,
                'fill_tflop_per_s': 2.0 * SDF_MAC_PER_POINT * stats['points_evaluated'] / (ms['fill'] * 1e-3) / 1e12}, ts

    if args.compare:
        res = args.compare
        dv, dt = net.extract_mesh(resolution=res)            # also the dense path's warm call
        sv, st = net.extract_mesh_sparse(resolution=res, brick=args.brick, lipschitz=args.lipschitz)
        same = bool(torch.equal(torch.from_numpy(dv), torch.from_numpy(sv)) and torch.equal(torch.from_numpy(dt), torch.from_numpy(st)))
        del dv, dt, sv, st
        line, _ = sparse_line(res, 1)
        td, tsp = [], []
        for _ in range(args.repeats):                        # alternated, so that both see the same state of the card
            td.append(clocked(lambda: net.extract_mesh(resolution=res))[0])
            tsp.append(clocked(lambda: net.extract_mesh_sparse(resolution=res, brick=args.brick, lipschitz=args.lipschitz))[0])
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        net.extract_mesh(resolution=res)
        line.update({'arrays_equal_dense': same, 'extract_mesh_ms': spread(td), 'extract_mesh_sparse_ms': spread(tsp),
                     'dense_peak_allocated_bytes': torch.cuda.max_memory_allocated(),
                     'speedup': sorted(td)[len(td) // 2] / sorted(tsp)[len(tsp) // 2]})
        print(json.dumps(line), flush=True)
        lines.append(line)
        if not same:
            raise SystemExit(f'bench_mesh_sparse: the sparse mesh differs from the dense mesh at {res}')
    for res in args.sparse:
        line, _ = sparse_line(res, max(1, args.repeats // 2 + 1 if res <= 1024 else 2))
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_mesh_sparse.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
