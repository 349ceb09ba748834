"""Mesh extraction on one H100: NeROShapeRenderer.extract_mesh on the perturbed bell parameters, at resolution 512
(extract_mesh.py's default) and 128 (val_geometry).

    python tools/bench_mesh.py [--resolutions 512 128] [--repeats 5] [--out DIR]

Per resolution: the SDF grid fill (engine.sdf_query in x-slabs), the marching-cubes kernels (count + scan + the one read of
the totals + emit; CUDA events over warm repeats), and extract_mesh end to end (host clock around a synchronised call).
The kernels' algorithmic bytes are the field read once plus 12 B per vertex and 12 B per triangle written; they are set
against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.  The card's name and power limit are read in the same run.
Prints one JSON line per resolution (and writes them to DIR/bench_mesh.json with --out).
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch

HBM_BYTES_PER_S = 3.35e12
SDF_MAC_PER_POINT = 524544      # SDFNetwork forward per query point (SURVEY.md section 8)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def timed(fn, repeats):
    """median seconds of fn() between CUDA events, after one warm call"""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    return sorted(ts)[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--resolutions', type=int, nargs='+', default=[512, 128])
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_mesh: needs a CUDA device')
    from nero_b200 import params as P, synthetic
    from nero_b200.mesh import marching_cubes_cuda
    from nero_b200.renderer import NeROShapeRenderer
    dev = torch.device('cuda', 0)
    cfg = {}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict(cfg, seed=6033)))
    net = net.to(dev)
    gpu = card()
    lines = []
    for res in args.resolutions:
        b = (-1.0, -1.0, -1.0), (1.0, 1.0, 1.0)
        t_fill = timed(lambda: net._fill_grid(*b, res), max(1, args.repeats // 2))
        u = net._fill_grid(*b, res)
        out = {}

        def cubes():
            out['v'], out['t'] = marching_cubes_cuda(u, 0.0)
        t_cubes = timed(cubes, args.repeats)
        V, T = out['v'].shape[0], out['t'].shape[0]
        del out['v'], out['t'], u
        torch.cuda.synchronize()
        net.extract_mesh(resolution=res)
        torch.cuda.synchronize()
        e2e = []
        for _ in range(max(1, args.repeats // 2)):
            t0 = time.perf_counter()
            net.extract_mesh(resolution=res)
            torch.cuda.synchronize()
            e2e.append(time.perf_counter() - t0)
        t_e2e = sorted(e2e)[len(e2e) // 2]
        n_pts = res ** 3
        n_cubes = (res - 1) ** 3
        alg_bytes = 4 * n_pts + 12 * V + 12 * T
        line = {'metric': 'extract_mesh', 'resolution': res, 'gpu': gpu, 'vertices': V, 'triangles': T,
                'field_fill_ms': round(t_fill * 1e3, 3), 'cube_kernels_ms': round(t_cubes * 1e3, 3),
                'extract_mesh_ms': round(t_e2e * 1e3, 3), 'cubes_per_s': n_cubes / t_cubes,
                'cube_kernels_alg_bytes': alg_bytes, 'cube_kernels_tb_per_s': alg_bytes / t_cubes / 1e12,
                'cube_kernels_frac_of_3p35': alg_bytes / t_cubes / HBM_BYTES_PER_S,
                'field_fill_tflop_per_s': 2.0 * SDF_MAC_PER_POINT * n_pts / t_fill / 1e12}
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_mesh.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
