"""Shape evaluation on one H100: the synthetic-data protocol on a large mesh, and the real-data nearest-distance size.

    python tools/bench_eval.py [--repeats 5] [--views 32] [--size 800] [--points 500000] [--out DIR]

Workload 1: the ~0.9 M-triangle bell mesh of tools/bench_relight.py (extract_mesh at resolution 512 on the perturbed bell
parameters) seen from `views` cameras at size x size pixels (a ring at elevation 30 degrees and distance 3, Blender's default
50 mm camera).  Times, each as the median over the repeats between CUDA events: depth maps of all views, point compaction
of the stacked maps, voxel down-sampling (0.01), and both nearest-distance passes against a second cloud (the same mesh
scaled by 1.01, processed the same way).  Rays/s counts one ray per pixel.
Workload 2: nearest distance of `points` x `points` uniform points in a unit cube (the 500 k clouds of the real-data
protocol), reported as pair evaluations/s and as a share of the FP32 issue rate: each pair costs 9 FP32 instructions
(3 subtractions, 3 multiplications, 2 additions, 1 minimum) and the card issues SMs x 128 lanes x max SM clock of them per
second.  Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np
import torch

from bench_mesh import card, timed

FP32_OPS_PER_PAIR = 9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--views', type=int, default=32)
    ap.add_argument('--size', type=int, default=800)
    ap.add_argument('--points', type=int, default=500_000)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval: needs a CUDA device')
    from nero_b200 import evaluate as E
    from nero_b200 import params as P, synthetic
    from nero_b200.relight import blender_default_K, relight_poses
    from nero_b200.renderer import NeROShapeRenderer
    gpu = card()
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    verts, tris = net.cuda().extract_mesh(resolution=args.resolution)
    del net
    torch.cuda.empty_cache()
    h = w = args.size
    K = blender_default_K(h, w).astype(np.float32)
    views = [(p.astype(np.float32), K, (h, w)) for p in relight_poses(args.views, 0.0, 30.0, 3.0)]
    r_pr, r_gt = E.DepthRenderer(verts, tris), E.DepthRenderer(np.asarray(verts) * 1.01, tris)
    dpr = torch.empty(args.views, h, w, device='cuda')
    dgt = torch.empty_like(dpr)

    def render(r, out):
        for i, (p, K_, _) in enumerate(views):
            r.render(p, K_, h, w, out=out[i])
    poses, Ks = [v[0] for v in views], [v[1] for v in views]
    t_depth = timed(lambda: render(r_pr, dpr), args.repeats)
    render(r_gt, dgt)
    t_points = timed(lambda: E.depth_to_points_cuda(dpr, poses, Ks), args.repeats)
    pts_pr, pts_gt = E.depth_to_points_cuda(dpr, poses, Ks), E.depth_to_points_cuda(dgt, poses, Ks)
    t_voxel = timed(lambda: E.voxel_down_sample_cuda(pts_pr), args.repeats)
    cpr, cgt = E.voxel_down_sample_cuda(pts_pr).float(), E.voxel_down_sample_cuda(pts_gt).float()
    t_nn_gt = timed(lambda: E.nearest_dist_cuda(cgt, cpr), args.repeats)
    t_nn_pr = timed(lambda: E.nearest_dist_cuda(cpr, cgt), args.repeats)
    chamfer = (E.nearest_dist_cuda(cgt, cpr).mean() + E.nearest_dist_cuda(cpr, cgt).mean()).item() / 2
    total = t_depth + t_points + t_voxel + t_nn_gt + t_nn_pr

    rng = np.random.RandomState(0)
    q = torch.from_numpy(rng.rand(args.points, 3).astype(np.float32)).cuda()
    t = torch.from_numpy(rng.rand(args.points, 3).astype(np.float32)).cuda()
    t_real = timed(lambda: E.nearest_dist_cuda(q, t), args.repeats)
    pairs = float(args.points) * args.points
    props = torch.cuda.get_device_properties(0)
    try:
        clock_hz = float(gpu.split(',')[2].split()[0]) * 1e6
    except (IndexError, ValueError):
        clock_hz = float('nan')
    issue = props.multi_processor_count * 128 * clock_hz
    ms = lambda x: round(x * 1e3, 3)
    line = {'metric': 'eval_shape', 'gpu': gpu, 'sms': props.multi_processor_count, 'triangles': int(tris.shape[0]),
            'views': args.views, 'width': w, 'height': h,
            'depth_ms': ms(t_depth), 'rays_per_s': args.views * h * w / t_depth, 'points_ms': ms(t_points),
            'points_pr': int(pts_pr.shape[0]), 'voxel_ms': ms(t_voxel), 'voxels_pr': int(cpr.shape[0]), 'voxels_gt': int(cgt.shape[0]),
            'nearest_gt_ms': ms(t_nn_gt), 'nearest_pr_ms': ms(t_nn_pr), 'protocol_ms': ms(total), 'chamfer': chamfer,
            'real_points': args.points, 'real_nearest_ms': ms(t_real), 'real_pairs_per_s': pairs / t_real,
            'real_fp32_issue_share': pairs * FP32_OPS_PER_PAIR / t_real / issue}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_eval.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
