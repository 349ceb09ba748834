"""Relit-frame denoising on one H100: the frame of tools/bench_relight.py traced with and without the feature buffers, the
filter's time, and the error of denoised and noisy frames against a converged frame.

    python tools/bench_denoise.py [--spp 64] [--bounces 4] [--repeats 5] [--reference 4096] [--out DIR]

The scene is that of tools/bench_relight.py: the 512^3 marching-cubes mesh of the perturbed bell field, seeded random
per-vertex materials, the synthetic 2048x1024 map, camera 0 of the default turntable at 800x800.
  * trace: Relighter.render (plain instance) and Relighter.render_sums (AOV instance) at --spp, alternated --repeats times
    after a warm-up, CUDA events around each call; medians and their ratio.
  * filter: denoise() at the default 5 iterations on the --spp sums, median of 20 calls (CUDA events), and its algorithmic
    bytes over that time: per iteration 25 taps x 64 B read + 16 B written per covered pixel (an uncovered pixel reads 32 B
    and writes 16 B), plus 144 B per pixel for prep and 48 B for finish.
  * quality: MSE over the fully covered pixels against a --reference spp frame traced with another seed, of the denoised
    frames at 16, 32 and 64 spp and the noisy frames at 64 and 256 spp.
Reports the card's name and power limit read in the same run.  Prints one JSON line (and writes it to DIR/bench_denoise.json
with --out).
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

from bench_mesh import card
from bench_relight import synthetic_env


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--spp', type=int, default=64)
    ap.add_argument('--bounces', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--reference', type=int, default=4096)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_denoise: needs a CUDA device')
    from nero_b200 import params as P, synthetic
    from nero_b200.denoise import denoise
    from nero_b200.relight import Relighter, blender_default_K, relight_poses
    from nero_b200.renderer import NeROShapeRenderer
    gpu = card()
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    verts, tris = net.cuda().extract_mesh(resolution=args.resolution)
    del net
    torch.cuda.empty_cache()
    V = verts.shape[0]
    rng = np.random.RandomState(1)
    mats = {'metallic': rng.rand(V, 1), 'roughness': 0.1 + 0.9 * rng.rand(V, 1), 'albedo': rng.rand(V, 3)}
    r = Relighter(verts, tris, mats, synthetic_env())
    h = w = 800
    pose, K = relight_poses(360, 0.0, 45.0, 3.0)[0], blender_default_K(h, w)
    f = float(K[0, 0])
    r.render(pose, K, h, w, 4, args.bounces)                    # warm-up of both instances and the filter
    accum, aov = r.render_sums(pose, K, h, w, 4, args.bounces)
    denoise(accum, aov, 4, f)
    torch.cuda.synchronize()
    ts = {'plain': [], 'aov': []}
    for _ in range(args.repeats):                               # alternated: both see the same clocks
        ts['plain'].append(timed(lambda: r.render(pose, K, h, w, args.spp, args.bounces))[0])
        t, (accum, aov) = timed(lambda: r.render_sums(pose, K, h, w, args.spp, args.bounces))
        ts['aov'].append(t)
    med = {k: sorted(v)[len(v) // 2] for k, v in ts.items()}
    tf = sorted(timed(lambda: denoise(accum, aov, args.spp, f))[0] for _ in range(20))
    filter_ms = tf[len(tf) // 2]
    covered = int((accum[..., 3] > 0).sum())
    iter_bytes = covered * (25 * 64 + 16) + (h * w - covered) * (32 + 16)
    filter_bytes = 5 * iter_bytes + h * w * (144 + 48)
    # quality against a converged frame of another seed
    ref = r.render(pose, K, h, w, args.reference, args.bounces, seed=1, spp_per_launch=64)
    full = ref[..., 3] == 1
    mse = {}
    for n in (16, 32, 64):
        img = r.render(pose, K, h, w, n, args.bounces, denoise=True)
        m = full & (img[..., 3] == 1)
        mse[f'denoised_{n}'] = float(((img[..., :3] - ref[..., :3])[m] ** 2).mean())
    for n in (64, 256):
        img = r.render(pose, K, h, w, n, args.bounces)
        m = full & (img[..., 3] == 1)
        mse[f'noisy_{n}'] = float(((img[..., :3] - ref[..., :3])[m] ** 2).mean())
    line = {'metric': 'relight_denoise', 'gpu': gpu, 'triangles': int(tris.shape[0]), 'width': w, 'height': h, 'spp': args.spp,
            'bounces': args.bounces, 'plain_ms': round(med['plain'], 2), 'aov_ms': round(med['aov'], 2),
            'aov_over_plain': round(med['aov'] / med['plain'], 4), 'plain_ms_all': [round(x, 2) for x in ts['plain']],
            'aov_ms_all': [round(x, 2) for x in ts['aov']], 'filter_ms': round(filter_ms, 3),
            'filter_ms_range': [round(tf[0], 3), round(tf[-1], 3)], 'covered_pixels': covered,
            'filter_bytes': filter_bytes, 'filter_GBps': round(filter_bytes / (filter_ms * 1e-3) / 1e9, 1),
            'reference_spp': args.reference, 'fully_covered_pixels': int(full.sum()), 'mse': mse}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_denoise.json'), 'w') as fo:
            json.dump(line, fo, indent=1)


if __name__ == '__main__':
    main()
