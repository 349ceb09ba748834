"""Relighting on one H100: one 800x800 frame of a ~0.9 M-triangle marching-cubes mesh under a synthetic 2048x1024 map.

    python tools/bench_relight.py [--spp 64] [--bounces 4] [--repeats 3] [--out DIR]

The mesh is NeROShapeRenderer.extract_mesh at resolution 512 on the perturbed bell parameters (the field tools/bench_mesh.py
uses), with seeded random per-vertex materials.  The frame is camera 0 of the reference's default turntable (360 frames,
elevation 45 degrees, distance 3, Blender's default 50 mm camera).  Reports the median frame time over the repeats (CUDA
events around Relighter.render), camera paths/s, rays/s (counted by the kernel: camera + shadow + continuation rays), the
projected time of the reference's default job (360 frames at 1024 spp) and the card's name and power limit, read in the same
run.  Prints one JSON line (and writes it to DIR/bench_relight.json with --out).
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


def synthetic_env(h=1024, w=2048, seed=0):
    """A sky gradient, a ground colour and two bright lamps: a map with both broad and concentrated light."""
    v =(np.arange(h)[::-1, None] + 0.5) / h
    u = (np.arange(w)[None, :] + 0.5) / w
    el, phi = (v - 0.5) * np.pi, (0.5 - u) * 2 * np.pi
    d = np.stack([np.cos(el) * np.cos(phi), np.cos(el) * np.sin(phi), np.sin(el) + 0 * phi], -1)
    sky = np.where(d[..., 2:] > 0, [0.4, 0.55, 0.9] * (0.5 + 0.5 * d[..., 2:]), [0.25, 0.2, 0.15])
    for c, p in (((0.6, 0.2, 0.77), 60.0), ((-0.7, -0.5, 0.5), 25.0)):
        sky = sky + p * (np.sum(d * np.asarray(c) / np.linalg.norm(c), -1, keepdims=True) > 0.995)
    rng = np.random.RandomState(seed)
    return (sky * (1 + 0.05 * rng.rand(h, w, 1))).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--spp', type=int, default=64)
    ap.add_argument('--bounces', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_relight: needs a CUDA device')
    from nero_b200 import params as P, synthetic
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
    img = r.render(pose, K, h, w, 4, args.bounces)             # warm-up
    torch.cuda.synchronize()
    ts, rays = [], []
    for _ in range(args.repeats):
        r.rays.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        img = r.render(pose, K, h, w, args.spp, args.bounces)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
        rays.append(int(r.rays.item()))
    t = sorted(ts)[len(ts) // 2]
    paths = h * w * args.spp
    line = {'metric': 'relight_frame', 'gpu': gpu, 'vertices': V, 'triangles': int(tris.shape[0]), 'width': w, 'height': h,
            'spp': args.spp, 'bounces': args.bounces, 'frame_ms': round(t * 1e3, 2), 'frame_ms_all': [round(x * 1e3, 2) for x in ts],
            'coverage': float(img[..., 3].mean()), 'camera_paths_per_s': paths / t, 'rays': rays[0], 'rays_per_s': rays[0] / t,
            'rays_per_path': rays[0] / paths, 'reference_job_hours': 360 * t * (1024 / args.spp) / 3600.0}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_relight.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
