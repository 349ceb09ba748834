"""Relighting from UV textures against per-vertex materials on one H100: the frame of tools/bench_relight.py rendered both ways.

    python tools/bench_relight_textured.py [--spp 64] [--bounces 4] [--repeats 3] [--size 1024] [--out DIR]

The mesh, the random per-vertex materials, the synthetic 2048x1024 map and the camera are those of tools/bench_relight.py
(camera 0 of the default turntable, 800x800).  The textured scene unwraps the mesh into a size^2 atlas with texmap.uv_atlas
(gutter 2) and fills each covered texel with the mean of its triangle's three vertex materials (roughness squared, since a
texture holds alpha itself); uncovered texels stay 0.  The two kernels are timed alternately in one run (CUDA events around
Relighter.render), so clock and power drift affect both alike.  Reports the median frame time of each, their ratio and the
card's name and power limit, read in the same run.  Prints one JSON line (and writes it to DIR/bench_relight_textured.json
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


def texture_from_vertices(verts, tris, vt, ft, mats, size):
    """[size,size] maps (row 0 = v_atlas 0, the file's top row): each covered texel holds its triangle's mean material."""
    from nero_b200 import texmap as TX
    r = TX.raster(vt, ft, verts, tris, size, size)
    owner = r['owner'].cpu().numpy().reshape(-1)
    cov = owner >= 0
    tri_mean = lambda a: np.asarray(a, np.float64).reshape(verts.shape[0], -1)[tris].mean(1)
    out = {}
    for k, a in (('albedo', mats['albedo']), ('metallic', mats['metallic']), ('roughness', np.asarray(mats['roughness']) ** 2)):
        m = tri_mean(a)
        img = np.zeros((size * size, m.shape[1]), np.float32)
        img[cov] = m[owner[cov]]
        out[k] = img.reshape(size, size, -1)
    return out, float(cov.mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--spp', type=int, default=64)
    ap.add_argument('--bounces', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_relight_textured: needs a CUDA device')
    from nero_b200 import params as P, synthetic
    from nero_b200 import texmap as TX
    from nero_b200.relight import Relighter, UVMaterials, blender_default_K, relight_poses
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
    vt, ft = TX.uv_atlas(verts, tris, args.size, args.size, 2)
    maps, tex_cover = texture_from_vertices(verts, tris, vt, ft, mats, args.size)
    vt_file = np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], -1)
    env = synthetic_env()
    renderers = {'vertex': Relighter(verts, tris, mats, env),
                 'textured': Relighter(verts, tris, UVMaterials(vt_file, ft, maps['albedo'], maps['metallic'], maps['roughness']), env)}
    h = w = 800
    pose, K = relight_poses(360, 0.0, 45.0, 3.0)[0], blender_default_K(h, w)
    for r in renderers.values():
        r.render(pose, K, h, w, 4, args.bounces)                # warm-up
    torch.cuda.synchronize()
    ts = {k: [] for k in renderers}
    imgs, rays = {}, {}
    for _ in range(args.repeats):
        for k, r in renderers.items():                          # alternated: both see the same clocks
            r.rays.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            imgs[k] = r.render(pose, K, h, w, args.spp, args.bounces)
            e1.record()
            torch.cuda.synchronize()
            ts[k].append(e0.elapsed_time(e1))
            rays[k] = int(r.rays.item())
    med = {k: sorted(v)[len(v) // 2] for k, v in ts.items()}
    line = {'metric': 'relight_textured_frame', 'gpu': gpu, 'vertices': V, 'triangles': int(tris.shape[0]), 'texture': args.size,
            'uv_vertices': int(vt.shape[0]), 'texels_covered': round(tex_cover, 4), 'width': w, 'height': h, 'spp': args.spp,
            'bounces': args.bounces, 'vertex_ms': round(med['vertex'], 2), 'textured_ms': round(med['textured'], 2),
            'textured_over_vertex': round(med['textured'] / med['vertex'], 4),
            'vertex_ms_all': [round(x, 2) for x in ts['vertex']], 'textured_ms_all': [round(x, 2) for x in ts['textured']],
            'coverage': float(imgs['textured'][..., 3].mean()), 'rays_vertex': rays['vertex'], 'rays_textured': rays['textured']}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_relight_textured.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
