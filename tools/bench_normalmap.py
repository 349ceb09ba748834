"""Normal-map bake on one H100: the perturbed-bell 2048^3 narrow-band mesh (the mesh of tools/bench_simplify.py)
simplified to 300 000 and 50 000 triangles, unwrapped at 1024^2 with ssaa 2 (a 2048^2 atlas), and baked against the
2048^3 mesh.

    python tools/bench_normalmap.py [--resolution 2048] [--faces 300000 50000] [--size 1024] [--repeats 5] [--spp 256] [--out DIR]

Per line: the card's name and power limit read in the same run, then
  * times: the vertex normals of the detail and the low mesh (the triangle CSR's torch sort included), the bake kernel
    (CUDA events, median of --repeats; rays/s = covered texels / time), inpaint + down-sample, and the host BVH build of
    the detail mesh; the hit / miss counts;
  * quality: camera 0 of the default turntable at 800^2, --spp samples, 4 bounces, the synthetic map of bench_relight.py,
    grey diffuse-dominated materials (albedo 0.5, metallic 0, alpha 0.3) on every mesh.  MSE against the 2048^3 mesh's frame
    of the low mesh shaded flat and of the low mesh with its map, over the pixels all three frames cover fully.
Prints one JSON line per measurement (and writes them to DIR/bench_normalmap.json with --out).
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
from bench_relight import synthetic_env


def events(fn, repeats):
    """seconds of each of `repeats` calls of fn() between CUDA events, after one warm call"""
    fn()
    out = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        out.append(e0.elapsed_time(e1) * 1e-3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--resolution', type=int, default=2048)
    ap.add_argument('--faces', type=int, nargs='*', default=[300000, 50000])
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--spp', type=int, default=256)
    ap.add_argument('--image', type=int, default=800)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_normalmap: needs a CUDA device')
    from nero_b200 import normalmap as NM, ops, params as P, synthetic
    from nero_b200 import relight as RL
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
    h = w = args.image
    pose, K = RL.relight_poses(360, 0.0, 45.0, 3.0)[0], RL.blender_default_K(h, w)
    env = synthetic_env()
    V = fv.shape[0]
    grey = {'albedo': np.full((V, 3), 0.5, np.float32), 'metallic': np.zeros((V, 1), np.float32),
            'roughness': np.full((V, 1), np.sqrt(0.3), np.float32)}
    t0 = time.perf_counter()
    ref = RL.Relighter(fv, ft, grey, env).render(pose, K, h, w, args.spp, 4, seed=0).cpu().numpy().astype(np.float64)
    ref_s = time.perf_counter() - t0
    for F in args.faces:
        lv, lt, _ = simplify_cuda(fv_d, ft_d, F)
        lv_d, lt_d = lv, lt
        lv, lt = lv.cpu().numpy(), lt.cpu().numpy()
        n = args.size
        t0 = time.perf_counter()
        vt, ftx = TX.uv_atlas(lv, lt, 2 * n, 2 * n, 4)
        atlas_s = time.perf_counter() - t0
        prof = {}
        b = NM.bake_cuda(lv, lt, vt, ftx, fv, ft, n, ssaa=2, profile=prof)
        cov = int(b['hit'].shape[0])
        hits = int(b['hit'].sum())
        normals_detail = spread(events(lambda: NM.vertex_normals_cuda(fv_d, ft_d), args.repeats))
        normals_low = spread(events(lambda: NM.vertex_normals_cuda(lv_d, lt_d), args.repeats))
        bake_t = events(lambda: ops.K('nero_normalmap_bake', *b['args']), args.repeats)
        post = spread(events(lambda: TX.downsample(TX.inpaint(b['img'], b['raster']['owner'])[0]), args.repeats))
        img, stats = NM.bake(lv, lt, vt, ftx, fv, ft, n, ssaa=2)
        emit({'metric': 'normalmap_bake', 'gpu': gpu, 'detail_triangles': int(ft.shape[0]), 'low_triangles': int(lt.shape[0]),
              'atlas': 2 * n, 'map': n, 'covered': cov, 'hits': hits, 'misses': cov - hits, 'miss_fraction': round((cov - hits) / cov, 6),
              'vertex_normals_detail_ms': normals_detail, 'vertex_normals_low_ms': normals_low, 'bake_kernel_ms': spread(bake_t),
              'bake_rays_per_s': round(cov / sorted(bake_t)[len(bake_t) // 2], 1), 'inpaint_downsample_ms': post,
              'bvh_build_host_detail_s': round(prof['bvh'] * 1e-3, 3), 'uv_atlas_host_s': round(atlas_s, 3)})
        vt_file = np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], -1)
        full = lambda c: np.full((n, n) + c, 1.0, np.float32)
        flat = RL.UVMaterials(vt_file, ftx, full((3,)) * 0.5, full(()) * 0, full(()) * 0.3)
        mapped = RL.UVMaterials(vt_file, ftx, flat.albedo, flat.metallic, flat.roughness, normal=NM.decode(img))
        frames = []
        for m in (flat, mapped):
            frames.append(RL.Relighter(lv, lt, m, env).render(pose, K, h, w, args.spp, 4, seed=0).cpu().numpy().astype(np.float64))
        both = (ref[..., 3] == 1) & (frames[0][..., 3] == 1) & (frames[1][..., 3] == 1)
        mse = [float(((f[..., :3] - ref[..., :3]) ** 2)[both].mean()) for f in frames]
        emit({'metric': 'normalmap_quality', 'gpu': gpu, 'low_triangles': int(lt.shape[0]), 'detail_triangles': int(ft.shape[0]),
              'image': h, 'spp': args.spp, 'pixels': int(both.sum()), 'mse_flat': mse[0], 'mse_mapped': mse[1],
              'gain': round(mse[0] / mse[1], 3), 'detail_frame_s': round(ref_s, 2)})
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_normalmap.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
