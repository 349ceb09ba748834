"""glTF export on one H100: the meshes of tools/bench_normalmap.py (the perturbed-bell 2048^3 narrow-band mesh simplified to
300 000 and 50 000 triangles, unwrapped at 2 x --size with ssaa 2) with --size^2 maps.

    python tools/bench_gltf.py [--resolution 2048] [--faces 300000 50000] [--size 1024] [--repeats 5] [--out DIR]

The object-space map is the bake of the 2048^3 mesh onto the low mesh (normalmap.bake); the material maps are synthetic
bytes (their content does not change any kernel's work).  Per line: the card's name and power limit read in the same run, the
vertex and texel counts, each kernel phase between CUDA events (median and spread of --repeats after a warm call: vertex
normals with the triangle CSR's sort, weld count + emit with the count's host read-back, tangents, raster + tangent-space
conversion + inpaint, the metallic-roughness texture), and host-clock times of the PNG / zlib encoding and of the whole
container write (glb_bytes), plus the file size.  Prints one JSON line per mesh (and writes them to DIR/bench_gltf.json with
--out).
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
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_gltf: needs a CUDA device')
    from nero_b200 import gltf as GL, normalmap as NM, params as P, synthetic
    from nero_b200 import relight as RL
    from nero_b200 import texmap as TX
    from nero_b200.renderer import NeROShapeRenderer
    from nero_b200.simplify import _vertex_triangles, simplify_cuda
    dev = torch.device('cuda', 0)
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    net = net.to(dev)
    gpu = card()
    lines = []
    fv, ft = net.extract_mesh_sparse(resolution=args.resolution)
    fv, ft = np.ascontiguousarray(fv, np.float32), np.ascontiguousarray(ft, np.int32)
    fv_d, ft_d = torch.from_numpy(fv).to(dev), torch.from_numpy(ft).to(dev)
    n = args.size
    rng = np.random.RandomState(0)
    albedo = rng.randint(0, 256, (n, n, 3)).astype(np.uint8)
    metallic, roughness = rng.randint(0, 256, (2, n, n)).astype(np.uint8)
    for F in args.faces:
        lv_d, lt_d, _ = simplify_cuda(fv_d, ft_d, F)
        lv, lt = lv_d.cpu().numpy(), lt_d.cpu().numpy()
        V, T = lv.shape[0], lt.shape[0]
        vt_atlas, ftx = TX.uv_atlas(lv, lt, 2 * n, 2 * n, 4)
        omap, _ = NM.bake(lv, lt, vt_atlas, ftx, fv, ft, n, ssaa=2)
        vt = np.stack([vt_atlas[:, 0], np.float32(1) - vt_atlas[:, 1]], -1)      # as the OBJ stores it
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        vt_d, ftx_d = up(vt), up(ftx)
        state = {}

        def normals():
            state['csr'] = _vertex_triangles(lt_d, V)
            state['n'] = NM.vertex_normals_cuda(lv_d, lt_d)

        def weld():
            state['w'] = GL.weld_cuda(lt_d, ftx_d, V, *state['csr'])

        def tangents():
            state['f'] = GL.frames_cuda(lv_d, lt_d, vt_d, ftx_d, *state['csr'], state['n'], *state['w'][:2])

        def convert():
            c = GL.tangent_space_cuda(lv, lt, vt, ftx, state['w'][2], *state['f'], omap)
            state['cov'] = int(c['raster']['texel'].shape[0])
            TX.inpaint(c['img'], c['raster']['owner'])

        def metal_rough():
            GL.metal_rough_cuda(metallic, roughness)
        times = {}
        for name, fn in (('vertex_normals', normals), ('weld', weld), ('tangents', tangents), ('tangent_space', convert),
                         ('metal_rough', metal_rough)):
            times[name + '_ms'] = spread(events(fn, args.repeats))
        prof = {}
        out = GL.export_arrays(lv, lt, vt, ftx, albedo, metallic, roughness, omap, profile=prof)
        t0 = time.perf_counter()
        pngs = [RL.png_bytes(im) for im in out['images'].values()]
        png_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        data = GL.glb_bytes(out['positions'], out['normals'], out['texcoords'], out['indices'], out['images'], out['tangents'],
                            GL.Z_UP_ROTATION)
        glb_s = time.perf_counter() - t0
        line = {'metric': 'gltf_export', 'gpu': gpu, 'triangles': T, 'positions': V, 'welded': int(out['wv'].shape[0]), 'map': n,
                'covered': state['cov'], **times, 'host_png_zlib_ms': round(png_s * 1e3, 1), 'host_container_ms': round(glb_s * 1e3, 1),
                'png_bytes': sum(len(p) for p in pngs), 'glb_bytes': len(data),
                'export_arrays_phases_ms': {k: round(v, 2) for k, v in prof.items()}}
        print(json.dumps(line), flush=True)
        lines.append(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_gltf.json'), 'w') as f:
            json.dump(lines, f, indent=1)


if __name__ == '__main__':
    main()
