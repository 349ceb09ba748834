"""UV texture-map export on one H100: the reference's default job (1024^2 output, ssaa 2, a 2048^2 atlas) on the ~0.9 M-triangle
marching-cubes bell mesh of tools/bench_relight.py with the perturbed stage-II parameters.

    python tools/bench_texmap.py [--size 1024] [--ssaa 2] [--repeats 3] [--out DIR]

Times each stage separately: the host unwrap (a CPU number, wall clock), then raster, compaction (count + scan + the one
read of the total + emit, with the uploads of the atlas and the mesh), materials (the stage-II material chain in batches of 2^18 rows), encode, inpaint, down-sample
(CUDA events, median over warm repeats) and the file writes (wall clock).  Reports the covered-texel count, the algorithmic
MLP FLOP/s (2 x 1 078 272 MAC per row) and the card's name and power limit, read in the same run.  Prints one JSON line (and
writes it to DIR/bench_texmap.json with --out).
"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

from bench_mesh import card

MAT_MAC_PER_ROW = 1078272        # feats network + three predictors per point (nero_b200/material.py)


def timed(fn, repeats):
    """(median seconds between CUDA events after one warm call, last result)"""
    out = fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e-3)
    return sorted(ts)[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--ssaa', type=int, default=2)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_texmap: needs a CUDA device')
    from nero_b200 import params as P, synthetic
    from nero_b200 import texmap as TX
    from nero_b200.material import NeROMaterialRenderer
    from nero_b200.renderer import NeROShapeRenderer
    gpu = card()
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    verts, tris = net.cuda().extract_mesh(resolution=args.resolution)
    del net
    torch.cuda.empty_cache()
    scfg = {'human_lights': False}
    mnet = NeROMaterialRenderer({'shader_cfg': scfg}, is_train=False, mesh=(verts, tris))
    mnet.load_state_dict(synthetic.perturb_params(P.build_material_state_dict(scfg, seed=6033)))
    mnet = mnet.cuda()
    n = args.size * args.ssaa
    t0 = time.time()
    vt, ft = TX.uv_atlas(verts, tris, n, n, 2 * args.ssaa)
    t_unwrap = time.time() - t0
    t_raster, r = timed(lambda: TX.raster(vt, ft, verts, tris, n, n), args.repeats)   # raster + compaction, split below
    import numpy as np
    from nero_b200 import ops
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    vt_d, ft_d = up(vt, np.float32), up(ft, np.int32)
    owner, cover = torch.empty(n * n, dtype=torch.int32, device='cuda'), torch.empty(n * n, dtype=torch.int32, device='cuda')
    t_rast, _ = timed(lambda: ops.K('nero_tex_raster', vt_d, ft_d, ft_d.shape[0], n, n, owner, cover), args.repeats)
    covered = int(r['texel'].shape[0])
    mnet.engine.prepare_weights()
    t_mat, mat = timed(lambda: TX.query_materials(mnet, r['xyz']), args.repeats)
    t_enc, img = timed(lambda: TX.encode(mat, r['texel'], n, n), args.repeats)
    t_inp, (img2, _) = timed(lambda: TX.inpaint(img, r['owner']), args.repeats)
    t_ds, small = timed(lambda: TX.downsample(img2), args.repeats) if args.ssaa == 2 else (0.0, img2)
    images = TX.split_images(small)
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.time()
        TX.write_textured_obj(tmp, verts, tris, vt, ft, images)
        t_write = time.time() - t0
    flops = 2.0 * MAT_MAC_PER_ROW * covered
    line = {'metric': 'texmap_export', 'gpu': gpu, 'vertices': int(verts.shape[0]), 'triangles': int(tris.shape[0]), 'atlas': n,
            'size': args.size, 'ssaa': args.ssaa, 'uv_vertices': int(vt.shape[0]), 'covered_texels': covered,
            'unwrap_host_s': round(t_unwrap, 3), 'raster_ms': round(t_rast * 1e3, 3),
            'upload_compaction_ms': round((t_raster - t_rast) * 1e3, 3), 'materials_ms': round(t_mat * 1e3, 3),
            'mlp_tflops': round(flops / t_mat / 1e12, 2), 'encode_ms': round(t_enc * 1e3, 3), 'inpaint_ms': round(t_inp * 1e3, 3),
            'downsample_ms': round(t_ds * 1e3, 3), 'write_s': round(t_write, 3),
            'gpu_total_ms': round((t_raster + t_mat + t_enc + t_inp + t_ds) * 1e3, 2)}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_texmap.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
