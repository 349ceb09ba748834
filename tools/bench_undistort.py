"""Lens undistortion on one H100: 48 synthetic RGB8 views at 1600 x 1200 of a SIMPLE_RADIAL camera with k = -0.05
(f = 0.9 w), resampled to the pinhole camera the rule picks.

    python tools/bench_undistort.py [--views 48] [--width 1600] [--height 1200] [--k -0.05] [--keypoints 8192] \\
        [--repeats 20] [--io-views 8] [--out DIR]

Per line: the card's name and power limit read in the same run, then
  * warp: per-view kernel time between CUDA events (every view once per repeat, back to back; median, min, max), and the
    algorithmic bytes, 3 read + 3 written per output pixel, over the median against the data sheet's 3.35 TB/s of HBM3
    (the four taps of a pixel mostly hit the cache, so the bytes the kernel gathers are not counted);
  * points: the keypoint inversion of --keypoints points per view;
  * host I/O per view, the part a user waits for: PNG decode (OpenCV), device upload and download, PNG encode
    (relight.write_png, stdlib zlib) and JPEG encode at quality 100 (OpenCV), over --io-views views.
Prints one JSON line per measurement (and writes them to DIR/bench_undistort.json with --out).
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
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

HBM = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=48)
    ap.add_argument('--width', type=int, default=1600)
    ap.add_argument('--height', type=int, default=1200)
    ap.add_argument('--k', type=float, default=-0.05)
    ap.add_argument('--keypoints', type=int, default=8192)
    ap.add_argument('--repeats', type=int, default=20)
    ap.add_argument('--io-views', type=int, default=8)
    ap.add_argument('--out', type=str, default=None)
    a = ap.parse_args()
    import cv2
    from nero_b200 import ops
    from nero_b200 import undistort as U
    from nero_b200.relight import write_png
    w, h, k = a.width, a.height, a.k
    f, cx, cy = 0.9 * w, w / 2, h / 2
    W, H, cx2, cy2 = U.camera(w, h, f, cx, cy, k)
    lines = [dict(card=card(), views=a.views, size=[w, h], k=k, out_size=[W, H])]
    g = torch.Generator(device='cuda').manual_seed(0)
    srcs = [torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device='cuda', generator=g) for _ in range(a.views)]
    dsts = [torch.empty(H, W, 3, dtype=torch.uint8, device='cuda') for _ in range(a.views)]

    def warp_all():
        for s, d in zip(srcs, dsts):
            ops.K('nero_undistort_image', s, w, h, f, cx, cy, k, d, W, H, cx2, cy2)

    ts = [t / a.views for t in events(warp_all, a.repeats)]
    sp = spread(ts)
    nbytes = 6 * W * H
    lines.append(dict(stage='warp', per_view_ms=sp, bytes_per_view=nbytes, gb_per_s=round(nbytes / (sp['median'] * 1e-3) / 1e9, 1),
                      share_of_hbm=round(nbytes / (sp['median'] * 1e-3) / HBM, 3)))
    rng = np.random.RandomState(1)
    xys = [torch.from_numpy(np.stack([rng.uniform(0, w, a.keypoints), rng.uniform(0, h, a.keypoints)], 1)).cuda()
           for _ in range(a.views)]
    xn = torch.empty(a.keypoints, 2, dtype=torch.float64, device='cuda')
    ok = torch.empty(a.keypoints, dtype=torch.int32, device='cuda')

    def points_all():
        for xy in xys:
            ops.K('nero_undistort_points', xy, a.keypoints, f, cx, cy, k, xn, ok)

    sp = spread([t / a.views for t in events(points_all, a.repeats)])
    lines.append(dict(stage='points', keypoints=a.keypoints, per_view_ms=sp,
                      points_per_s=float(f"{a.keypoints / (sp['median'] * 1e-3):.4g}")))
    tmp = tempfile.mkdtemp(prefix='nero_bench_undistort_')
    times = {n: [] for n in ('decode_png', 'upload', 'warp_and_download', 'encode_png', 'encode_jpeg')}
    for i in range(a.io_views):
        path = os.path.join(tmp, f'in_{i}.png')
        cv2.imwrite(path, srcs[i].cpu().numpy())
        t0 = time.perf_counter()
        rgb = np.ascontiguousarray(cv2.imread(path, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)[..., ::-1])
        t1 = time.perf_counter()
        x = torch.from_numpy(rgb).cuda()
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        out = U.image(x, f, cx, cy, k, W, H, cx2, cy2).cpu().numpy()
        t3 = time.perf_counter()
        write_png(os.path.join(tmp, f'out_{i}.png'), out)
        t4 = time.perf_counter()
        cv2.imwrite(os.path.join(tmp, f'out_{i}.jpg'), np.ascontiguousarray(out[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, 100])
        t5 = time.perf_counter()
        for n, t in zip(times, (t1 - t0, t2 - t1, t3 - t2, t4 - t3, t5 - t4)):
            times[n].append(t)
    shutil.rmtree(tmp)
    lines.append(dict(stage='host_io', io_views=a.io_views, per_view_ms={n: spread(v) for n, v in times.items()}))
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_undistort.json'), 'w') as fh:
            fh.write('\n'.join(json.dumps(ln) for ln in lines) + '\n')


if __name__ == '__main__':
    main()
