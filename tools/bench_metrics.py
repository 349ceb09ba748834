"""Image metrics on one H100: quantisation + exact PSNR + SSIM of 32 views at 800 x 800 x 3, the size of the GlossySynthetic
test split, on the GPU and in the CPU oracle.

    python tools/bench_metrics.py [--views 32] [--size 800] [--repeats 5] [--cpu-views 2] [--out DIR]

GPU: CUDA events around the whole batch (median over warm repeats): fp32 renders -> uint8 (nero_metrics_quantize), then
nero_b200.metrics.psnr and ssim on the [32, 800, 800, 3] batch, each stage alone and the three together (psnr and ssim
each read their result back to the host once).  CPU: the numpy / scipy oracle (oracle/nero_oracle_metrics.py) on
--cpu-views views, scaled to the batch.  Prints the card's name, power limit and maximum SM clock read in the same run, and
one JSON line (also written to DIR/bench_metrics.json with --out).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools'), os.path.join(ROOT, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

from bench_mesh import card
from bench_texmap import timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--views', type=int, default=32)
    ap.add_argument('--size', type=int, default=800)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--cpu-views', type=int, default=2)
    ap.add_argument('--out', type=str, default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_metrics: needs a CUDA device')
    import nero_oracle_metrics as OM
    from nero_b200 import metrics as M

    name = card()
    print(name)
    B, S = a.views, a.size
    g = torch.Generator(device='cuda').manual_seed(0)
    gt = torch.rand(B, S, S, 3, device='cuda', generator=g)
    pr = (gt + 0.05 * torch.randn(B, S, S, 3, device='cuda', generator=g)).clamp_(-0.1, 1.1)
    qg, qp = M.color_map_backward(gt), M.color_map_backward(pr)

    t_quant, _ = timed(lambda: (M.color_map_backward(gt), M.color_map_backward(pr)), a.repeats)
    t_psnr, p = timed(lambda: M.psnr(qg, qp), a.repeats)
    t_ssim, s = timed(lambda: M.ssim(qg, qp), a.repeats)

    def all_three():
        g8, p8 = M.color_map_backward(gt), M.color_map_backward(pr)
        return M.psnr(g8, p8), M.ssim(g8, p8)
    t_all, (p2, s2) = timed(all_three, a.repeats)
    assert np.array_equal(p, p2) and np.array_equal(s, s2)

    n = min(a.cpu_views, B)
    hg, hp = gt[:n].cpu().numpy(), pr[:n].cpu().numpy()
    t0 = time.perf_counter()
    for i in range(n):
        og, op = OM.color_map_backward(hg[i]), OM.color_map_backward(hp[i])
        ops_ = (OM.psnr_exact(og, op), OM.ssim(og, op))
    t_cpu = (time.perf_counter() - t0) / n * B
    assert ops_[0] == p[n - 1] and abs(ops_[1] - s[n - 1]) <= 1e-12

    # bytes the algorithm needs: quantise 4 B in + 1 B out per value and image; SSE 2 B; SSIM 2 B in, 5 fp64 planes written
    # and read once, 16 B of S map not stored
    vals = B * S * S * 3
    res = {'card': name, 'views': B, 'size': S, 'quantize_ms': t_quant * 1e3, 'psnr_ms': t_psnr * 1e3, 'ssim_ms': t_ssim * 1e3,
           'total_ms': t_all * 1e3, 'cpu_oracle_s': t_cpu, 'speedup': t_cpu / t_all,
           'ssim_gb_per_s': (vals * (2 + 5 * 8 * 2)) / t_ssim * 1e-9, 'mean_psnr': float(np.mean(p)), 'mean_ssim': float(np.mean(s))}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'bench_metrics.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
