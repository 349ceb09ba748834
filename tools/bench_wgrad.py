"""Developer micro-benchmark of the weight-gradient GEMM alone (run on the GPU box).

    ROWS=127232 REPS=20 python tools/bench_wgrad.py [--peak] [--finish]

--peak adds TB/s and the share of the data-sheet HBM peak (3.35 TB/s, H100 SXM) to each shape; --finish also times the
finish (nero_wgrad_finish_batch over the shape's one job) on its own, after the GEMM.
"""
import argparse
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import torch
from nero_b200 import ops
from test_gemm_gpu import _mk_layer
ap = argparse.ArgumentParser()
ap.add_argument('--peak', action='store_true', help='report TB/s and the share of the HBM data-sheet peak')
ap.add_argument('--finish', action='store_true', help='also time the finish launch on its own')
args = ap.parse_args()
HBM_PEAK = 3.35e12
dev = torch.device('cuda')
M = int(os.environ.get('ROWS', 127232))
reps = int(os.environ.get('REPS', 20))
res = {}
for (N, K, two) in [(256, 256, False), (256, 256, True), (128, 256, False), (256, 64, False)]:
    L, W, b = _mk_layer(ops, N, K, dev)
    ws = ops.WgradWorkspace(dev)
    ws.defer = True
    dY = torch.randn(M, 256, device=dev) * 0.1
    X = torch.randn(M, 320, device=dev)
    dY2 = torch.randn(M, 256, device=dev) * 0.1 if two else None
    X2 = torch.randn(M, 320, device=dev) if two else None
    gw, gg, gb = torch.zeros_like(L.weight), torch.zeros_like(L.g), torch.zeros(N, device=dev)
    def run():
        ops.wgrad(ws, ops.Mat(dY), N, ops.Mat(X), L.k_valid, L, gw, gg, gb, ops.Mat(dY2) if two else None, ops.Mat(X2) if two else None)
        ws.jobs, ws.dest, ws.keep = [], set(), []      # time the GEMM only (no finish)
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    byts = M * (N + K) * 4 * (2 if two else 1)
    r = res[f'N{N}_K{K}_{"two" if two else "one"}'] = {'us': round(us, 1), 'GBs': round(byts / us / 1e3, 1)}
    if args.peak:
        r['TBs'] = round(byts / us / 1e6, 3)
        r['of_peak'] = round(byts / (us * 1e-6) / HBM_PEAK, 3)
    if args.finish:
        ops.wgrad(ws, ops.Mat(dY), N, ops.Mat(X), L.k_valid, L, gw, gg, gb, ops.Mat(dY2) if two else None, ops.Mat(X2) if two else None)
        jobs = list(ws.jobs)
        ws.flush()                      # uploads the job table once
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            ws.jobs = list(jobs)
            ws.flush()
        e1.record()
        torch.cuda.synchronize()
        r['finish_us'] = round(e0.elapsed_time(e1) * 1e3 / reps, 1)
print(json.dumps({'lib': os.environ.get('NERO_LIB', 'default'), **res}))
