"""Per-launch profile of the weight-gradient pass of one training step (run on the GPU box).

    python tools/profile_wgrad.py [--workload bell|bear] [--out DIR] [--table]     # NERO_LIB=... selects another build

Warms up three resident steps of the bench workload, then records one more under torch.profiler (CUDA activities).  Every
`gemm_wgrad_kernel<NW>` launch is matched, in issue order, to the `nero_wgrad` call that made it, which gives its rows
(the device count, read after the step), NW, number of pairs and output rows.  Algorithmic bytes of a launch = each
operand read once (dY columns [0, n_valid), X columns [k0, k0 + NW) clipped to k_valid, per pair) + the slice windows
written once (P x rows x NW fp32 + the bias sums).  Also reported: `nero_wgrad_finish_batch`, the accumulator memsets
(torch fill / zero kernels) and the step total, with the GPU name and power limit of the run.  Prints one JSON line;
`--table` also prints one line per kernel (launches, time, algorithmic GB, TB/s and share of the data-sheet HBM peak),
the finish on a line of its own.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    sys.path.insert(0, p)
import torch
from torch.profiler import profile, ProfilerActivity

import bench
from nero_b200 import ops

HBM_PEAK = 3.35e12      # NVIDIA H100 SXM data sheet, 700 W


def gpu_info():
    try:
        o = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=10).stdout.strip().splitlines()[0]
        name, pl, clk = [s.strip() for s in o.split(',')]
        return {'name': name, 'power_limit': pl, 'max_sm_clock': clk}
    except Exception as e:        # noqa: BLE001
        return {'error': str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='bell', choices=['bell', 'bear'])
    ap.add_argument('--out', default=None, help='also write the JSON and the kernel table here')
    ap.add_argument('--table', action='store_true', help='also print a per-kernel table (time, bytes, TB/s, share of peak)')
    args = ap.parse_args()
    dev = torch.device('cuda')
    wl = bench.Workload(args.workload == 'bear', 0, 1, dev)
    for _ in range(3):
        wl.resident_step()
    torch.cuda.synchronize()

    calls = []
    k_orig = ops.K

    def k_rec(name, *a, **kw):
        if name == 'nero_wgrad':
            dY, ldy, n_valid, X, ldx, k_valid, dY2 = a[:7]
            n_rows_pad, k_pad, P, m_ptr, m_cap = a[14:19]
            calls.append(dict(n_valid=n_valid, k_valid=k_valid, pairs=2 if dY2 is not None else 1, n_rows_pad=n_rows_pad,
                              k_pad=k_pad, P=P, m_ptr=m_ptr, m_cap=m_cap))
        return k_orig(name, *a, **kw)

    ops.K = k_rec         # ops.wgrad looks K up in its module at call time
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            wl.resident_step()
            torch.cuda.synchronize()
    finally:
        ops.K = k_orig
    evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA], key=lambda e: e.time_range.start)
    step_us = (evs[-1].time_range.end - evs[0].time_range.start) if evs else 0.0
    busy_us = sum(e.device_time for e in evs)

    # expected launch sequence: each nero_wgrad call covers k_pad with 256-, then 128-, then 64-column launches
    launches = []
    for c in calls:
        M = c['m_cap']
        if isinstance(c['m_ptr'], torch.Tensor):
            M = min(int(c['m_ptr'].reshape(-1)[0].item()), c['m_cap'])
        n_tiles = (c['n_rows_pad'] + 127) // 128
        k0 = 0
        while k0 < c['k_pad']:
            rem = c['k_pad'] - k0
            nw = 256 if rem >= 256 else 128 if rem >= 128 else 64
            xcols = max(0, min(nw, c['k_valid'] - k0))
            rows_out = min(n_tiles * 128, 256)
            byts = c['pairs'] * M * (c['n_valid'] + xcols) * 4 + c['P'] * rows_out * (nw + (1 if k0 == 0 else 0)) * 4
            launches.append(dict(NW=nw, rows=M, pairs=c['pairs'], n_out=c['n_valid'], tiles=n_tiles, bytes=byts))
            k0 += nw
    wk = [e for e in evs if 'gemm_wgrad_kernel' in e.name]
    matched = len(wk) == len(launches)
    for l, e in zip(launches, wk):
        l['us'] = round(e.device_time, 1)
        l['TBs'] = round(l['bytes'] / (e.device_time * 1e-6) / 1e12, 3)
        l['frac_of_hbm_peak'] = round(l['bytes'] / (e.device_time * 1e-6) / HBM_PEAK, 3)

    def agg(pred):
        sel = [e for e in evs if pred(e.name)]
        return {'launches': len(sel), 'ms': round(sum(e.device_time for e in sel) / 1e3, 3)}

    by_nw = {}
    for l in launches:
        d = by_nw.setdefault(f'gemm_wgrad_kernel<{l["NW"]}>', {'launches': 0, 'us': 0.0, 'bytes': 0})
        d['launches'] += 1
        d['us'] += l.get('us', 0.0)
        d['bytes'] += l['bytes']
    for d in by_nw.values():
        d['ms'] = round(d.pop('us') / 1e3, 3)
        d['TBs'] = round(d['bytes'] / (d['ms'] * 1e-3) / 1e12, 3) if d['ms'] else None
    fill = lambda n: ('FillFunctor' in n or 'Zero' in n or 'zero' in n or 'Memset' in n) and 'gemm' not in n
    res = {'lib': os.environ.get('NERO_LIB', 'default'), 'workload': args.workload, 'gpu': gpu_info(),
           'counts': dict(zip(('n_in', 'n_out', 'p_occ'), wl.counts())),
           'step_span_ms': round(step_us / 1e3, 3), 'kernel_busy_ms': round(busy_us / 1e3, 3),
           'wgrad_calls': len(calls), 'wgrad_launches': len(wk), 'matched': matched, 'wgrad_by_nw': by_nw,
           'finish_batch': agg(lambda n: 'wgrad_finish_batch' in n), 'finish_single': agg(lambda n: 'wgrad_finish_kernel' in n),
           'memsets': agg(fill), 'slot_memsets': agg(lambda n: 'multi_tensor_apply' in n),
           'wgrad_pass_ms': round(sum(d['ms'] for d in by_nw.values()) + agg(lambda n: 'wgrad_finish' in n)['ms'] + agg(fill)['ms'], 3)}
    top = {}
    for e in evs:
        t = top.setdefault(e.name[:90], [0, 0.0])
        t[0] += 1
        t[1] += e.device_time
    res['top_kernels'] = [[k, n, round(us / 1e3, 3)] for k, (n, us) in sorted(top.items(), key=lambda kv: -kv[1][1])[:14]]
    print(json.dumps(res))
    if args.table:
        print(f'# {res["gpu"].get("name")} at {res["gpu"].get("power_limit")}, peak {HBM_PEAK / 1e12:.2f} TB/s (data sheet)')
        print(f'{"kernel":28s} {"launches":>8s} {"ms":>8s} {"GB":>8s} {"TB/s":>7s} {"of peak":>8s}')
        for k, d in sorted(by_nw.items()):
            tbs = d['bytes'] / (d['ms'] * 1e-3) / 1e12 if d['ms'] else 0.0
            print(f'{k:28s} {d["launches"]:8d} {d["ms"]:8.3f} {d["bytes"] / 1e9:8.2f} {tbs:7.3f} {tbs * 1e12 / HBM_PEAK:8.1%}')
        fb = res['finish_batch']
        print(f'{"nero_wgrad_finish_batch":28s} {fb["launches"]:8d} {fb["ms"]:8.3f}')
        print(f'{"whole pass":28s} {"":8s} {res["wgrad_pass_ms"]:8.3f}')
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f'wgrad_{args.workload}_{os.path.basename(res["lib"])}.json'), 'w') as f:
            json.dump({**res, 'launches': launches}, f, indent=1)


if __name__ == '__main__':
    main()
