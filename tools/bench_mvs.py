"""Time dense multi-view stereo (nero_b200.mvs) on a synthetic project: grey preparation, PatchMatch and the geometric
filter per view, and the whole reconstruction.

    python tools/bench_mvs.py [--views 48] [--width 1600] [--height 1200] [--sources 8] [--iterations 8] [--repeat 2]

The project is the table / box / sphere scene of oracle/nero_oracle_mvs.py, rendered on the CPU into a temporary
directory (not timed).  Work counts are computed from the shapes: a pass evaluates at most 11 hypotheses per pixel of its
colour (the current one reuses its stored cost; neighbours that leave the depth range or face away are skipped), the
initialisation one per pixel, each against S sources with (2r/step + 1)^2 bilinear samples.  So the rates below are
upper bounds of the work done per second.  The card's name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else 'unknown'
    except (OSError, subprocess.SubprocessError):
        return 'unknown'


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--views', type=int, default=48)
    ap.add_argument('--width', type=int, default=1600)
    ap.add_argument('--height', type=int, default=1200)
    ap.add_argument('--sources', type=int, default=8)
    ap.add_argument('--iterations', type=int, default=8)
    ap.add_argument('--repeat', type=int, default=2)
    ap.add_argument('--json', type=str, default=None, help='also write the result here')
    a = ap.parse_args()
    import numpy as np
    import torch
    import nero_oracle_mvs as OM
    from nero_b200 import mvs, objprep
    tmp = tempfile.mkdtemp(prefix='bench_mvs_')
    t0 = time.time()
    OM.project(tmp, a.views, a.width, a.height, seed=0, per_view=80, cell=0.01, workers=max(1, os.cpu_count() or 1))
    t_render = time.time() - t0
    views, pts, tracks = objprep.read_colmap_model(os.path.join(tmp, 'sparse', '0'), tracks=True)
    reader = mvs.image_reader(os.path.join(tmp, 'images'))
    items = sorted(views.items(), key=lambda kv: kv[1][0])
    poses = np.stack([v[1] for _, v in items])
    _, plan = mvs.select_sources(pts, tracks, poses, [i for i, _ in items], a.sources)
    rgbs = [torch.from_numpy(reader(v[0])).cuda() for _, v in items]
    Ks = [mvs.scale_K(v[2], mvs.grey_scale(a.width, a.height)) for _, v in items]
    ev = lambda: torch.cuda.Event(enable_timing=True)

    def timed(fn):
        e0, e1 = ev(), ev()
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        return out, e0.elapsed_time(e1)

    # warm-up: every kernel once at the timed shapes
    s = mvs.grey_scale(a.width, a.height)
    greys = [mvs.prepare_grey(x, s) for x in rgbs]
    use = [i for i, e in enumerate(plan) if not e['skip']]
    i0 = use[0]
    src0 = plan[i0]['sources']
    geo0 = mvs.pm_table(Ks[i0], poses[i0], [Ks[j] for j in src0], [poses[j] for j in src0])
    mvs.patchmatch(greys[i0], Ks[i0], [greys[j] for j in src0], geo0, plan[i0]['range'], i0, 1)
    torch.cuda.synchronize()
    res = {'t_prep': [], 't_pm': [], 't_filter': [], 't_total': [], 'samples': 0, 'hyps': 0}
    for rep in range(a.repeat):
        greys, t = timed(lambda: [mvs.prepare_grey(x, s) for x in rgbs])
        res['t_prep'].append(t / len(rgbs))
        planes, cost, t_pm, samples, hyps = {}, {}, 0.0, 0, 0
        for i in use:
            src = plan[i]['sources']
            geo = mvs.pm_table(Ks[i], poses[i], [Ks[j] for j in src], [poses[j] for j in src])
            (planes[i], cost[i]), t = timed(lambda: mvs.patchmatch(greys[i], Ks[i], [greys[j] for j in src], geo, plan[i]['range'], i,
                                                                   a.iterations))
            t_pm += t
            h, w = greys[i].shape
            n_h = h * w * (1 + 11 * a.iterations)
            hyps += n_h
            samples += n_h * len(src) * (2 * mvs.RADIUS // mvs.STEP + 1) ** 2
        res['t_pm'].append(t_pm / len(use))
        t_f = 0.0
        for i in use:
            src = [(Ks[j], poses[j], planes[j], cost[j]) for j in plan[i]['sources'] if j in planes]
            (d, _), t = timed(lambda: mvs.geometric_filter(Ks[i], poses[i], planes[i], cost[i], src))
            t_f += t
        res['t_filter'].append(t_f / len(use))
        torch.cuda.synchronize()
        t1 = time.time()
        cloud, info = mvs.reconstruct(views, pts, tracks, reader, iterations=a.iterations, sources=a.sources)
        torch.cuda.synchronize()
        res['t_total'].append((time.time() - t1) * 1e3)
        res['samples'], res['hyps'] = samples, hyps
    best = lambda k: min(res[k])
    out = dict(card=card(), views=a.views, width=a.width, height=a.height, sources=a.sources, iterations=a.iterations,
               views_reconstructed=len(use), fused_points=int(info['fused']), render_s=round(t_render, 1),
               prep_ms_per_view=round(best('t_prep'), 3), patchmatch_ms_per_view=round(best('t_pm'), 2),
               filter_ms_per_view=round(best('t_filter'), 3), end_to_end_s=round(best('t_total') / 1e3, 2),
               end_to_end_s_per_view=round(best('t_total') / 1e3 / a.views, 3),
               hypotheses_per_s_upper=f'{res["hyps"] / (best("t_pm") * len(use) / 1e3):.3e}',
               samples_per_s_upper=f'{res["samples"] / (best("t_pm") * len(use) / 1e3):.3e}',
               repeats_ms_pm=[round(x, 2) for x in res['t_pm']])
    shutil.rmtree(tmp)
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
