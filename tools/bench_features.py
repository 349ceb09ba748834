"""Time sparse features (nero_b200.features) on a synthetic project: extraction per view, all-pair matching with its
achieved int8 rate, verification and the database write.

    python tools/bench_features.py [--views 48] [--width 1600] [--height 1200] [--max-features 8192] [--repeat 2]

The project is the table / box / sphere scene of oracle/nero_oracle_mvs.py that tools/bench_mvs.py uses, rendered on the
CPU into a temporary directory (not timed).  The matcher's work is counted from the shapes: both directions of every pair
i < j, each row tile of 128 against all of the other image's 128-column chunks (padding included, which is what the
tensor cores execute) at 2 x 128 operations per multiply-add row; the rate is that over the matcher launches' CUDA-event
time, and its share of the dense int8 figure of NVIDIA's H100 SXM data sheet (1979 TOP/s at up to 700 W).  The card's
name, power limit and SM clock are read in the same run.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

INT8_DENSE_TOPS = 1979.0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--views', type=int, default=48)
    ap.add_argument('--width', type=int, default=1600)
    ap.add_argument('--height', type=int, default=1200)
    ap.add_argument('--max-features', type=int, default=8192)
    ap.add_argument('--repeat', type=int, default=2)
    ap.add_argument('--json', type=str, default=None, help='also write the result here')
    a = ap.parse_args()
    import numpy as np
    import torch
    import nero_oracle_mvs as OM
    from bench_mvs import card
    from nero_b200 import features as Ft, mvs, ops
    tmp = tempfile.mkdtemp(prefix='bench_features_')
    try:
        OM.project(tmp, a.views, a.width, a.height, seed=0, per_view=10, cell=0.01, workers=max(1, os.cpu_count() or 1))
        img_dir = os.path.join(tmp, 'images')
        rgbs = [mvs.read_rgb(os.path.join(img_dir, n)) for n in Ft.list_images(img_dir)]
        ev = lambda: torch.cuda.Event(enable_timing=True)
        res = dict(card=card(), views=a.views, width=a.width, height=a.height)
        for rep in range(a.repeat + 1):         # the first round warms every shape up and is not reported
            torch.cuda.synchronize()
            t0 = time.time()
            feats = [Ft.extract(rgb, max_features=a.max_features) for rgb in rgbs]
            torch.cuda.synchronize()
            t_ext = time.time() - t0
            descs = [d for _, d, _ in feats]
            # the matcher launches alone (one per batch of pairs), between events
            evs = []
            orig = ops.K

            def timed_K(name, *args, **kw):
                if name == 'nero_features_match':
                    evs.append((ev(), ev()))
                    evs[-1][0].record()
                    orig(name, *args, **kw)
                    evs[-1][1].record()
                else:
                    orig(name, *args, **kw)
            ops.K = timed_K
            try:
                torch.cuda.synchronize()
                t0 = time.time()
                matches, info = Ft.match_all(descs)
                torch.cuda.synchronize()
                t_match = time.time() - t0
            finally:
                ops.K = orig
            ms_kernel = sum(b0.elapsed_time(b1) for b0, b1 in evs)
            ops_count = sum(2 * 128 * 128 * (-(-int(t[3]) // 128) * 128) for t in info['tiles'])
            keys = sorted(matches)
            pts = [np.concatenate([feats[i][0][matches[i, j][:, 0].cpu().numpy(), :2], feats[j][0][matches[i, j][:, 1].cpu().numpy(), :2]], 1)
                   .astype(np.float64) for i, j in keys]
            torch.cuda.synchronize()
            t0 = time.time()
            F, best, count, inl = Ft.verify(pts)
            t_ver = time.time() - t0
            db = os.path.join(tmp, f'db_{rep}.db')
            t0 = time.time()
            Ft.write_database(db, [(k + 1, f'img_{k:03d}.png', 1) for k in range(a.views)],
                              Ft.cameras_for([(a.width, a.height)], True)[0], {k + 1: f[0] for k, f in enumerate(feats)},
                              {k + 1: f[1].cpu().numpy() for k, f in enumerate(feats)},
                              {(i + 1, j + 1): matches[i, j].cpu().numpy() for i, j in keys}, {})
            t_write = time.time() - t0
            if rep == 0:
                continue
            tops = ops_count / (ms_kernel * 1e-3) / 1e12
            res.setdefault('rounds', []).append(dict(
                extract_ms_per_view=1e3 * t_ext / a.views, features=int(sum(f[0].shape[0] for f in feats)),
                match_s=t_match, match_launches=len(evs), match_kernel_ms=ms_kernel, match_tops=tops, match_share_of_int8_dense=tops / INT8_DENSE_TOPS,
                pairs=len(keys), matches=int(sum(int(m.shape[0]) for m in matches.values())), verify_s=t_ver,
                verified=int((count >= Ft.MIN_INLIERS).sum()), write_s=t_write))
        print(json.dumps(res))
        if a.json:
            with open(a.json, 'w') as f:
                json.dump(res, f, indent=1)
    finally:
        shutil.rmtree(tmp)


if __name__ == '__main__':
    main()
