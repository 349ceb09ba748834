"""Time the GPU mapper (nero_b200.sfm) on a synthetic project: track building, all registrations, triangulation, one
bundle-adjustment iteration at the final size with its achieved fp64 rate, and the whole mapper.

    python tools/bench_sfm.py [--views 48] [--width 1600] [--height 1200] [--repeat 1] [--same_camera]
        [--camera-model SIMPLE_RADIAL [--k -0.05]]

The project is the 48-view table / box / sphere scene of tools/bench_features.py, rendered on the CPU and run through
features.build_database (neither is timed).  The mapper then runs repeat + 1 times; the first round warms every shape up
and is not reported.  --same_camera writes the database with one camera for every image, the case in which the
reduced system's focal segments hold every (o, o') pair.  One bundle-adjustment iteration (linearisation, point
elimination, reduced system, Cholesky, back-substitution and the cost of the candidate) is timed with CUDA events on the
final model's problem as the mapper builds it (Mapper.problem: the same gauge and focal rule), over 10 repetitions.  Its
fp64 operations are counted from the shapes by `ba_flops` below (multiplies and adds of each kernel's formulas, the
Cholesky as ncol^3 / 3); the rate is shown against the fp64 (non-tensor) figure of NVIDIA's H100 SXM data sheet,
34 TFLOP/s at up to 700 W.  The card's name, power limit and SM clock are read in the same run.

--camera-model SIMPLE_RADIAL renders the same views through SIMPLE_RADIAL k = --k (oracle/nero_oracle_sfm_radial.py),
writes SIMPLE_RADIAL cameras and runs the mapper that estimates k.  It adds |k^ - k| per camera, and times the pinhole
bundle-adjustment iteration on the same final model in the same session (pinhole_ba_iteration_ms), so the radial
iteration's cost is read against it.
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

FP64_TFLOPS = 34.0


def ba_flops(n, P, pairs, ncol):
    """fp64 operations of one iteration: per observation linearisation (~150), elimination (~260), right-hand side (~70),
    back-substitution (~130) and cost (~30); per (o, o') pair the 49 reduced-system entries at ~20 each; the dense
    Cholesky and two triangular solves."""
    return n * (150 + 260 + 70 + 130 + 30) + P * 40 + pairs * 49 * 20 + ncol ** 3 / 3 + 2 * ncol ** 2


def iteration_ms(pr):
    """CUDA-event time of one bundle-adjustment iteration (linearisation, step, cost of the candidate) of Problem pr: two
    warm-up iterations, then the mean of ten."""
    import torch
    ev = lambda: torch.cuda.Event(enable_timing=True)
    for k in range(12):
        if k == 2:
            e0 = ev()
            e0.record()
        pr.linearize()
        cand = pr.step(1e-4)
        pr.cost(*cand)
    e1 = ev()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 10


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--views', type=int, default=48)
    ap.add_argument('--width', type=int, default=1600)
    ap.add_argument('--height', type=int, default=1200)
    ap.add_argument('--repeat', type=int, default=1)
    ap.add_argument('--same_camera', action='store_true', help='one camera for every image (its focal segments hold every pair)')
    ap.add_argument('--camera-model', choices=('SIMPLE_PINHOLE', 'SIMPLE_RADIAL'), default='SIMPLE_PINHOLE')
    ap.add_argument('--k', type=float, default=-0.05, help='the lens of the SIMPLE_RADIAL renders')
    ap.add_argument('--json', type=str, default=None, help='also write the result here')
    a = ap.parse_args()
    import torch
    import nero_oracle_mvs as OM
    from bench_mvs import card
    from nero_b200 import features as Ft, sfm
    tmp = tempfile.mkdtemp(prefix='bench_sfm_')
    try:
        radial = a.camera_model == 'SIMPLE_RADIAL'
        if radial:
            import nero_oracle_sfm_radial as OR
            OR.project(tmp, a.views, a.width, a.height, a.k, seed=0, cell=0.01, workers=max(1, os.cpu_count() or 1))
        else:
            OM.project(tmp, a.views, a.width, a.height, seed=0, per_view=10, cell=0.01, workers=max(1, os.cpu_count() or 1))
        db_path = os.path.join(tmp, 'database.db')
        Ft.build_database(os.path.join(tmp, 'images'), db_path, same_camera=a.same_camera, camera_model=a.camera_model)
        res = dict(card=card(), views=a.views, width=a.width, height=a.height, same_camera=a.same_camera)
        if radial:
            res.update(camera_model=a.camera_model, k=a.k)
        for rep in range(a.repeat + 1):
            db = sfm.read_database(db_path)
            torch.cuda.synchronize()
            t0 = time.time()
            mp = sfm.Mapper(db, camera_model=a.camera_model).run()
            torch.cuda.synchronize()
            t_all = time.time() - t0
            if rep == 0:
                continue
            pr, _, _, tracks = mp.problem()            # the final adjustment's problem, with the mapper's gauge
            ms = iteration_ms(pr)
            n, P, pairs, ncol = pr.n, int(tracks.shape[0]), int(pr.ent.shape[0] // 4), pr.ncol
            fl = ba_flops(n, P, pairs, ncol)
            t = mp.times
            res.setdefault('rounds', []).append(dict(
                registered=int(mp.reg.sum()), points=P, observations=n, tracks_s=t['tracks'], init_s=t['init'], register_s=t['register'],
                triangulate_s=t['triangulate'], bundle_s=t['bundle'], mapper_s=t_all,
                ba_iteration_ms=ms, ba_pairs=pairs, ba_columns=ncol, ba_gflop=fl / 1e9, ba_tflops=fl / (ms * 1e-3) / 1e12,
                ba_share_of_fp64_datasheet=fl / (ms * 1e-3) / 1e12 / FP64_TFLOPS))
            if radial:
                mp.radial, k_hat = None, mp.radial        # the same model as a pinhole problem, for the same-session comparison
                pin = iteration_ms(mp.problem()[0])
                mp.radial = k_hat
                res['rounds'][-1].update(k_error=[abs(float(k) - a.k) for k in k_hat], pinhole_ba_iteration_ms=pin)
        print(json.dumps(res))
        if a.json:
            with open(a.json, 'w') as f:
                json.dump(res, f, indent=1)
    finally:
        shutil.rmtree(tmp)


if __name__ == '__main__':
    main()
