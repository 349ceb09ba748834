"""Mesh clean-up and surface sampling on one H100, against the numpy / scipy oracle on the host CPU.

    python tools/bench_meshpts.py [--repeats 5] [--resolution 512] [--out DIR]

Workload: the ~0.9 M-triangle bell mesh of tools/bench_relight.py / bench_eval.py (extract_mesh at resolution 512 on the
perturbed bell parameters), uploaded once.  Times, each the median over the repeats between CUDA events after a warm call:
clean_mesh (areas + crop + components + component areas and selection + compaction, including the read-backs of the
component count and the totals) at min_component 0.01, and sample_surface of 500 k and 5 M points on the cleaned mesh
(areas, cumulative areas, the read of the total, sampling).  The oracle's clean-up and 500 k samples are timed once on the
host with a wall clock.  Prints one JSON line with the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

from bench_mesh import card, timed


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--resolution', type=int, default=512)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_meshpts: needs a CUDA device')
    import nero_oracle_meshpts as O
    from nero_b200 import evaluate as E
    from nero_b200 import params as P, synthetic
    from nero_b200.renderer import NeROShapeRenderer
    gpu = card()
    net = NeROShapeRenderer({}, training=False)
    net.load_state_dict(synthetic.perturb_params(P.build_shape_state_dict({}, seed=6033)))
    verts, tris = net.cuda().extract_mesh(resolution=args.resolution)
    del net
    torch.cuda.empty_cache()
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    v = torch.from_numpy(verts).cuda()
    t = torch.from_numpy(tris).cuda()
    frac = 0.01
    res = {}

    def clean():
        res['v'], res['t'], res['info'] = E.clean_mesh_cuda(v, t, min_component=frac)
    t_clean = timed(clean, args.repeats)
    cv, ct, info = res['v'], res['t'], res['info']
    t_500k = timed(lambda: E.sample_surface(cv, ct, 500_000), args.repeats)
    t_5m = timed(lambda: E.sample_surface(cv, ct, 5_000_000), args.repeats)
    same = bool(np.array_equal(E.sample_surface(cv, ct, 500_000).cpu().numpy(), O.sample(cv.cpu().numpy(), ct.cpu().numpy(), 500_000)[0]))

    h0 = time.perf_counter()
    oc = O.clean(verts, tris, min_component=frac)
    h1 = time.perf_counter()
    O.sample(oc['verts'], oc['tris'], 500_000)
    h2 = time.perf_counter()
    ms = lambda x: round(x * 1e3, 3)
    line = {'metric': 'mesh_points', 'gpu': gpu, 'triangles': int(tris.shape[0]), 'vertices': int(verts.shape[0]),
            'components': info['components'], 'kept_components': info['kept_components'],
            'kept_triangles': info['kept_triangles'], 'clean_ms': ms(t_clean), 'sample_500k_ms': ms(t_500k),
            'sample_5m_ms': ms(t_5m), 'samples_per_s_5m': 5e6 / t_5m, 'oracle_clean_s': round(h1 - h0, 3),
            'oracle_sample_500k_s': round(h2 - h1, 3), 'samples_equal_oracle': same,
            'clean_equal_oracle': bool(np.array_equal(ct.cpu().numpy(), oc['tris']))}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_meshpts.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
