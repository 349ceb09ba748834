"""Measure a mesh against a reference mesh on the GPU: point-to-surface accuracy, completeness, Chamfer, Hausdorff and
F-score (nero_b200/meshdist.py), and optionally the predicted mesh coloured by its distance to the reference.

    python tools/compare_meshes.py --pr pred.ply --gt ref.ply [--samples N] [--seed S] [--threshold T ...] \\
        [--errors errors.ply] [--json metrics.json] [--align icp|auto [--align-rigid]]

Prints one `name value` line per metric.  --errors writes the predicted mesh with each vertex coloured by its distance to
the reference surface at the first threshold (blue on the surface, red at the threshold and beyond) and the distance as the
per-vertex `quality`.

--align registers the predicted mesh to the reference first (nero_b200/align.py: ICP from the identity, or from the
principal axes with `auto`; --align-rigid fixes the scale) on samples of its own (seed + 2), prints the transform and the
undetermined degrees of freedom, and measures in the reference's frame: accuracy from the predicted samples mapped in
float64, completeness from the reference samples mapped back by the inverse against the untouched predicted mesh, times the
scale.  --errors then writes the aligned predicted mesh.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402

from nero_b200.meshdist import THRESHOLDS  # noqa: E402


def lines(m):
    """(name, value) pairs of a metrics dict, in print order."""
    out = [('samples', m['samples']), ('seed', m['seed'])]
    for side in ('accuracy', 'completeness'):
        out += [(f'{side}.{k}', v) for k, v in m[side].items()]
    out += [('chamfer', m['chamfer']), ('hausdorff', m['hausdorff'])]
    for t in m['thresholds']:
        out += [(f'{k}@{t["threshold"]:g}', t[k]) for k in ('precision', 'recall', 'fscore')]
    return out


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--pr', type=str, required=True, help='predicted mesh (PLY)')
    parser.add_argument('--gt', type=str, required=True, help='reference mesh (PLY)')
    parser.add_argument('--samples', type=int, default=1_000_000, help='surface samples per mesh (default 1000000)')
    parser.add_argument('--seed', type=int, default=0, help='sample seed of the predicted mesh; the reference uses seed + 1')
    parser.add_argument('--threshold', type=float, nargs='+', default=list(THRESHOLDS),
                        help='F-score thresholds in scene units (default %(default)s: choices, not tuned values)')
    parser.add_argument('--errors', type=str, default=None, help='write the predicted mesh coloured by distance (PLY)')
    parser.add_argument('--json', type=str, default=None, help='write the metrics as JSON')
    parser.add_argument('--align', choices=('icp', 'auto'), default=None,
                        help='register --pr to --gt first: ICP from the identity, or from the principal axes (auto)')
    parser.add_argument('--align-rigid', action='store_true', help='with --align: fix the scale to 1')
    flags = parser.parse_args(argv)
    for path in (flags.pr, flags.gt):
        if not os.path.exists(path):
            raise SystemExit(f'compare_meshes: {path} does not exist')
    if flags.samples < 1:
        raise SystemExit(f'compare_meshes: --samples must be >= 1, got {flags.samples}')
    if any(not t > 0 for t in flags.threshold):
        raise SystemExit(f'compare_meshes: thresholds must be positive, got {flags.threshold}')

    from nero_b200.material import read_ply
    from nero_b200.meshdist import MeshDistance, compare_index, error_colors
    from nero_b200.mesh import write_ply

    pv, pt = read_ply(flags.pr)
    gv, gt = read_ply(flags.gt)
    pr, ref = MeshDistance(pv, pt), MeshDistance(gv, gt)
    if flags.align:
        return aligned(flags, pv, pt, pr, ref)
    m = compare_index(pr, ref, flags.samples, flags.seed, flags.threshold)
    m['pr'], m['gt'] = flags.pr, flags.gt
    for name, value in lines(m):
        print(f'{name} {value}')
    if flags.errors:
        d = ref.query(pr.verts.double())[0].cpu().numpy()
        write_ply(flags.errors, pv, pt, colors=error_colors(d, flags.threshold[0]), quality=d)
        print(f'errors {flags.errors}')
    if flags.json:
        with open(flags.json, 'w') as f:
            json.dump(m, f, indent=1)
    return m


def aligned(flags, pv, pt, pr, ref):
    """main() with --align: register pr to ref, then the metrics in ref's frame (module docstring)."""
    from align_meshes import describe, jsonable
    from nero_b200.align import align, apply, inverse
    from nero_b200.evaluate import sample_surface
    from nero_b200.meshdist import error_colors, metrics
    from nero_b200.mesh import write_ply
    if not 0 <= flags.seed < 2 ** 32 - 3:
        raise SystemExit(f'compare_meshes: --seed must be in [0, 2^32 - 3) with --align, got {flags.seed}')
    res = align((pr.verts, pr.tris), ref, rigid=flags.align_rigid, init='auto' if flags.align == 'auto' else 'identity',
                samples=flags.samples, seed=flags.seed + 2)
    for name, value in describe(res):
        print(f'align.{name} {value}')
    M = res['matrix']
    acc = ref.query(apply(M, sample_surface(pr.verts, pr.tris, flags.samples, flags.seed)))[0]
    comp = pr.query(apply(inverse(M), sample_surface(ref.verts, ref.tris, flags.samples, flags.seed + 1)))[0] * res['scale']
    m = metrics(acc, comp, flags.threshold)
    m['samples'], m['seed'] = int(flags.samples), int(flags.seed)
    m['pr'], m['gt'] = flags.pr, flags.gt
    m['align'] = jsonable(res)
    for name, value in lines(m):
        print(f'{name} {value}')
    if flags.errors:
        p = apply(M, pr.verts)
        d = ref.query(p)[0].cpu().numpy()
        write_ply(flags.errors, p.cpu().numpy().astype(np.float32), pt, colors=error_colors(d, flags.threshold[0]), quality=d)
        print(f'errors {flags.errors}')
    if flags.json:
        with open(flags.json, 'w') as f:
            json.dump(m, f, indent=1)
    return m


if __name__ == '__main__':
    main()
