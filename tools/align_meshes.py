"""Register a mesh or point cloud to a reference mesh on the GPU: a trimmed point-to-plane similarity ICP
(nero_b200/align.py), started from the identity, the principal axes (--init auto) or a matrix file.

    python tools/align_meshes.py --src src.ply --dst ref.ply [--init identity|auto|matrix.txt] [--rigid] [--samples N] \\
        [--max-distance D] [--iterations K] [--out aligned.ply] [--matrix matrix.txt] [--json result.json]

A source PLY without faces is a point cloud.  Prints the 4 x 4 matrix of y = s R x + t (source to reference), the scale,
the iterations, the last RMS point-to-plane residual and the degrees of freedom the reference's shape leaves undetermined.
--out writes the source mapped into the reference frame (mesh or points), --matrix the matrix as 4 lines of 4 numbers,
readable back through --init.  The defaults of align.py (first inlier distance 0.1 of the reference's RMS radius, 200000
samples, ...) are choices, not tuned values.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def read_matrix(path):
    """A 4 x 4 matrix from 4 lines of 4 numbers."""
    rows = [ln.split() for ln in open(path).read().splitlines() if ln.strip()]
    if len(rows) != 4 or any(len(r) != 4 for r in rows):
        raise SystemExit(f'align_meshes: {path} must hold 4 lines of 4 numbers')
    return np.asarray(rows, np.float64)


def write_matrix(path, M):
    with open(path, 'w') as f:
        for row in np.asarray(M, np.float64):
            f.write(' '.join(repr(float(x)) for x in row) + '\n')


def has_faces(path):
    """Whether the PLY header declares a face element with at least one face."""
    with open(path, 'rb') as f:
        for line in f:
            t = line.decode('ascii', 'replace').split()
            if t[:1] == ['end_header']:
                return False
            if len(t) == 3 and t[0] == 'element' and t[1] == 'face':
                return int(t[2]) > 0
    return False


def parse(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0], epilog=__doc__.split('\n\n', 2)[2],
                                     formatter_class=argparse.RawDescriptionHelpFormatter)
    parser.add_argument('--src', type=str, required=True, help='source mesh or point cloud (PLY)')
    parser.add_argument('--dst', type=str, required=True, help='reference mesh (PLY)')
    parser.add_argument('--init', type=str, default='identity', help="'identity' (default), 'auto' or a 4 x 4 matrix file")
    parser.add_argument('--rigid', action='store_true', help='fix the scale to 1')
    parser.add_argument('--samples', type=int, default=200_000, help='surface samples of a mesh (default 200000)')
    parser.add_argument('--seed', type=int, default=0, help='sample seed of the source; the reference uses seed + 1')
    parser.add_argument('--max-distance', type=float, default=None, help='first inlier distance (default 0.1 RMS radius)')
    parser.add_argument('--iterations', type=int, default=50, help='most ICP iterations (default 50)')
    parser.add_argument('--out', type=str, default=None, help='write the aligned source (PLY)')
    parser.add_argument('--matrix', type=str, default=None, help='write the matrix (4 lines of 4 numbers)')
    parser.add_argument('--json', type=str, default=None, help='write the result as JSON')
    return parser.parse_args(argv)


def describe(res):
    """(name, value) lines of an align() result, in print order."""
    out = [(f'matrix.{i}', ' '.join(f'{x:.17g}' for x in row)) for i, row in enumerate(res['matrix'])]
    out += [('scale', res['scale']), ('iterations', res['iterations']), ('converged', res['converged']),
            ('rms', res['rms'][-1]), ('inliers', res['inliers'][-1])]
    und = res['undetermined']
    out.append(('undetermined', ', '.join(u['kind'] for u in und) if und else 'none'))
    return out


def jsonable(res):
    return {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in res.items()}


def main(argv=None):
    flags = parse(argv)
    for path in (flags.src, flags.dst):
        if not os.path.exists(path):
            raise SystemExit(f'align_meshes: {path} does not exist')
    init = flags.init if flags.init in ('identity', 'auto') else read_matrix(flags.init)

    from nero_b200.align import align, apply
    from nero_b200.evaluate import read_points_ply, write_points_ply
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    from nero_b200.meshdist import MeshDistance

    mesh = has_faces(flags.src)
    src = read_ply(flags.src) if mesh else read_points_ply(flags.src)
    dst = MeshDistance(*read_ply(flags.dst))
    try:
        res = align(src, dst, rigid=flags.rigid, init=init, samples=flags.samples, seed=flags.seed,
                    max_distance=flags.max_distance, max_iters=flags.iterations)
    except ValueError as e:
        raise SystemExit(f'align_meshes: {e}')
    for name, value in describe(res):
        print(f'{name} {value}')
    if flags.out:
        p = apply(res['matrix'], src[0] if mesh else src).cpu().numpy()
        write_ply(flags.out, p.astype(np.float32), src[1]) if mesh else write_points_ply(flags.out, p)
        print(f'out {flags.out}')
    if flags.matrix:
        write_matrix(flags.matrix, res['matrix'])
    if flags.json:
        with open(flags.json, 'w') as f:
            json.dump(jsonable(res), f, indent=1)
    return res


if __name__ == '__main__':
    main()
