"""Chamfer distance of a mesh against a GlossySynthetic object, on the GPU (the reference's eval_synthetic_shape.py).

    python tools/eval_synthetic_shape.py --object bell --mesh data/meshes/bell_shape-300000.ply

Reads data/GlossySynthetic/<object> (<k>-camera.pkl, <k>.png, <k>-depth.png) and the test split
configs/synthetic_split_128.pkl; both paths are relative to the working directory, as in the reference.  The ground-truth
points are read from <object dir>/eval_pts.ply when it exists and written there otherwise.  Prints `<mesh stem> <chamfer>`
and appends the same line to data/geometry.log.  The protocol is stated in nero_b200/evaluate.py.
"""
import argparse
import os
import sys
from pathlib import Path

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--mesh', type=str, required=True)
    parser.add_argument('--object', type=str, required=True)
    parser.add_argument('--batch_size', type=int, default=1024,
                        help='accepted for command-line compatibility with the reference and ignored')
    flags = parser.parse_args(argv)

    from nero_b200 import evaluate as E
    pts_gt, pts_pr = E.synthetic_eval_points(f'data/GlossySynthetic/{flags.object}', flags.mesh)
    chamfer, _, _ = E.chamfer_distance(pts_gt, pts_pr)
    line = E.result_line(Path(flags.mesh).stem, chamfer)
    print(line)
    with open('data/geometry.log', 'a') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
