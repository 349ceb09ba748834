"""Chamfer distance between the vertex sets of two PLY files, on the GPU (the reference's eval_real_shape.py).

    python tools/eval_real_shape.py --pr data/meshes/bear_shape-300000.ply --gt data/GlossyReal/bear/eval_pts.ply

Prints `<pr stem> <chamfer>` and appends the same line to data/geometry.log (relative to the working directory).
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
    parser.add_argument('--pr', type=str, required=True)
    parser.add_argument('--gt', type=str, required=True)
    parser.add_argument('--batch_size', type=int, default=512,
                        help='accepted for command-line compatibility with the reference and ignored')
    flags = parser.parse_args(argv)

    from nero_b200 import evaluate as E
    pts_pr = E.read_points_ply(flags.pr)
    pts_gt = E.read_points_ply(flags.gt)
    chamfer, _, _ = E.chamfer_distance(pts_gt, pts_pr)
    line = E.result_line(Path(flags.pr).stem, chamfer)
    print(line)
    with open('data/geometry.log', 'a') as f:
        f.write(line + '\n')


if __name__ == '__main__':
    main()
