"""Reduce a triangle mesh to about N triangles on the GPU by quadric edge collapse (nero_b200/simplify.py).

    python tools/simplify_mesh.py --mesh in.ply --out out.ply --faces N

Reads a PLY (ascii or binary little-endian, triangles), writes a binary PLY and prints the statistics.  A closed mesh ends
with exactly N triangles for even N (N or N + 1 for odd N); boundary vertices and their edges are kept as they are, and a
mesh whose remaining edges may not collapse ends above N, which the statistics show.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--mesh', type=str, required=True, help='input PLY')
    parser.add_argument('--out', type=str, required=True, help='output PLY')
    parser.add_argument('--faces', type=int, required=True, help='target triangle count (>= 4)')
    flags = parser.parse_args(argv)
    if flags.faces < 4:
        raise SystemExit(f'simplify_mesh: --faces must be >= 4, got {flags.faces}')
    if not os.path.exists(flags.mesh):
        raise SystemExit(f'simplify_mesh: {flags.mesh} does not exist')

    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    from nero_b200.simplify import simplify, stats_line

    verts, tris = read_ply(flags.mesh)
    t0 = time.perf_counter()
    v, t, stats = simplify(verts, tris, flags.faces)
    dt = time.perf_counter() - t0
    write_ply(flags.out, v, t)
    print(f'{flags.mesh}: {verts.shape[0]} vertices, {tris.shape[0]} triangles -> {flags.out}: {v.shape[0]} vertices, '
          f'{t.shape[0]} triangles in {dt:.2f} s')
    print(stats_line(stats))
    return flags.out


if __name__ == '__main__':
    main()
