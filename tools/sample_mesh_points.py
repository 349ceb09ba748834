"""Sample an evaluation point cloud on a mesh, on the GPU: the clean-up and sampling steps of the real-data shape protocol.

    python tools/sample_mesh_points.py --mesh data/meshes/bear_shape-300000.ply --out data/point_cloud/bear-nero.ply \\
        [--num 500000] [--seed 0] [--crop-sphere cx cy cz r] [--crop-box x0 y0 z0 x1 y1 z1] [--min-component f] [--mesh-out <ply>]

Crops the mesh to the sphere and / or box (a triangle is kept iff its three vertices are inside), keeps the connected
components whose area is at least f times the largest one's, samples --num area-uniform points on what is left and writes
them as a `double x y z` PLY, which tools/eval_real_shape.py reads.  Run it on the ground-truth mesh too (for example to
data/point_cloud/bear-gt.ply), then: python tools/eval_real_shape.py --pr data/point_cloud/bear-nero.ply --gt
data/point_cloud/bear-gt.ply.  --mesh-out writes the cleaned mesh, to inspect what was kept.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--mesh', type=str, required=True, help='input PLY mesh')
    parser.add_argument('--out', type=str, required=True, help='output point-cloud PLY')
    parser.add_argument('--num', type=int, default=500_000, help='number of points (default 500000)')
    parser.add_argument('--seed', type=int, default=0)
    parser.add_argument('--crop-sphere', type=float, nargs=4, default=None, metavar=('CX', 'CY', 'CZ', 'R'))
    parser.add_argument('--crop-box', type=float, nargs=6, default=None, metavar=('X0', 'Y0', 'Z0', 'X1', 'Y1', 'Z1'))
    parser.add_argument('--min-component', type=float, default=0.0,
                        help='keep components with at least this fraction of the largest component\'s area (default 0: all)')
    parser.add_argument('--mesh-out', type=str, default=None, help='also write the cleaned mesh here')
    flags = parser.parse_args(argv)
    if flags.num < 1:
        parser.error(f'--num must be >= 1, got {flags.num}')
    if not 0 <= flags.seed < 2 ** 32:
        parser.error(f'--seed must lie in [0, 2^32), got {flags.seed}')
    if not 0.0 <= flags.min_component <= 1.0:
        parser.error(f'--min-component must lie in [0, 1], got {flags.min_component}')
    if flags.crop_sphere is not None and not flags.crop_sphere[3] > 0:
        parser.error(f'--crop-sphere radius must be positive, got {flags.crop_sphere[3]}')
    if flags.crop_box is not None and not all(flags.crop_box[a] <= flags.crop_box[a + 3] for a in range(3)):
        parser.error(f'--crop-box needs x0 <= x1, y0 <= y1, z0 <= z1, got {flags.crop_box}')
    if not os.path.exists(flags.mesh):
        parser.error(f'--mesh {flags.mesh} does not exist')
    return flags


def main(argv=None):
    flags = parse_args(argv)
    from nero_b200 import evaluate as E
    from nero_b200.material import read_ply
    from nero_b200.mesh import write_ply
    verts, tris = read_ply(flags.mesh)
    v, t, info = E.clean_mesh_cuda(verts, tris, flags.crop_sphere, flags.crop_box, flags.min_component)
    if flags.mesh_out:
        write_ply(flags.mesh_out, v.cpu().numpy(), t.cpu().numpy())
    pts = E.sample_surface(v, t, flags.num, flags.seed).cpu().numpy()
    area = float(info['comp_area'][info['comp_keep']].sum())
    os.makedirs(os.path.dirname(os.path.abspath(flags.out)), exist_ok=True)
    E.write_points_ply(flags.out, pts)
    n_crop = int(info['keep'].sum())
    print(f'{flags.mesh}: {info["triangles"]} triangles, {n_crop} inside the crop, {info["components"]} components, '
          f'{info["kept_components"]} kept ({info["kept_triangles"]} triangles, {info["kept_vertices"]} vertices), '
          f'area {area:.6g}')
    print(f'{flags.out}: {pts.shape[0]} points, seed {flags.seed}')


if __name__ == '__main__':
    main()
