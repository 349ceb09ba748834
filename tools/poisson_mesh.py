"""Mesh an oriented point cloud on the GPU with screened Poisson reconstruction: a surface from dense_points.py --normals.

    python tools/poisson_mesh.py --points data/custom/kettle/points.ply --out kettle_mvs.ply [--resolution 513] [--screen 4] [--scale 1.1]
        [--trim T] [--min-component F] [--crop-sphere cx cy cz r | --crop-box x0 y0 z0 x1 y1 z1] [--custom-frame <root>]
        [--force]

Replaces COLMAP's poisson_mesher, the last step of run_colmap.py's dense pipeline.  The workflow becomes
match_features.py -> map_sparse.py -> dense_points.py --normals -> poisson_mesh.py: a surface to look at before training,
and the multi-view-stereo baseline that compare_meshes.py measures NeRO's mesh against.  The protocol is stated in
nero_b200/poisson.py.

--points: a PLY with x y z nx ny nz (float or double; COLMAP's fused.ply reads too).  Points with a zero normal are
skipped and counted.  --crop-sphere / --crop-box keep the points inside the region before the solve (objprep.crop_points).
--trim T (default 0: the watertight surface) drops triangles whose sample density, over its median, is below T; 0.1 to 0.3
removes the surface Poisson invents where there are no samples.  The surface that closes an open cloud bulges past the
samples; where it meets the grid's boundary it stays open there, and a larger --scale (e.g. 2) gives it room.
--min-component F then keeps the connected components with at least F times the largest one's area
(evaluate.clean_mesh_cuda).  --custom-frame <root> writes the mesh in the
frame NeRO trains <root> in (objprep.normalization of <root>/object_point_cloud.ply and <root>/meta_info.txt), so
compare_meshes.py against a NeRO mesh of that object needs no --align.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

RESOLUTIONS = (33, 65, 129, 257, 513)      # nero_b200.poisson.RESOLUTIONS


def parse(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--points', required=True, help='oriented point cloud PLY (x y z nx ny nz)')
    parser.add_argument('--out', required=True, help='output mesh PLY')
    parser.add_argument('--resolution', type=int, default=513, help=f'grid nodes per axis, one of {RESOLUTIONS}')
    parser.add_argument('--screen', type=float, default=4.0, help='screening weight (PoissonRecon point weight)')
    parser.add_argument('--scale', type=float, default=1.1, help='grid cube over the bounding cube')
    parser.add_argument('--tol', type=float, default=1e-5, help='relative residual that ends the solve')
    parser.add_argument('--max-iters', type=int, default=200)
    parser.add_argument('--trim', type=float, default=0.0, help='drop triangles below this density over the median')
    parser.add_argument('--min-component', type=float, default=0.0, help='keep components with this fraction of the largest area')
    parser.add_argument('--crop-sphere', type=float, nargs=4, default=None, metavar=('CX', 'CY', 'CZ', 'R'))
    parser.add_argument('--crop-box', type=float, nargs=6, default=None, metavar=('X0', 'Y0', 'Z0', 'X1', 'Y1', 'Z1'))
    parser.add_argument('--custom-frame', default=None, metavar='ROOT', help='write the mesh in the training frame of this custom object')
    parser.add_argument('--force', action='store_true', help='overwrite an existing output file')
    flags = parser.parse_args(argv)
    if not os.path.isfile(flags.points):
        parser.error(f'--points {flags.points} does not exist')
    if flags.resolution not in RESOLUTIONS:
        parser.error(f'--resolution must be one of {RESOLUTIONS}, got {flags.resolution}')
    if not flags.screen > 0 or not flags.scale > 1:
        parser.error(f'need --screen > 0 and --scale > 1, got {flags.screen}, {flags.scale}')
    if not flags.trim >= 0:
        parser.error(f'--trim must be >= 0, got {flags.trim}')
    if not 0 <= flags.min_component <= 1:
        parser.error(f'--min-component must lie in [0, 1], got {flags.min_component}')
    if flags.crop_sphere is not None and not flags.crop_sphere[3] > 0:
        parser.error(f'--crop-sphere radius must be positive, got {flags.crop_sphere[3]}')
    if flags.crop_box is not None and not all(a <= b for a, b in zip(flags.crop_box[:3], flags.crop_box[3:])):
        parser.error(f'--crop-box needs x0 <= x1, y0 <= y1, z0 <= z1, got {flags.crop_box}')
    if flags.custom_frame is not None:
        for f in ('object_point_cloud.ply', 'meta_info.txt'):
            if not os.path.isfile(os.path.join(flags.custom_frame, f)):
                parser.error(f'--custom-frame: {os.path.join(flags.custom_frame, f)} does not exist')
    if os.path.exists(flags.out) and not flags.force:
        parser.error(f'{flags.out} already exists: pass --force to overwrite')
    return flags


def custom_frame(root):
    """(scale, offset, R) of objprep.normalization for the custom object at root: x' = scale (x + offset) R^T."""
    import numpy as np
    from nero_b200 import objprep
    from nero_b200.evaluate import read_points_ply
    meta = np.loadtxt(os.path.join(root, 'meta_info.txt'))
    nz = objprep.normalization(read_points_ply(os.path.join(root, 'object_point_cloud.ply')), meta[0], meta[1])
    return nz['scale'], nz['offset'], nz['R']


def main(argv=None):
    flags = parse(argv)
    import numpy as np
    import torch
    from nero_b200 import objprep, poisson
    from nero_b200.evaluate import clean_mesh_cuda, read_oriented_points_ply
    from nero_b200.mesh import write_ply
    pts, nrm = read_oriented_points_ply(flags.points)
    good = np.linalg.norm(nrm, axis=1) > 0
    if not good.all():
        print(f'{flags.points}: skipping {int((~good).sum())} points with a zero normal')
        pts, nrm = pts[good], nrm[good]
    n_read = pts.shape[0]
    if flags.crop_sphere is not None or flags.crop_box is not None:
        if n_read == 0:
            raise SystemExit(f'{flags.points}: no points')
        keep, _, pts_c = objprep.crop_points(pts, flags.crop_sphere, flags.crop_box)
        pts, nrm = pts_c.cpu().numpy(), nrm[keep.cpu().numpy().astype(bool)]
        print(f'crop: {pts.shape[0]} of {n_read} points kept')
    t0 = time.time()
    try:
        verts, tris, info = poisson.reconstruct(pts, nrm, flags.resolution, flags.screen, flags.scale, flags.tol, flags.max_iters, flags.trim)
    except ValueError as e:
        raise SystemExit(f'{flags.points}: {e}')
    torch.cuda.synchronize()
    print(f'{pts.shape[0]} points, grid {flags.resolution}^3 (h = {info["h"]:.6g}), sigma {info["sigma"]:.4g} samples per cell area; '
          f'{info["iterations"]} iterations, residual {info["history"][-1]:.3e}, iso {info["iso"]:.6g}; '
          f'{info["triangles_before"]} triangles, {info["triangles_after"]} after --trim {flags.trim:g}; {time.time() - t0:.2f} s')
    if tris.shape[0] == 0:
        raise SystemExit('the reconstruction has no triangles')
    if flags.min_component > 0:
        verts, tris, cinfo = clean_mesh_cuda(verts, tris, min_component=flags.min_component)
        print(f'--min-component {flags.min_component:g}: {cinfo["kept_components"]} of {cinfo["components"]} components, '
              f'{cinfo["kept_triangles"]} triangles')
    v = verts.cpu().numpy().astype(np.float64)
    if flags.custom_frame is not None:
        s, offset, R = custom_frame(flags.custom_frame)
        v = s * (v + offset) @ R.T
        print(f'--custom-frame {flags.custom_frame}: scale {s:.6g}')
    write_ply(flags.out, v.astype(np.float32), tris.cpu().numpy())
    print(f'wrote {flags.out}')


if __name__ == '__main__':
    main()
