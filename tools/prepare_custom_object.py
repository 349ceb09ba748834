"""Prepare a custom object for training, on the GPU: object_point_cloud.ply and meta_info.txt from a COLMAP reconstruction.

    python tools/prepare_custom_object.py --root data/custom/kettle [--points <fused ply>] [--sparse <model dir>]
        [--crop-sphere cx cy cz r] [--crop-box x0 y0 z0 x1 y1 z1] [--up x y z] [--forward x y z | --forward-image NAME]
        [--hypotheses 1024] [--seed 0] [--min-component 1.0] [--tol T] [--above A] [--voxel V] [--preview NAME] [--force]

Replaces the CloudCompare steps of the custom-object workflow (after COLMAP has run): crops the fused cloud (by default to
a sphere around the point the cameras look at), fits the support plane by RANSAC and two least-squares refits, orients its
normal toward the cameras (up), keeps the connected part of the cloud standing on the plane, and takes forward from the
object centre toward a camera, projected onto the plane.  Writes <root>/object_point_cloud.ply and <root>/meta_info.txt,
which CustomDatabase reads, and prints what training will do with them.  The protocol and its defaults are stated in
nero_b200/objprep.py.

--sparse defaults to <root>/colmap/sparse/0 (what CustomDatabase reads), else <root>/sparse/0 (where run_colmap.py
writes); --points to <root>/colmap/point.ply or <root>/points.ply, else the sparse points.  --tol, --above and --voxel are
in COLMAP units (default: fractions of the median camera distance).  --preview NAME writes <root>/object_preview.png: the
kept points (green) and the removed ones (red) projected into image NAME (drawn over <root>/images/NAME when it can be
read).
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

OUTPUTS = ('object_point_cloud.ply', 'meta_info.txt')


def _first(paths):
    return next((p for p in paths if os.path.exists(p)), None)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--root', type=str, required=True, help='data/custom/<object>')
    parser.add_argument('--points', type=str, default=None, help='fused point cloud PLY')
    parser.add_argument('--sparse', type=str, default=None, help='COLMAP sparse model directory')
    parser.add_argument('--crop-sphere', type=float, nargs=4, default=None, metavar=('CX', 'CY', 'CZ', 'R'))
    parser.add_argument('--crop-box', type=float, nargs=6, default=None, metavar=('X0', 'Y0', 'Z0', 'X1', 'Y1', 'Z1'))
    parser.add_argument('--up', type=float, nargs=3, default=None, metavar=('X', 'Y', 'Z'), help='use this up instead of the fit')
    group = parser.add_mutually_exclusive_group()
    group.add_argument('--forward', type=float, nargs=3, default=None, metavar=('X', 'Y', 'Z'))
    group.add_argument('--forward-image', type=str, default=None, help='forward points toward this image\'s camera')
    parser.add_argument('--hypotheses', type=int, default=1024)
    parser.add_argument('--seed', type=int, default=0)
    parser.add_argument('--min-component', type=float, default=1.0,
                        help='keep voxel components with at least this fraction of the largest one\'s points (default 1: the largest)')
    parser.add_argument('--tol', type=float, default=None, help='plane inlier tolerance')
    parser.add_argument('--above', type=float, default=None, help='least height of an object point over the plane')
    parser.add_argument('--voxel', type=float, default=None, help='voxel size of the connected components')
    parser.add_argument('--preview', type=str, default=None, metavar='NAME', help='write object_preview.png seen from this image')
    parser.add_argument('--force', action='store_true', help='overwrite existing output files')
    flags = parser.parse_args(argv)
    if not os.path.isdir(flags.root):
        parser.error(f'--root {flags.root} is not a directory')
    if flags.sparse is None:
        flags.sparse = _first([os.path.join(flags.root, 'colmap', 'sparse', '0'), os.path.join(flags.root, 'sparse', '0')])
        if flags.sparse is None:
            parser.error(f'no COLMAP model in {flags.root}/colmap/sparse/0 or {flags.root}/sparse/0 (give --sparse)')
    elif not os.path.isdir(flags.sparse):
        parser.error(f'--sparse {flags.sparse} is not a directory')
    if flags.points is None:
        flags.points = _first([os.path.join(flags.root, 'colmap', 'point.ply'), os.path.join(flags.root, 'points.ply')])
    elif not os.path.isfile(flags.points):
        parser.error(f'--points {flags.points} does not exist')
    if flags.hypotheses < 1:
        parser.error(f'--hypotheses must be >= 1, got {flags.hypotheses}')
    if not 0 <= flags.seed < 2 ** 32:
        parser.error(f'--seed must lie in [0, 2^32), got {flags.seed}')
    if not 0.0 <= flags.min_component <= 1.0:
        parser.error(f'--min-component must lie in [0, 1], got {flags.min_component}')
    if flags.crop_sphere is not None and not flags.crop_sphere[3] > 0:
        parser.error(f'--crop-sphere radius must be positive, got {flags.crop_sphere[3]}')
    if flags.crop_box is not None and not all(flags.crop_box[a] <= flags.crop_box[a + 3] for a in range(3)):
        parser.error(f'--crop-box needs x0 <= x1, y0 <= y1, z0 <= z1, got {flags.crop_box}')
    for name in ('tol', 'voxel'):
        v = getattr(flags, name)
        if v is not None and not v > 0:
            parser.error(f'--{name} must be positive, got {v}')
    if flags.up is not None and not any(flags.up):
        parser.error('--up must not be the zero vector')
    if flags.forward is not None and not any(flags.forward):
        parser.error('--forward must not be the zero vector')
    existing = [f for f in OUTPUTS if os.path.exists(os.path.join(flags.root, f))]
    if existing and not flags.force:
        parser.error(f'{", ".join(existing)} already exist in {flags.root}: pass --force to overwrite')
    return flags


def preview(path, view, image_path, kept, removed):
    """uint8 RGB: the removed points in red, then the kept points in green, projected with the view's pose and K."""
    import numpy as np
    from nero_b200.relight import write_png
    _, pose, K = view
    w, h = int(round(2 * K[0, 2])), int(round(2 * K[1, 2]))
    img = np.full((h, w, 3), 40, np.uint8)
    try:
        from PIL import Image
        img = np.asarray(Image.open(image_path).convert('RGB'), np.uint8).copy()
        h, w = img.shape[:2]
    except Exception:   # the preview only needs a canvas: without the image (or an image library) the points go on grey
        pass
    P = (K.astype(np.float64) @ pose.astype(np.float64))
    for pts, colour in ((removed, (255, 40, 40)), (kept, (40, 255, 40))):
        x = np.concatenate([pts, np.ones((pts.shape[0], 1))], 1) @ P.T
        ok = x[:, 2] > 0
        u = np.floor(x[ok, 0] / x[ok, 2]).astype(np.int64)
        v = np.floor(x[ok, 1] / x[ok, 2]).astype(np.int64)
        on = (u >= 0) & (u < w) & (v >= 0) & (v < h)
        img[v[on], u[on]] = colour
    write_png(path, img)


def main(argv=None):
    flags = parse_args(argv)
    import numpy as np
    from nero_b200 import objprep as OP
    from nero_b200.evaluate import read_points_ply, write_points_ply
    views, sparse_pts = OP.read_colmap_model(flags.sparse)
    if not views:
        raise SystemExit(f'{flags.sparse}: the model has no images')
    pts = read_points_ply(flags.points) if flags.points else sparse_pts
    center, D, names, centers = OP.scene_scale(views)
    by_name = {v[0]: v for v in views.values()}
    for n in (flags.forward_image, flags.preview):
        if n is not None and n not in by_name:
            raise SystemExit(f'image {n} is not in the model')
    sphere = flags.crop_sphere
    if sphere is None and flags.crop_box is None:
        sphere = list(center) + [OP.CROP_FRAC * D]
    tol = flags.tol if flags.tol is not None else OP.TOL_FRAC * D
    above = flags.above if flags.above is not None else OP.ABOVE_TOLS * tol
    voxel = flags.voxel if flags.voxel is not None else OP.VOXEL_FRAC * D
    plane, finfo = OP.fit_support_plane(pts, tol, sphere, flags.crop_box, flags.hypotheses, flags.seed, centers)
    up = plane[:3]
    if flags.up is not None:       # the object is still cut at the fitted plane, its normal turned toward the given up
        up = np.asarray(flags.up, np.float64) / np.linalg.norm(flags.up)
        plane = plane if plane[:3] @ up >= 0 else -plane
    obj, iinfo = OP.isolate_object(pts, plane, above, voxel, sphere, flags.crop_box, flags.min_component)
    obj = obj.cpu().numpy()
    if flags.forward is not None:
        forward = OP.project_forward(flags.forward, up)
    else:
        cam = centers[names.index(flags.forward_image or names[0])]
        forward = OP.forward_direction(center, cam, up)
    norm = OP.normalization(obj, up, forward, centers)
    write_points_ply(os.path.join(flags.root, OUTPUTS[0]), obj)
    OP.write_meta_info(os.path.join(flags.root, OUTPUTS[1]), up, forward)
    n_in = int(norm['inside'].sum())
    print(f'{flags.points or flags.sparse}: {pts.shape[0]} points, {finfo["kept"]} inside the crop; camera distance {D:.6g}, '
          f'tol {tol:.6g}, above {above:.6g}, voxel {voxel:.6g}')
    print(f'plane: normal ({plane[0]:.6f}, {plane[1]:.6f}, {plane[2]:.6f}), d {plane[3]:.6g}, inliers {finfo["inliers"]} '
          f'({finfo["inliers"] / finfo["kept"]:.1%} of the crop), best hypothesis {finfo["best"]} of {flags.hypotheses}')
    print(f'object: {iinfo["components"]} components, {iinfo["kept_components"]} kept, {iinfo["kept"]} points')
    print(f'up ({up[0]:.6f}, {up[1]:.6f}, {up[2]:.6f}), forward ({forward[0]:.6f}, {forward[1]:.6f}, {forward[2]:.6f})')
    print(f'normalisation: scale {norm["scale"]:.6g}, closest normalised camera distance {norm["camera_dist"].min():.4f}'
          + (f'; {n_in} cameras inside the unit sphere' if n_in else ''))
    if flags.preview:
        keep = iinfo['point_keep'].cpu().numpy().astype(bool)
        crop = iinfo['keep'].cpu().numpy().astype(bool)
        preview(os.path.join(flags.root, 'object_preview.png'), by_name[flags.preview],
                os.path.join(flags.root, 'images', flags.preview), obj, np.asarray(pts)[crop & ~keep])
    print(f'wrote {", ".join(os.path.join(flags.root, f) for f in OUTPUTS)}')


if __name__ == '__main__':
    main()
