"""Reconstruct a custom object's dense point cloud on the GPU: <root>/points.ply from a COLMAP sparse model and its images.

    python tools/dense_points.py --root data/custom/kettle [--sparse <model dir>] [--images <dir>] [--output <ply>]
        [--max-size 1600] [--sources 8] [--iterations 8] [--radius 4] [--step 2] [--seed 0] [--voxel V] [--force]

Replaces the dense half of run_colmap.py (image_undistorter, patch_match_stereo, stereo_fusion), which needs a CUDA build
of COLMAP: PatchMatch stereo per view, a forward-backward geometric filter against the source views, and the surviving
pixels unprojected into one cloud.  The output goes where run_colmap.py writes its fused cloud, so
tools/prepare_custom_object.py finds it there.  The workflow becomes: run_colmap.py (sparse half only) -> dense_points.py
-> prepare_custom_object.py.  The protocol and its defaults are stated in nero_b200/mvs.py.

--sparse defaults to <root>/colmap/sparse/0, else <root>/sparse/0; --images to <root>/images.  --voxel (COLMAP units)
thins the cloud to one point per voxel.  Views without enough source views or sparse points are skipped and reported.

Mirror-like parts of a glossy object mostly fail photo-consistency (their appearance changes with the viewpoint) and are
filtered out.  The table and the less reflective parts of the object still carry the crop, the support plane and the
object's extent that prepare_custom_object.py needs.  SIMPLE_RADIAL distortion is ignored, as training ignores it.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def _first(paths):
    return next((p for p in paths if os.path.exists(p)), None)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--root', type=str, required=True, help='data/custom/<object>')
    parser.add_argument('--sparse', type=str, default=None, help='COLMAP sparse model directory')
    parser.add_argument('--images', type=str, default=None, help='image directory (default <root>/images)')
    parser.add_argument('--output', type=str, default=None, help='output PLY (default <root>/points.ply)')
    parser.add_argument('--max-size', type=int, default=1600, help='longest side of the matched images')
    parser.add_argument('--sources', type=int, default=8, help='source views per reference view')
    parser.add_argument('--iterations', type=int, default=8)
    parser.add_argument('--radius', type=int, default=4, help='matching window half-size in pixels')
    parser.add_argument('--step', type=int, default=2, help='matching window sample step in pixels')
    parser.add_argument('--seed', type=int, default=0)
    parser.add_argument('--voxel', type=float, default=None, help='thin the cloud to one point per voxel of this size')
    parser.add_argument('--force', action='store_true', help='overwrite an existing output file')
    flags = parser.parse_args(argv)
    if not os.path.isdir(flags.root):
        parser.error(f'--root {flags.root} is not a directory')
    if flags.sparse is None:
        flags.sparse = _first([os.path.join(flags.root, 'colmap', 'sparse', '0'), os.path.join(flags.root, 'sparse', '0')])
        if flags.sparse is None:
            parser.error(f'no COLMAP model in {flags.root}/colmap/sparse/0 or {flags.root}/sparse/0 (give --sparse)')
    elif not os.path.isdir(flags.sparse):
        parser.error(f'--sparse {flags.sparse} is not a directory')
    if flags.images is None:
        flags.images = os.path.join(flags.root, 'images')
    if not os.path.isdir(flags.images):
        parser.error(f'--images {flags.images} is not a directory')
    if flags.output is None:
        flags.output = os.path.join(flags.root, 'points.ply')
    if flags.max_size < 1:
        parser.error(f'--max-size must be >= 1, got {flags.max_size}')
    if not 2 <= flags.sources <= 16:
        parser.error(f'--sources must lie in [2, 16], got {flags.sources}')
    if flags.iterations < 0:
        parser.error(f'--iterations must be >= 0, got {flags.iterations}')
    if not 0 <= flags.radius <= 64 or flags.step < 1:
        parser.error(f'--radius must lie in [0, 64] and --step be >= 1, got {flags.radius}, {flags.step}')
    if not 0 <= flags.seed < 2 ** 32:
        parser.error(f'--seed must lie in [0, 2^32), got {flags.seed}')
    if flags.voxel is not None and not flags.voxel > 0:
        parser.error(f'--voxel must be positive, got {flags.voxel}')
    if os.path.exists(flags.output) and not flags.force:
        parser.error(f'{flags.output} already exists: pass --force to overwrite')
    return flags


def main(argv=None):
    flags = parse_args(argv)
    from nero_b200 import mvs, objprep
    from nero_b200.evaluate import write_points_ply
    views, pts, tracks = objprep.read_colmap_model(flags.sparse, tracks=True)
    if not views:
        raise SystemExit(f'{flags.sparse}: the model has no images')
    t0 = time.time()
    cloud, info = mvs.reconstruct(views, pts, tracks, mvs.image_reader(flags.images), flags.max_size, flags.sources, flags.iterations,
                                  flags.radius, flags.step, flags.seed, flags.voxel, log=print)
    cloud = cloud.cpu().numpy()
    if info['views_used'] == 0:
        raise SystemExit('no view has enough source views and sparse points: nothing to reconstruct')
    write_points_ply(flags.output, cloud)
    kept = [int((d > 0).sum()) for d in info['depth'] if d is not None]
    print(f'{flags.sparse}: {len(views)} views, {info["views_used"]} reconstructed, {pts.shape[0]} sparse points; '
          f'{info["fused"]} fused points ({sum(kept) / max(1, len(kept)):.0f} per view)'
          + (f', {cloud.shape[0]} after the {flags.voxel:g} voxel grid' if flags.voxel else '') + f'; {time.time() - t0:.1f} s')
    print(f'wrote {flags.output}')


if __name__ == '__main__':
    main()
