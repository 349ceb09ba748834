"""Undistort a custom object's images on the GPU: a pinhole project from a COLMAP model with SIMPLE_RADIAL cameras.

    python tools/undistort_images.py --root data/custom/kettle --output <dir> [--sparse <model dir>] [--images <dir>] [--force]

Replaces run_colmap.py's image_undistorter step.  Writes <output>/images/<same name> and <output>/sparse/0 with
SIMPLE_PINHOLE cameras, the same image ids, names and poses, POINTS2D in the undistorted images and the same points3D.
Pinhole cameras (SIMPLE_PINHOLE, PINHOLE) pass through and their images are copied unchanged; any other camera model is
refused.  The rule that picks each undistorted camera, and the resampling, are stated in nero_b200/undistort.py.

--sparse defaults to <root>/colmap/sparse/0, else <root>/sparse/0; --images to <root>/images.  The workflow for a lens
with distortion is: match_features.py --camera-model SIMPLE_RADIAL -> colmap mapper -> undistort_images.py ->
dense_points.py --root <output> -> prepare_custom_object.py --root <output>.
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
    parser.add_argument('--output', type=str, required=True, help='directory of the undistorted project')
    parser.add_argument('--sparse', type=str, default=None, help='COLMAP sparse model directory')
    parser.add_argument('--images', type=str, default=None, help='image directory (default <root>/images)')
    parser.add_argument('--force', action='store_true', help='write into an existing output directory')
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
    if os.path.exists(flags.output) and not flags.force:
        parser.error(f'{flags.output} already exists: pass --force to write into it')
    return flags


def main(argv=None):
    flags = parse_args(argv)
    from nero_b200 import undistort
    try:
        undistort.plan(flags.sparse)              # every refusal of the model before any GPU work
    except (ValueError, FileNotFoundError) as e:
        raise SystemExit(f'{flags.sparse}: {e}')
    t0 = time.time()
    try:
        info = undistort.project(flags.sparse, flags.images, flags.output, log=print)
    except (ValueError, FileNotFoundError) as e:
        raise SystemExit(f'{flags.sparse}: {e}')
    for cid, (model, w, h, par) in info['cameras'].items():
        print(f'camera {cid}: {model} {w} x {h} ' + ' '.join(f'{v:.6g}' for v in par))
    print(f'{flags.sparse}: {info["warped"]} images undistorted, {info["copied"]} copied, {info["points"]} points; '
          f'{time.time() - t0:.1f} s')
    print(f'wrote {flags.output}/images and {flags.output}/sparse/0')
    print(f'next: python tools/dense_points.py --root {flags.output}')
    return info


if __name__ == '__main__':
    main()
