"""Reconstruct cameras, poses and sparse points of a custom object on the GPU: <root>/sparse/0 from <root>/database.db.

    python tools/map_sparse.py --root data/custom/kettle [--database <db>] [--output <dir>] [--images <dir>]
        [--camera-model SIMPLE_PINHOLE|SIMPLE_RADIAL] [--force]

Replaces `colmap mapper` of run_colmap.py: an incremental mapper (initial pair, P3P registration, triangulation and
bundle adjustment after every image) over the verified matches that match_features.py stored, written as the COLMAP
binary model (cameras.bin, images.bin, points3D.bin) that dense_points.py and prepare_custom_object.py read.  The
workflow becomes: match_features.py -> map_sparse.py -> dense_points.py -> prepare_custom_object.py.  The images only give
the points' colours.  The protocol and its defaults are stated in nero_b200/sfm.py.

--camera-model SIMPLE_RADIAL estimates each camera's radial distortion k beside its focal, for a database written by
match_features.py --camera-model SIMPLE_RADIAL (photos from a phone or a kit lens); the model then has SIMPLE_RADIAL
cameras, and undistort_images.py turns it into the pinhole project that dense_points.py reads.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MODEL_FILES = ('cameras.bin', 'images.bin', 'points3D.bin')


def parse_args(argv=None):
    """Parse and check the arguments; every refusal happens here, before any GPU work.  -> (flags, database)."""
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--root', type=str, required=True, help='data/custom/<object>')
    parser.add_argument('--database', type=str, default=None, help='COLMAP database (default <root>/database.db)')
    parser.add_argument('--output', type=str, default=None, help='model directory (default <root>/sparse/0)')
    parser.add_argument('--images', type=str, default=None, help='image directory for the point colours (default <root>/images)')
    parser.add_argument('--camera-model', choices=('SIMPLE_PINHOLE', 'SIMPLE_RADIAL'), default='SIMPLE_PINHOLE',
                        help='camera model to estimate; every camera of the database must have it (default SIMPLE_PINHOLE)')
    parser.add_argument('--force', action='store_true', help='overwrite an existing model')
    flags = parser.parse_args(argv)
    if not os.path.isdir(flags.root):
        parser.error(f'--root {flags.root} is not a directory')
    flags.database = flags.database or os.path.join(flags.root, 'database.db')
    flags.output = flags.output or os.path.join(flags.root, 'sparse', '0')
    flags.images = flags.images or os.path.join(flags.root, 'images')
    if any(os.path.exists(os.path.join(flags.output, f)) for f in MODEL_FILES) and not flags.force:
        parser.error(f'{flags.output} holds a model (give --force to overwrite it)')
    if not os.path.isfile(flags.database):
        parser.error(f'{flags.database}: no database (run match_features.py first)')
    from nero_b200 import sfm
    db = sfm.read_database(flags.database)
    try:
        sfm.check_database(db, flags.camera_model)
    except ValueError as e:
        parser.error(f'{flags.database}: {e}')
    if not os.path.isdir(flags.images):
        parser.error(f'--images {flags.images} is not a directory')
    return flags, db


def main(argv=None):
    flags, _ = parse_args(argv)
    from nero_b200 import sfm
    s = sfm.map_sparse(flags.database, flags.output, flags.images, log=print, camera_model=flags.camera_model)
    n = len(s['names'])
    print(f'{flags.output}: {len(s["registered"])} of {n} images registered')
    if s['unregistered']:
        print('  not registered: ' + ', '.join(s['names'][i] for i in s['unregistered']))
    print(f'  {s["points"]} points, mean track length {s["mean_track"]:.2f}, mean reprojection error {s["mean_error"]:.3f} px')
    print('  focal: ' + ', '.join(f'camera {c} {f:.2f}' for c, f in s['focals'].items()))
    if 'radial' in s:
        print('  k: ' + ', '.join(f'camera {c} {k:.5f}' for c, k in s['radial'].items()))
        for w in s['warnings']:
            print(f'  warning: undistort_images.py will refuse {w}')
    t = s['times']
    print('  time: ' + ', '.join(f'{k} {t[k]:.2f} s' for k in ('read', 'tracks', 'init', 'register', 'triangulate', 'bundle', 'write', 'total')))
    return s


if __name__ == '__main__':
    main()
