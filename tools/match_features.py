"""Extract and match SIFT features of a custom object's images on the GPU: <root>/database.db, ready for map_sparse.py.

    python tools/match_features.py --root data/custom/kettle [--images <dir>] [--same_camera] [--max-size 3200]
        [--max-features 8192] [--camera-model SIMPLE_PINHOLE|SIMPLE_RADIAL] [--force]

Replaces the first three steps of run_colmap.py: the database with one SIMPLE_PINHOLE camera per image (or one shared
camera with --same_camera), COLMAP's feature_extractor and its exhaustive_matcher.  The database holds the cameras,
images, keypoints, descriptors, the matches of every image pair and the verified two-view geometries, in COLMAP's
schema.  The next step is map_sparse.py, the GPU mapper (COLMAP's CPU `colmap mapper` reads the same database); the
tool prints both commands.  The workflow becomes: match_features.py -> map_sparse.py -> dense_points.py ->
prepare_custom_object.py.
--camera-model SIMPLE_RADIAL gives every camera SIMPLE_RADIAL (f, w / 2, h / 2, 0), for a mapper that estimates the lens
distortion (COLMAP's); undistort_images.py then turns that model and its images into a pinhole project.
The protocol and its defaults are stated in nero_b200/features.py.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse_args(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--root', type=str, required=True, help='data/custom/<object>')
    parser.add_argument('--images', type=str, default=None, help='image directory (default <root>/images)')
    parser.add_argument('--same_camera', action='store_true', help='one camera for every image')
    parser.add_argument('--max-size', type=int, default=3200, help='longest side of the grey images features are extracted from')
    parser.add_argument('--max-features', type=int, default=8192, help='features per image')
    parser.add_argument('--camera-model', choices=('SIMPLE_PINHOLE', 'SIMPLE_RADIAL'), default='SIMPLE_PINHOLE',
                        help='camera model of every camera of the database')
    parser.add_argument('--force', action='store_true', help='overwrite an existing database')
    flags = parser.parse_args(argv)
    if not os.path.isdir(flags.root):
        parser.error(f'--root {flags.root} is not a directory')
    if flags.images is None:
        flags.images = os.path.join(flags.root, 'images')
    if not os.path.isdir(flags.images):
        parser.error(f'--images {flags.images} is not a directory')
    if flags.max_size < 1 or flags.max_features < 1:
        parser.error('--max-size and --max-features must be >= 1')
    flags.database = os.path.join(flags.root, 'database.db')
    if os.path.exists(flags.database) and not flags.force:
        parser.error(f'{flags.database} exists (give --force to overwrite it)')
    return flags


def main(argv=None):
    flags = parse_args(argv)
    from nero_b200 import features
    if os.path.exists(flags.database):
        os.remove(flags.database)
    info = features.build_database(flags.images, flags.database, flags.same_camera, flags.max_size, flags.max_features, log=print,
                                   camera_model=flags.camera_model)
    t = info['times']
    print(f'{flags.database}: {len(info["names"])} images, {sum(info["features"])} features, {info["pairs"]} matched pairs, '
          f'{info["verified"]} verified (extract {t["extract"]:.2f} s, match {t["match"]:.2f} s, verify {t["verify"]:.2f} s, '
          f'write {t["write"]:.2f} s)')
    os.makedirs(os.path.join(flags.root, 'sparse'), exist_ok=True)
    if flags.camera_model == 'SIMPLE_RADIAL':
        print('next: colmap mapper --database_path {0}/database.db --image_path {1} --output_path {0}/sparse, then '
              'python tools/undistort_images.py --root {0} --output <dir>'.format(flags.root, flags.images))
        return info
    print(f'next: python tools/map_sparse.py --root {flags.root}')
    print('  (or COLMAP\'s CPU mapper: colmap mapper --database_path {0}/database.db --image_path {1} --output_path {0}/sparse)'
          .format(flags.root, flags.images))
    return info


if __name__ == '__main__':
    main()
