"""Generate tests/golden/colmap_database.npz by running the UNMODIFIED reference database set-up on CPU.

    python oracle/make_golden_colmapdb.py [<path to the reference checkout>]

run_colmap.run_sfm runs through ref_shim with `true` in place of the COLMAP executable, on a directory of tiny images whose
names mix .jpg, .png, .PNG and .JPG, once per --same_camera setting: it creates database.db with its cameras and images,
and every COLMAP command it would run does nothing.  The same COLMAPDatabase (colmap/database.py) then adds known
keypoint, descriptor, match and two-view rows, one match set given in the reverse pair order.  The fixture holds the image
files, both databases as bytes and the known rows.  Two numpy-2 removals are shimmed for the reference: np.NaN (a default
argument of add_image) and ndarray.tostring (array_to_blob, restated as tobytes).  skimage.io.imread reads through cv2.
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
sys.path.insert(0, HERE)

# (name, width, height): ids follow the sorted paths of *.jpg, *.png, *.PNG, *.JPG
IMAGES = (('b_view.jpg', 24, 16), ('A_view.png', 20, 18), ('c_view.PNG', 16, 12), ('a_view.JPG', 22, 14), ('B2.jpg', 18, 18))


def known_rows():
    rng = np.random.RandomState(7)
    kp = {1: (rng.rand(5, 6) * 20).astype(np.float32), 2: (rng.rand(3, 6) * 20).astype(np.float32)}
    desc = {1: rng.randint(0, 256, (5, 128)).astype(np.uint8), 2: rng.randint(0, 256, (3, 128)).astype(np.uint8)}
    m12 = np.array([[0, 2], [3, 1], [4, 0]], np.uint32)
    m32 = np.array([[1, 0], [2, 2]], np.uint32)          # given as (image 3, image 2)
    F = rng.randn(3, 3)
    E = rng.randn(3, 3)
    return kp, desc, m12, m32, F, E


def main(ref):
    os.environ['NERO_REFERENCE_ROOT'] = ref
    import ref_shim
    ref_shim.REFERENCE_ROOT = ref
    ref_shim.install()
    import cv2
    np.NaN = np.nan
    sys.modules['skimage.io'].imread = lambda fn: cv2.imread(str(fn), cv2.IMREAD_COLOR)[..., ::-1]
    import colmap.database as cdb
    cdb.array_to_blob = lambda a: a.tobytes()
    import run_colmap
    kp, desc, m12, m32, F, E = known_rows()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        img_dir = os.path.join(tmp, 'images')
        os.makedirs(img_dir)
        rng = np.random.RandomState(3)
        for k, (name, w, h) in enumerate(IMAGES):
            path = os.path.join(img_dir, name)
            cv2.imwrite(path, rng.randint(0, 256, (h, w, 3)).astype(np.uint8))
            with open(path, 'rb') as f:
                out[f'image_{k}'] = np.frombuffer(f.read(), np.uint8)
        out['image_names'] = np.asarray([n for n, _, _ in IMAGES])
        for same in (False, True):
            proj = os.path.join(tmp, f'proj_{int(same)}')
            run_colmap.run_sfm(img_dir, proj, same_camera=same, colmap_path='true')
            db = cdb.COLMAPDatabase.connect(os.path.join(proj, 'database.db'))
            for i in (1, 2):
                db.add_keypoints(i, kp[i])
                db.add_descriptors(i, desc[i])
            db.add_matches(1, 2, m12)
            db.add_matches(3, 2, m32)
            db.add_two_view_geometry(1, 2, m12[:2], F=F, E=E, H=np.zeros((3, 3)), config=3)
            db.commit()
            db.close()
            with open(os.path.join(proj, 'database.db'), 'rb') as f:
                out[f'database_same{int(same)}'] = np.frombuffer(f.read(), np.uint8)
    for i in (1, 2):
        out[f'kp_{i}'], out[f'desc_{i}'] = kp[i], desc[i]
    out['m12'], out['m32'], out['F'], out['E'] = m12, m32, F, E
    path = os.path.join(GOLD, 'colmap_database.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: {len(IMAGES)} images, databases of {out["database_same0"].size} and {out["database_same1"].size} bytes')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
