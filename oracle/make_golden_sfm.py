"""Generate tests/golden/colmap_model.npz by running the UNMODIFIED reference model writer on CPU.

    python oracle/make_golden_sfm.py [<path to the reference checkout>]

colmap/read_write_model.write_model writes a small fixed model as .bin: 3 cameras (SIMPLE_PINHOLE, PINHOLE and
SIMPLE_RADIAL), 4 images (one without any POINTS2D entry, the others mixing keypoints with and without a point3D id) and
6 points with tracks of 2 to 5 observations.  The fixture holds the model's arrays and the three files' bytes, so the
package writer (nero_b200.objprep.write_colmap_model) can be checked byte for byte without the reference.
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), 'tests', 'golden')


def model():
    """(cameras, images, points) in the package writer's form, ids in insertion order."""
    rng = np.random.RandomState(11)
    cameras = {1: ('SIMPLE_PINHOLE', 640, 480, [576.5, 320.0, 240.0]), 2: ('PINHOLE', 800, 600, [700.25, 701.5, 400.0, 300.0]),
               3: ('SIMPLE_RADIAL', 320, 240, [290.0, 160.0, 120.0, -0.01])}
    tracks = {1: [(1, 0), (2, 1)], 2: [(1, 2), (2, 0), (3, 4)], 3: [(2, 3), (3, 0), (1, 4), (4, 1)],
              4: [(1, 1), (2, 2), (3, 1), (4, 0), (4, 3)], 5: [(3, 2), (4, 2)], 6: [(1, 3), (3, 3), (2, 4)]}
    nkp = {1: 6, 2: 5, 3: 5, 4: 4, 5: 0}
    p3d = {i: np.full(n, -1, np.int64) for i, n in nkp.items()}
    for pid, tr in tracks.items():
        for i, k in tr:
            p3d[i][k] = pid
    images = {}
    for iid, cid, name in ((1, 1, 'img_000.png'), (2, 2, 'b/img 001.jpg'), (3, 3, 'img_002.JPG'), (5, 1, 'empty.png'), (4, 2, 'img_003.png')):
        q = rng.randn(4)
        q /= np.linalg.norm(q)
        images[iid] = (q * np.sign(q[0]), rng.randn(3), cid, name, rng.rand(nkp[iid], 2) * 500, p3d[iid])
    points = {pid: (rng.randn(3), [int(v) for v in rng.randint(0, 256, 3)], float(rng.rand()), [i for i, _ in tr], [k for _, k in tr])
              for pid, tr in tracks.items()}
    return cameras, images, points


def main(ref):
    sys.path.insert(0, os.path.join(ref, 'colmap'))
    import read_write_model as rwm
    cameras, images, points = model()
    rc = {cid: rwm.Camera(id=cid, model=m, width=w, height=h, params=np.asarray(p, np.float64)) for cid, (m, w, h, p) in cameras.items()}
    ri = {iid: rwm.Image(id=iid, qvec=np.asarray(q), tvec=np.asarray(t), camera_id=cid, name=n, xys=np.asarray(x), point3D_ids=np.asarray(p))
          for iid, (q, t, cid, n, x, p) in images.items()}
    rp = {pid: rwm.Point3D(id=pid, xyz=np.asarray(x), rgb=np.asarray(c), error=e, image_ids=np.asarray(ii), point2D_idxs=np.asarray(kk))
          for pid, (x, c, e, ii, kk) in points.items()}
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        rwm.write_model(rc, ri, rp, tmp, '.bin')
        for n in ('cameras', 'images', 'points3D'):
            with open(os.path.join(tmp, f'{n}.bin'), 'rb') as f:
                out[f'{n}_bin'] = np.frombuffer(f.read(), np.uint8)
    path = os.path.join(GOLD, 'colmap_model.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: ' + ', '.join(f'{k} {v.size} bytes' for k, v in out.items()))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
