"""Generate tests/golden/objprep_colmap.npz by running the UNMODIFIED reference reader and normaliser on CPU.

    python oracle/make_golden_objprep.py [<path to the reference checkout>]

The fixture holds a small synthetic COLMAP model (the cameras of nero_oracle_objprep.scene, with PINHOLE, SIMPLE_RADIAL and
SIMPLE_PINHOLE cameras, image ids descending while names ascend) written from the published format in both the binary
and the text form, an object_point_cloud.ply written by nero_b200.evaluate.write_points_ply and a meta_info.txt written by
nero_b200.objprep.write_meta_info, all as bytes.  What runs unmodified (through ref_shim): colmap/read_write_model.read_model,
CustomDatabase._parse_colmap (poses, Ks, names, image order), and CustomDatabase._normalize with its PLY reader
colmap/plyfile and _compute_rotation (ref_points, scale_rect, offset_rect, R_rect).  TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import nero_oracle_objprep as OO  # noqa: E402

FILES = ('cameras', 'images', 'points3D')


def fixture():
    sc = OO.scene(n_table=3000, n_obj=2000, n_cams=7, seed=3)
    cams, images, points = OO.scene_model(sc)
    obj = sc['points'][sc['label'] == 1][:500]
    up = sc['up']
    v = sc['poses'][2]
    c = -v[:, :3].T @ v[:, 3]
    f = c - sc['center']
    forward = (f - (f @ up) * up) / np.linalg.norm(f - (f @ up) * up)
    return sc, cams, images, points, obj, up, forward


def main(ref):
    os.environ['NERO_REFERENCE_ROOT'] = ref
    import ref_shim
    ref_shim.REFERENCE_ROOT = ref
    ref_shim.install()
    from dataset.database import CustomDatabase
    from colmap.read_write_model import read_model
    from nero_b200.evaluate import write_points_ply
    from nero_b200.objprep import write_meta_info
    sc, cams, images, points, obj, up, forward = fixture()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for fmt in ('bin', 'txt'):
            root = os.path.join(tmp, fmt)
            model = os.path.join(root, 'colmap', 'sparse', '0')
            OO.write_colmap_model(model, cams, images, points, fmt)
            for n in FILES:
                with open(os.path.join(model, f'{n}.{fmt}'), 'rb') as f:
                    out[f'{n}_{fmt}'] = np.frombuffer(f.read(), np.uint8)
            write_points_ply(os.path.join(root, 'object_point_cloud.ply'), obj)
            write_meta_info(os.path.join(root, 'meta_info.txt'), up, forward)
            db = object.__new__(CustomDatabase)
            db.root = root
            db._parse_colmap()
            ids = list(db.img_ids)
            out[f'ids_{fmt}'] = np.asarray(ids, np.int64)
            out[f'names_{fmt}'] = np.asarray([db.image_names[i] for i in ids])
            out[f'poses_{fmt}'] = np.stack([db.poses[i] for i in ids])
            out[f'Ks_{fmt}'] = np.stack([db.Ks[i] for i in ids])
            out[f'points_{fmt}'] = np.stack([p.xyz for p in read_model(model)[2].values()])
            db._normalize()
            out[f'ref_points_{fmt}'] = db.ref_points
            out[f'scale_rect_{fmt}'] = np.float64(db.scale_rect)
            out[f'offset_rect_{fmt}'] = db.offset_rect
            out[f'R_rect_{fmt}'] = db.R_rect
        with open(os.path.join(tmp, 'bin', 'object_point_cloud.ply'), 'rb') as f:
            out['ply'] = np.frombuffer(f.read(), np.uint8)
        with open(os.path.join(tmp, 'bin', 'meta_info.txt'), 'rb') as f:
            out['meta_info'] = np.frombuffer(f.read(), np.uint8)
    out['obj'], out['up'], out['forward'] = obj, up, forward
    for fmt in ('bin', 'txt'):
        assert np.array_equal(out[f'poses_{fmt}'], out['poses_bin']) and np.array_equal(out[f'Ks_{fmt}'], out['Ks_bin'])
    path = os.path.join(GOLD, 'objprep_colmap.npz')
    np.savez_compressed(path, **out)
    print(f'wrote {path}: {len(out["ids_bin"])} images, {out["points_bin"].shape[0]} sparse points, {obj.shape[0]} object points')


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
