"""Generate tests/golden/eval_shape.npz by running the UNMODIFIED reference glue of eval_synthetic_shape.py on CPU.

    python oracle/make_golden_eval.py [<path to the reference checkout>]

What runs unmodified (through ref_shim, .cuda() mapped to the CPU): main, get_mesh_eval_points, nearest_dist,
rasterize_depth_map, get_database_eval_points, get_database_split, GlossySyntheticDatabase.get_depth / get_K / get_pose,
project_points, mask_depth_to_pts, pose_inverse, pose_apply.
What is stubbed: the database's image reader (returns the fixture's 16-bit depth PNGs and RGB images of the right size),
trimesh.load_mesh (returns the fixture mesh), dr.rasterize (records the clip-space vertices it is given and answers with the
oracle rasteriser, nero_oracle_eval.rasterize), Open3D's PointCloud.voxel_down_sample (records its input and answers with
nero_oracle_eval.voxel_down_sample) and read/write_point_cloud (no cache: the ground truth is computed).
This pins the reference's camera, NDC and unprojection conventions and its glue; the two third-party boundaries stay
restatements (DESIGN.md section 2).  TEST INFRASTRUCTURE ONLY.
"""
import os
import pickle
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
sys.path.insert(0, HERE)

import nero_oracle_eval as OE  # noqa: E402
import nero_oracle_mat as OM  # noqa: E402

H, W = 24, 32
IDS = ['2', '0', '1']              # test split order differs from file order on purpose


def look_at(c, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    c = np.asarray(c, np.float64)
    z = np.asarray(target) - c
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 0)
    return np.concatenate([R, (-R @ c)[:, None]], 1)


def fixture():
    verts, tris = OM.test_scene(1)
    poses = [look_at([2.2, 0.4, 0.6]), look_at([-0.5, 2.0, -0.8]), look_at([0.3, -1.1, 1.9])]
    Ks = [np.asarray([[30.0, 0, 15.2], [0, 28.0, 11.7], [0, 0, 1]]), np.asarray([[26.0, 0, 17.0], [0, 26.0, 12.4], [0, 0, 1]]),
          np.asarray([[33.0, 0, 16.5], [0, 31.0, 10.9], [0, 0, 1]])]
    # ground-truth depth PNGs: the oracle depth of a slightly larger mesh, 65535 (= 15, masked out) where empty
    depths = []
    for pose, K in zip(poses, Ks):
        d, m = OE.render_depth(verts * 1.02, tris, pose.astype(np.float32), K.astype(np.float32), H, W)
        depths.append(np.where(m, np.round(d / 15 * 65535), 65535).astype(np.uint16))
    return verts, tris, poses, Ks, depths


def main(ref):
    os.environ['NERO_REFERENCE_ROOT'] = ref
    import ref_shim
    ref_shim.REFERENCE_ROOT = ref
    verts, tris, poses, Ks, depths = fixture()
    rec = {'clip': [], 'voxel_in': [], 'nearest': []}

    o3d = types.ModuleType('open3d')

    class PointCloud:
        def __init__(self):
            self.points = None

        def voxel_down_sample(self, voxel_size):
            rec['voxel_in'].append(np.asarray(self.points).copy())
            out = PointCloud()
            out.points = OE.voxel_down_sample(self.points, voxel_size)
            return out
    o3d.geometry = types.SimpleNamespace(PointCloud=PointCloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a, np.float64))
    o3d.io = types.SimpleNamespace(read_point_cloud=None, write_point_cloud=lambda fn, pcd: None)
    sys.modules['open3d'] = o3d

    def rasterize(ctx, pos, tri, resolution):
        import torch
        clip = pos[0].numpy().astype(np.float64)
        rec['clip'].append(clip.copy())
        rast = OE.rasterize(clip, tri.numpy(), *resolution)
        return torch.from_numpy(rast[None].astype(np.float32)), None

    ref_shim.install()
    import nvdiffrast.torch as dr
    dr.rasterize = rasterize
    dr.RasterizeGLContext = lambda *a, **k: None
    import trimesh
    trimesh.load_mesh = lambda path: types.SimpleNamespace(vertices=verts, faces=tris)
    import eval_synthetic_shape as ES
    import dataset.database as DB

    def imread(path):
        name = os.path.basename(path)
        if name.endswith('-depth.png'):
            return depths[int(name.split('-')[0])]
        return np.zeros((H, W, 4), np.uint8)
    DB.imread = imread
    ref_nearest = ES.nearest_dist

    def nearest(p0, p1, batch_size=512):
        d = ref_nearest(p0, p1, batch_size)
        rec['nearest'].append((np.asarray(p0, np.float32), np.asarray(p1, np.float32), d))
        return d
    ES.nearest_dist = nearest

    db = DB.GlossySyntheticDatabase.__new__(DB.GlossySyntheticDatabase)
    db.root = 'data/GlossySynthetic/fixture'
    db.img_num = 3
    db.img_ids = ['0', '1', '2']
    db.cams = [(poses[k], Ks[k]) for k in range(3)]
    db.scale_factor = 1.0
    ES.parse_database_name = lambda name: db
    ES.args = types.SimpleNamespace(mesh='fixture_mesh.ply', object='fixture', batch_size=512)
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, 'configs'))
        os.makedirs(os.path.join(tmp, 'data', 'GlossySynthetic', 'fixture'))
        with open(os.path.join(tmp, 'configs', 'synthetic_split_128.pkl'), 'wb') as f:
            pickle.dump([np.asarray(IDS), ['3']], f)
        old = os.getcwd()
        os.chdir(tmp)
        try:
            ES.main()
            with open('data/geometry.log') as f:
                line = f.read().strip()
        finally:
            os.chdir(old)
    (gt0, pr0, dist_gt), (pr1, gt1, dist_pr) = rec['nearest']
    out = {'verts': verts, 'tris': tris, 'poses': np.stack(poses), 'Ks': np.stack(Ks), 'depth_png': np.stack(depths),
           'ids': np.asarray([int(i) for i in IDS]), 'hw': np.asarray([H, W]),
           'clip': np.stack(rec['clip']), 'gt_points_in': rec['voxel_in'][0], 'pr_points_in': rec['voxel_in'][1],
           'pts_gt': gt0, 'pts_pr': pr0, 'dist_gt': dist_gt, 'dist_pr': dist_pr,
           'chamfer': np.float64(float(line.split()[1])), 'chamfer_exact': np.float64((np.mean(dist_gt) + np.mean(dist_pr)) / 2)}
    assert np.array_equal(gt0, gt1) and np.array_equal(pr0, pr1)
    np.savez_compressed(os.path.join(GOLD, 'eval_shape.npz'), **out)
    print('eval_shape saved', line, {k: np.shape(v) for k, v in out.items()})


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else '/root/reference')
