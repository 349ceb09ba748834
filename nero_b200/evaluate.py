"""Shape evaluation on the GPU: the Chamfer distance of eval_synthetic_shape.py and eval_real_shape.py, stated once.

Reference being replaced (paths relative to the reference repository):
  eval_synthetic_shape.py:16-25     nearest_dist: brute force in torch fp32, norm of the difference, minimum
  eval_synthetic_shape.py:39-60     rasterize_depth_map: nvdiffrast with an OpenGL context
  eval_synthetic_shape.py:62-84     get_mesh_eval_points: the 32 test views, unprojection, Open3D voxel_down_sample(0.01)
  eval_synthetic_shape.py:86-99     main: chamfer = (mean(nearest_dist(gt, pr)) + mean(nearest_dist(pr, gt))) / 2
  eval_real_shape.py                the same distance between the vertex sets of two PLY files
  dataset/database.py:227-259       GlossySyntheticDatabase: <k>-camera.pkl = (pose, K), <k>.png, <k>-depth.png
  dataset/database.py:422-458       test split configs/synthetic_split_128.pkl; ground-truth points and the eval_pts.ply cache
  utils/base_utils.py:44-52, 72-81  mask_depth_to_pts, project_points; :562-565, 583-584 pose_inverse, pose_apply

The protocol:
  * Predicted points.  For each test view the mesh's depth map is rendered (render_depth), the covered pixels are unprojected
    at their integer pixel coordinates (depth_to_points), moved to world space with the inverse pose, concatenated over the
    views in order and reduced by voxel_down_sample(0.01).
  * Ground-truth points.  <root>/eval_pts.ply when it exists; otherwise the same unprojection of the dataset's 16-bit depth
    PNGs, depth = v / 65535 * 15 kept where depth < 14.5, down-sampled the same way and written to eval_pts.ply as `double
    x y z` (what Open3D writes), so the cache is interchangeable with the reference's in both directions.
  * Chamfer = (mean(nearest_dist(gt, pr)) + mean(nearest_dist(pr, gt))) / 2 with fp32 distances and numpy's fp32 means.

Three consequences of the reference's rasteriser call, reproduced on purpose:
  1. Depth is interpolated linearly in screen space, because the clip-space w is 1.  For the closest hit of the ray through
     a pixel centre, with 3-D barycentrics b and vertex camera depths z_i, the rasteriser's depth is
     sum b_i z_i^2 / sum b_i z_i, not the ray depth sum b_i z_i.  It is slightly larger inside every triangle.
  2. There is a half-pixel shift.  nvdiffrast samples pixel (x, y) at projected coordinate (x + 1/2, y + 1/2), but the point
     is unprojected at (x, y).  The ground-truth path unprojects the same integer coordinates.
  3. Only depths in [0.5, 100] survive clipping (near and far planes of the clip-space z).  The ray cast keeps the closest
     hit only, so a surface nearer than 0.5 leaves the pixel empty where the rasteriser would show the surface behind it;
     the protocol's cameras are far from the object, so this does not arise in evaluation.

Two boundaries are restated rather than pinned (DESIGN.md section 2): nvdiffrast's coverage rule on silhouette edges (a ray
cast counts a pixel centre on an edge as covered) and Open3D's output order (hash order; here ascending voxel key).
"""
import os
import pickle

import numpy as np

NEAR, FAR = 0.5, 100.0        # rasterize_depth_map's clip planes (eval_synthetic_shape.py:48)
VOXEL = 0.01                  # voxel_down_sample(voxel_size=0.01)
GT_DEPTH_SCALE = 15.0         # GlossySyntheticDatabase.get_depth: v / 65535 * 15
GT_DEPTH_MAX = 14.5           #                                     mask = depth < 14.5
SPLIT = 'configs/synthetic_split_128.pkl'
_KEY_LIMIT = 1 << 21          # voxel index bits per axis (k_eval.cu)


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ depth maps
class DepthRenderer:
    """A triangle mesh resident on the GPU (BVH built once) whose depth maps render() produces as the reference's
    rasterize_depth_map does (rules 1-3 of the module docstring)."""

    def __init__(self, verts, tris, device='cuda'):
        torch = _torch()
        ops = _ops()
        ops.require_cuda(device, 'DepthRenderer')
        self.dev = torch.device(device)
        self.verts = np.ascontiguousarray(verts, np.float32).reshape(-1, 3)
        self.tris = np.ascontiguousarray(tris, np.int32).reshape(-1, 3)
        if self.tris.shape[0] == 0:
            raise ValueError('DepthRenderer needs at least one triangle')
        if self.tris.min() < 0 or self.tris.max() >= self.verts.shape[0]:
            raise ValueError('DepthRenderer: triangle index out of range')
        nodes, tri, ids = ops.bvh_build(self.verts, self.tris)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        self.nodes, self.tri, self.tri_ids, self.faces, self.verts_d = up(nodes), up(tri), up(ids), up(self.tris), up(self.verts)

    def render(self, pose, K, h, w, out=None, near=NEAR, far=FAR):
        """Depth map -> CUDA float32 [h,w], 0 where nothing is hit or the depth is outside [near, far].  pose: world -> camera
        [3,4] (OpenCV axes), K: [3,3] pinhole intrinsics without skew.  out: optional CUDA float32 tensor of h*w elements."""
        torch = _torch()
        K = np.asarray(K, np.float64)
        if K.shape != (3, 3) or K[0, 1] != 0 or K[1, 0] != 0 or tuple(K[2]) != (0, 0, 1):
            raise ValueError(f'render_depth needs pinhole intrinsics without skew, got {K.tolist()}')
        if out is None:
            out = torch.empty(h, w, dtype=torch.float32, device=self.dev)
        ops = _ops()
        q = ops.DepthParams().set(nodes=self.nodes, tris=self.tri, tri_ids=self.tri_ids, faces=self.faces, verts=self.verts_d, depth=out)
        q.pose[:] = [float(x) for x in np.asarray(pose, np.float32).reshape(12)]
        q.K[:] = [float(x) for x in K.astype(np.float32).reshape(9)]
        q.width, q.height, q.near_z, q.far_z = w, h, near, far
        ops.K('nero_depth_render', q)
        return out.view(h, w)


def render_depth(verts, tris, pose, K, h, w):
    """Replaces rasterize_depth_map(mesh, pose, K, (h, w)): (depth float32 [h,w], mask bool [h,w]) as numpy arrays."""
    d = DepthRenderer(verts, tris).render(pose, K, h, w).cpu().numpy()
    return d, d > 0


# ------------------------------------------------------------------------------------------------ points
def camera_table(poses, Ks):
    """[n,16] float64 rows (camera -> world rotation, camera centre, fx, fy, cx, cy), the layout nero_depth_points_emit reads:
    pose_inverse (base_utils.py:562-565) of each world -> camera pose."""
    rows = []
    for pose, K in zip(poses, Ks):
        pose = np.asarray(pose, np.float64)
        K = np.asarray(K, np.float64)
        if K[0, 1] != 0 or K[1, 0] != 0 or tuple(K[2]) != (0, 0, 1):
            raise ValueError(f'depth_to_points needs pinhole intrinsics without skew, got {K.tolist()}')
        R, t = pose[:, :3], pose[:, 3]
        rows.append(np.concatenate([R.T.reshape(9), -R.T @ t, [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]]))
    return np.asarray(rows, np.float64).reshape(-1, 16)


def depth_to_points_cuda(depth, poses, Ks, lo=0.0, hi=float('inf')):
    """World points of the pixels with lo < depth < hi of CUDA depth maps [n_views,h,w] (or [h,w] with one pose), in (view,
    row, column) order -> CUDA float32 [n,3].  poses [n_views,3,4] world -> camera, Ks [n_views,3,3].  Reads the point count
    back once to size the output."""
    torch = _torch()
    ops = _ops()
    ops.require_cuda(depth.device, 'depth_to_points')
    d = depth.to(torch.float32).contiguous()
    if d.dim() == 2:
        d, poses, Ks = d[None], [poses], [Ks]
    nv, h, w = d.shape
    cams = torch.from_numpy(camera_table(poses, Ks)).to(d.device)
    if cams.shape[0] != nv:
        raise ValueError(f'{cams.shape[0]} cameras for {nv} depth maps')
    nblk = ops.ceil_div(nv * h * w, 1024)
    blk_cnt = torch.empty(nblk, dtype=torch.int32, device=d.device)
    blk_off = torch.empty(nblk, dtype=torch.int64, device=d.device)
    total = torch.empty(1, dtype=torch.int64, device=d.device)
    ops.K('nero_depth_points_count', d, nv, h, w, lo, hi, blk_cnt, blk_off, total, launches=2)
    n = int(total.item())
    pts = torch.empty(n, 3, dtype=torch.float32, device=d.device)
    ops.K('nero_depth_points_emit', d, nv, h, w, lo, hi, cams, blk_off, n, pts, launches=int(n > 0))
    return pts


def depth_to_points(depth, K, pose, lo=0.0, hi=float('inf')):
    """Replaces mask_depth_to_pts(depth > lo & depth < hi, depth, K) followed by pose_apply(pose_inverse(pose), .):
    numpy depth [h,w] -> world points float32 [n,3] in row-major pixel order.  The reference's masks are (0, inf) for a
    rendered depth map (covered pixels) and (-inf, 14.5) for a GlossySynthetic depth PNG."""
    torch = _torch()
    d = torch.from_numpy(np.ascontiguousarray(depth, np.float32)).cuda()
    return depth_to_points_cuda(d, pose, K, lo, hi).cpu().numpy()


# ------------------------------------------------------------------------------------------------ voxel down-sampling
def voxel_down_sample_cuda(pts, voxel=VOXEL):
    """Open3D's PointCloud.voxel_down_sample in fp64 on a CUDA tensor [n,3] -> CUDA float64 [m,3].

    As Open3D: min bound = the cloud's minimum - voxel/2, voxel index floor((p - min bound) / voxel), each output point the
    mean of its voxel's points.  The sums run in input order.  Output order is ascending voxel key (i, j, k), where Open3D's
    is the iteration order of its hash map; the set of points is the same.  Raises ValueError if the grid would need more
    than 2^21 cells along an axis."""
    torch = _torch()
    ops = _ops()
    ops.require_cuda(pts.device, 'voxel_down_sample')
    if not voxel > 0:
        raise ValueError(f'voxel size must be positive, got {voxel}')
    p = pts.to(torch.float64).reshape(-1, 3).contiguous()
    n = p.shape[0]
    if n == 0:
        return p.new_zeros(0, 3)
    lo, hi = p.amin(0).cpu().numpy(), p.amax(0).cpu().numpy()
    bounds = np.ascontiguousarray(np.concatenate([lo - voxel * 0.5, hi]), np.float64)
    if (np.floor((bounds[3:] - bounds[:3]) / voxel) >= _KEY_LIMIT).any() or not np.isfinite(bounds).all():
        raise ValueError(f'voxel_down_sample: extent {hi - lo} at voxel {voxel} needs more than {_KEY_LIMIT} cells along an axis')
    keys = torch.empty(n, dtype=torch.int64, device=p.device)
    ops.K('nero_voxel_keys', p, n, bounds, voxel, keys)
    skeys, order = torch.sort(keys, stable=True)            # plumbing: stable, so each voxel keeps its points in input order
    _, counts = torch.unique_consecutive(skeys, return_counts=True)
    ends = torch.cumsum(counts, 0)
    m = ends.shape[0]
    out = torch.empty(m, 3, dtype=torch.float64, device=p.device)
    ops.K('nero_voxel_mean', p, order, ends, m, out)
    return out


def voxel_down_sample(points, voxel=VOXEL):
    """Replaces open3d PointCloud.voxel_down_sample(voxel): numpy [n,3] -> float64 [m,3] (see voxel_down_sample_cuda)."""
    torch = _torch()
    p = torch.from_numpy(np.ascontiguousarray(points, np.float64).reshape(-1, 3)).cuda()
    return voxel_down_sample_cuda(p, voxel).cpu().numpy()


# ------------------------------------------------------------------------------------------------ distances
def nearest_dist_cuda(q, t):
    """Exact nearest distance from each row of q [n,3] to the set t [m,3] (CUDA tensors, cast to float32) -> CUDA float32 [n]."""
    torch = _torch()
    ops = _ops()
    ops.require_cuda(q.device, 'nearest_dist')
    q = q.to(torch.float32).reshape(-1, 3).contiguous()
    t = t.to(torch.float32).reshape(-1, 3).contiguous()
    if q.shape[0] == 0 or t.shape[0] == 0:
        raise ValueError(f'nearest_dist needs two non-empty point sets, got {q.shape[0]} and {t.shape[0]} points')
    out = torch.empty(q.shape[0], dtype=torch.float32, device=q.device)
    ops.K('nero_nearest_dist', q, q.shape[0], t, t.shape[0], out)
    return out


def nearest_dist(pts0, pts1, batch_size=None):
    """Replaces eval_synthetic_shape.nearest_dist(pts0, pts1, batch_size): numpy in, float32 numpy out.  batch_size is
    accepted for compatibility and ignored (the kernel tiles the targets itself)."""
    torch = _torch()
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32).reshape(-1, 3)).cuda()
    return nearest_dist_cuda(up(pts0), up(pts1)).cpu().numpy()


def chamfer_distance(pts_gt, pts_pr):
    """(chamfer, dist_gt, dist_pr) as main() computes them: fp32 distances both ways and (mean + mean) / 2 with numpy."""
    dist_gt = nearest_dist(pts_gt, pts_pr)
    dist_pr = nearest_dist(pts_pr, pts_gt)
    return (np.mean(dist_gt) + np.mean(dist_pr)) / 2, dist_gt, dist_pr


def result_line(stem, chamfer):
    """The line the reference prints and appends to data/geometry.log."""
    return f'{stem} {chamfer:.5f}'


# ------------------------------------------------------------------------------------------------ GlossySynthetic data
def png_size(path):
    """(height, width) from a PNG's IHDR chunk."""
    with open(path, 'rb') as f:
        head = f.read(24)
    if head[:8] != b'\x89PNG\r\n\x1a\n' or head[12:16] != b'IHDR':
        raise ValueError(f'{path}: not a PNG file')
    return int.from_bytes(head[20:24], 'big'), int.from_bytes(head[16:20], 'big')


def read_camera(root, img_id):
    """(pose float32 [3,4] world -> camera, K float32 [3,3]) from <root>/<id>-camera.pkl (GlossySyntheticDatabase)."""
    with open(os.path.join(root, f'{img_id}-camera.pkl'), 'rb') as f:
        pose, K = pickle.load(f)[:2]
    return np.asarray(pose).astype(np.float32), np.asarray(K).astype(np.float32)


def read_gt_depth(root, img_id):
    """get_depth: float32 depth [h,w] = v / 65535 * 15 of the 16-bit <root>/<id>-depth.png."""
    import cv2
    path = os.path.join(root, f'{img_id}-depth.png')
    raw = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if raw is None:
        raise FileNotFoundError(path)
    if raw.ndim == 3:
        raw = raw[..., 0]
    return raw.astype(np.float32) / 65535 * GT_DEPTH_SCALE


def split_test_ids(split_path=SPLIT):
    """get_database_split(database, 'test'): the first list of the split pickle."""
    with open(split_path, 'rb') as f:
        return [str(i) for i in pickle.load(f)[0]]


def read_views(root, ids):
    """[(pose, K, (h, w))] of the given views; the size comes from the header of <root>/<id>.png."""
    return [read_camera(root, i) + (png_size(os.path.join(root, f'{i}.png')),) for i in ids]


def _stack_points(depths, views, lo, hi):
    """World points of several depth maps (CUDA [h,w] each), concatenated in view order; views of one size share a launch."""
    torch = _torch()
    out, i = [], 0
    while i < len(depths):
        j = i
        while j < len(depths) and depths[j].shape == depths[i].shape:
            j += 1
        out.append(depth_to_points_cuda(torch.stack(depths[i:j]), [v[0] for v in views[i:j]], [v[1] for v in views[i:j]], lo, hi))
        i = j
    return torch.cat(out, 0)


def mesh_eval_points_cuda(verts, tris, views, voxel=VOXEL):
    """get_mesh_eval_points: CUDA float64 [m,3] voxel means of the mesh's rendered depth over the views."""
    r = DepthRenderer(verts, tris)
    depths = [r.render(pose, K, h, w) for pose, K, (h, w) in views]
    return voxel_down_sample_cuda(_stack_points(depths, views, 0.0, float('inf')), voxel)


def gt_eval_points_cuda(root, views_ids, views, voxel=VOXEL):
    """get_database_eval_points without the cache: CUDA float64 [m,3] voxel means of the dataset's depth PNGs."""
    torch = _torch()
    depths = [torch.from_numpy(read_gt_depth(root, i)).cuda() for i in views_ids]
    return voxel_down_sample_cuda(_stack_points(depths, views, float('-inf'), GT_DEPTH_MAX), voxel)


def synthetic_eval_points(root, mesh_path, split_path=SPLIT):
    """(pts_gt, pts_pr) as numpy arrays for a GlossySynthetic object directory and a mesh.  Reads <root>/eval_pts.ply when it
    exists (float64, as Open3D returns it); otherwise computes the ground truth and writes that file."""
    from .material import read_ply
    ids = split_test_ids(split_path)
    views = read_views(root, ids)
    cache = os.path.join(root, 'eval_pts.ply')
    if os.path.exists(cache):
        pts_gt = read_points_ply(cache)
    else:
        g = gt_eval_points_cuda(root, ids, views).cpu().numpy()
        write_points_ply(cache, g)
        print(f'point number {len(g)} ...')
        pts_gt = g.astype(np.float32)
    verts, tris = read_ply(mesh_path)
    pts_pr = mesh_eval_points_cuda(verts, tris, views).cpu().numpy().astype(np.float32)
    return pts_gt, pts_pr


# ------------------------------------------------------------------------------------------------ point-cloud PLY
_PLY_TYPES = {'char': 'i1', 'uchar': 'u1', 'short': 'i2', 'ushort': 'u2', 'int': 'i4', 'uint': 'u4', 'float': 'f4', 'double': 'f8',
              'int8': 'i1', 'uint8': 'u1', 'int16': 'i2', 'uint16': 'u2', 'int32': 'i4', 'uint32': 'u4', 'float32': 'f4',
              'float64': 'f8'}


def read_points_ply(path):
    """Vertex positions float64 [n,3] of a PLY file (the point cloud of Open3D's read_point_cloud, or the vertices of
    read_triangle_mesh).  ascii or binary_little_endian; x, y, z float or double; other vertex properties are skipped; the
    vertex element must come first, and later elements (faces) are not read."""
    with open(path, 'rb') as f:
        if f.readline().strip() != b'ply':
            raise ValueError(f'{path}: not a PLY file')
        fmt, elems = None, []
        while True:
            line = f.readline()
            if not line:
                raise ValueError(f'{path}: PLY header has no end_header')
            t = line.decode('ascii', 'replace').split()
            if not t or t[0] in ('comment', 'obj_info'):
                continue
            if t[0] == 'end_header':
                break
            if t[0] == 'format':
                fmt = t[1]
            elif t[0] == 'element':
                elems.append((t[1], int(t[2]), []))
            elif t[0] == 'property' and elems:
                elems[-1][2].append(t[1:])
        if fmt not in ('ascii', 'binary_little_endian'):
            raise ValueError(f'{path}: PLY format {fmt} is not supported')
        if not elems or elems[0][0] != 'vertex':
            raise ValueError(f'{path}: the first PLY element must be vertex')
        _, n, props = elems[0]
        names = [p[-1] for p in props]
        if any(c not in names for c in 'xyz'):
            raise ValueError(f'{path}: vertex element lacks x, y or z')
        if fmt == 'ascii':
            rows = [f.readline().split() for _ in range(n)]
            if any(p[0] == 'list' for p in props):
                return np.asarray([[float(r[names.index(c)]) for c in 'xyz'] for r in rows], np.float64).reshape(-1, 3)
            a = np.asarray(rows, np.float64).reshape(n, len(props))
            return np.ascontiguousarray(a[:, [names.index(c) for c in 'xyz']])
        if any(p[0] == 'list' for p in props):
            raise ValueError(f'{path}: list properties in a binary vertex element are not supported')
        dt = np.dtype([(p[-1], '<' + _PLY_TYPES[p[0]]) for p in props])
        raw = np.frombuffer(f.read(dt.itemsize * n), dtype=dt, count=n)
        return np.stack([raw[c].astype(np.float64) for c in 'xyz'], -1)


def write_points_ply(path, points):
    """Binary little-endian PLY with `double x y z` per vertex and no other element, the layout of Open3D's
    write_point_cloud for a cloud without normals or colours."""
    p = np.ascontiguousarray(points, '<f8').reshape(-1, 3)
    header = (f'ply\nformat binary_little_endian 1.0\ncomment Created by nero_b200\nelement vertex {p.shape[0]}\n'
              'property double x\nproperty double y\nproperty double z\nend_header\n')
    with open(path, 'wb') as f:
        f.write(header.encode('ascii'))
        f.write(p.tobytes())
