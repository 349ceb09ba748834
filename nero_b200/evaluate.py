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

The real-data protocol (the reference's eval.md, "Evaluate the Glossy Real dataset") cleans the stage-I mesh by hand in
MeshLab, samples 500 k points uniformly on its surface and on the ground-truth mesh in CloudCompare, and runs
eval_real_shape.py on the two clouds.  clean_mesh and sample_surface replace the two GUI steps (k_meshpts.cu):
  * Crop.  A triangle is kept iff its three vertices lie inside the sphere (centre, radius) and / or the axis-aligned box,
    tested in fp64.  Triangles are never clipped.
  * Components.  Two kept triangles are connected when they share a vertex index (vertices are not welded by position:
    marching cubes shares them exactly).  A component's label is its smallest vertex index.
  * Selection.  A component's area is the fp64 sum of its triangles' areas 0.5 |(v1 - v0) x (v2 - v0)| in ascending
    triangle index; it is kept iff its area >= min_component * the largest component's area (0 keeps everything).  The
    kept triangles and the vertices they reference keep their original order.
  * Sampling.  Sample i of a seed takes the first triangle whose inclusive cumulative area exceeds u0 * total area, with a
    53-bit uniform u0, and the point (1 - s) v0 + s (1 - r2) v1 + s r2 v2 with s = sqrt(r1): i.i.d. area-uniform samples.
    Each sample depends on (seed, i) and the mesh only, so a cloud is the same however it is split into launches.
Two third-party boundaries are restated rather than pinned (DESIGN.md section 2): the MeshLab step is an explicit crop plus
the area-fraction rule, not a hand selection, and no claim is made about CloudCompare's sampling scheme beyond
area-uniformity.
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


# ------------------------------------------------------------------------------------------------ mesh clean-up and sampling
_BLOCK = 256                  # NERO_MESHPTS_BLOCK / NERO_MESHPTS_CHUNK (include/nero_meshpts.h)
_INT32_MAX = 2 ** 31 - 1


def _check_mesh_shape(v_shape, t_shape, what):
    if len(v_shape) != 2 or v_shape[1] != 3 or len(t_shape) != 2 or t_shape[1] != 3:
        raise ValueError(f'{what} needs verts [V,3] and tris [T,3], got {tuple(v_shape)} and {tuple(t_shape)}')
    if v_shape[0] < 1 or t_shape[0] < 1:
        raise ValueError(f'{what}: the mesh is empty ({v_shape[0]} vertices, {t_shape[0]} triangles)')
    if v_shape[0] > _INT32_MAX or t_shape[0] > _INT32_MAX:
        raise ValueError(f'{what}: {v_shape[0]} vertices / {t_shape[0]} triangles do not fit int32 indices')


def _mesh_cuda(verts, tris, what):
    """(verts float32 [V,3], tris int32 [T,3]) as contiguous CUDA tensors from numpy arrays or tensors.  The shapes, the index
    range and finiteness are checked (on the host for numpy input) before any kernel runs."""
    torch = _torch()
    if torch.is_tensor(verts) or torch.is_tensor(tris):
        v, t = torch.as_tensor(verts).detach(), torch.as_tensor(tris).detach()
        _check_mesh_shape(v.shape, t.shape, what)
        dev = v.device if v.device.type == 'cuda' else t.device if t.device.type == 'cuda' else torch.device('cuda')
        v = v.to(dev, torch.float32).contiguous()
        t = t.to(dev, torch.int64)
        lo, hi = int(t.min()), int(t.max())
        finite = bool(torch.isfinite(v).all())
        t = t.to(torch.int32).contiguous()
    else:
        v, t = np.asarray(verts), np.asarray(tris)
        _check_mesh_shape(v.shape, t.shape, what)
        if not np.issubdtype(t.dtype, np.integer):
            raise ValueError(f'{what}: triangle indices must be integers, got {t.dtype}')
        lo, hi = int(t.min()), int(t.max())
        v = np.ascontiguousarray(v, np.float32)
        finite = bool(np.isfinite(v).all())
    if lo < 0 or hi >= v.shape[0]:
        raise ValueError(f'{what}: triangle index out of range [0, {v.shape[0]}): min {lo}, max {hi}')
    if not finite:
        raise ValueError(f'{what}: vertex coordinates must be finite')
    if not torch.is_tensor(v):
        v = torch.from_numpy(v).cuda()
        t = torch.from_numpy(np.ascontiguousarray(t, np.int32)).cuda()
    _ops().require_cuda(v.device, what)
    return v, t


def _region(sphere, box, min_component):
    """Host copies of the crop arguments (None or float64 arrays), checked."""
    if not 0.0 <= min_component <= 1.0:
        raise ValueError(f'min_component must lie in [0, 1], got {min_component}')
    sph = bx = None
    if sphere is not None:
        sph = np.ascontiguousarray(sphere, np.float64).reshape(-1)
        if sph.shape != (4,) or not np.isfinite(sph).all():
            raise ValueError(f'sphere must be 4 finite numbers (cx, cy, cz, r), got {sphere}')
        if not sph[3] > 0:
            raise ValueError(f'sphere radius must be positive, got {sph[3]}')
    if box is not None:
        bx = np.ascontiguousarray(box, np.float64).reshape(-1)
        if bx.shape != (6,) or not np.isfinite(bx).all():
            raise ValueError(f'box must be 6 finite numbers (x0, y0, z0, x1, y1, z1), got {box}')
        if not (bx[:3] <= bx[3:]).all():
            raise ValueError(f'box needs x0 <= x1, y0 <= y1, z0 <= z1, got {box}')
    return sph, bx


def clean_mesh_cuda(verts, tris, sphere=None, box=None, min_component=0.0):
    """clean_mesh with its intermediate results: (verts, tris, info).  info holds CUDA tensors area [T] (fp64), keep [T]
    (uint8, the crop), label [T] (int32; V for cropped triangles), comp_label [m] (int32, ascending), comp_area [m] (fp64),
    comp_keep [m] (bool), and the ints triangles, components, kept_components, kept_triangles, kept_vertices."""
    torch = _torch()
    ops = _ops()
    sph, bx = _region(sphere, box, min_component)
    v, t = _mesh_cuda(verts, tris, 'clean_mesh')
    V, T = v.shape[0], t.shape[0]
    dev = v.device
    with torch.cuda.device(dev):
        area = torch.empty(T, dtype=torch.float64, device=dev)
        keep = torch.empty(T, dtype=torch.uint8, device=dev)
        ops.K('nero_meshpts_areas', v, V, t, T, sph, bx, area, keep)
        parent = torch.empty(V, dtype=torch.int32, device=dev)
        label = torch.empty(T, dtype=torch.int32, device=dev)
        ops.K('nero_meshpts_components', t, T, keep, V, parent, label, launches=4 + (V - 1).bit_length())
        skeys, order = torch.sort(label, stable=True)    # plumbing: stable, so each component lists its triangles in order
        labs, counts = torch.unique_consecutive(skeys, return_counts=True)
        ends = torch.cumsum(counts, 0)
        if int(labs[-1]) == V:                           # the cropped triangles
            labs, ends = labs[:-1], ends[:-1]
        m = labs.shape[0]
        if m == 0:
            raise ValueError('clean_mesh: no triangle lies inside the crop region')
        comp_area = torch.empty(m, dtype=torch.float64, device=dev)
        root_keep = torch.empty(V, dtype=torch.uint8, device=dev)
        ops.K('nero_meshpts_component_areas', area, order, ends, labs, m, float(min_component), comp_area, root_keep, launches=2)
        nbt, nbv = ops.ceil_div(T, _BLOCK), ops.ceil_div(V, _BLOCK)
        tri_flag = torch.empty(T, dtype=torch.uint8, device=dev)
        vert_flag = torch.empty(V, dtype=torch.uint8, device=dev)
        blk_cnt = torch.empty(nbt + nbv, dtype=torch.int32, device=dev)
        blk_off = torch.empty(nbt + nbv, dtype=torch.int64, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)
        ops.K('nero_meshpts_compact_count', t, T, keep, label, root_keep, V, tri_flag, vert_flag, blk_cnt, blk_off, totals, launches=5)
        nv, nt = totals.tolist()
        remap = torch.empty(V, dtype=torch.int32, device=dev)
        vo = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        to = torch.empty(nt, 3, dtype=torch.int32, device=dev)
        ops.K('nero_meshpts_compact_emit', v, V, t, T, tri_flag, vert_flag, blk_off, nv, nt, remap, vo, to, launches=2)
        comp_keep = root_keep[labs.long()].bool()
    info = dict(area=area, keep=keep, label=label, comp_label=labs, comp_area=comp_area, comp_keep=comp_keep, triangles=T,
                components=m, kept_components=int(comp_keep.sum()), kept_triangles=nt, kept_vertices=nv)
    return vo, to, info


def clean_mesh(verts, tris, sphere=None, box=None, min_component=0.0):
    """Replaces the MeshLab step of the real-data protocol: crop to the sphere (cx, cy, cz, r) and / or the box (x0, y0, z0,
    x1, y1, z1), split the rest into connected components and keep those whose area is at least min_component (in [0, 1])
    times the largest one's.  verts [V,3] / tris [T,3] as numpy arrays or tensors -> (verts CUDA float32 [V',3], tris CUDA
    int32 [T',3]): the kept triangles and the vertices they use, in their original order."""
    v, t, _ = clean_mesh_cuda(verts, tris, sphere, box, min_component)
    return v, t


def sample_surface(verts, tris, n, seed=0, first=0):
    """Replaces CloudCompare's 'sample points on a mesh': n i.i.d. area-uniform points on the surface -> CUDA float64 [n,3].
    Returns samples first .. first + n - 1 of the seed's sequence, so a cloud can be produced in pieces.  Raises ValueError
    for an empty mesh or one without area."""
    torch = _torch()
    ops = _ops()
    if int(n) != n or n < 1:
        raise ValueError(f'sample_surface needs n >= 1 points, got {n}')
    if int(seed) != seed or not 0 <= seed < 2 ** 32:
        raise ValueError(f'seed must be an integer in [0, 2^32), got {seed}')
    if int(first) != first or first < 0:
        raise ValueError(f'first must be a non-negative integer, got {first}')
    v, t = _mesh_cuda(verts, tris, 'sample_surface')
    V, T = v.shape[0], t.shape[0]
    dev = v.device
    with torch.cuda.device(dev):
        area = torch.empty(T, dtype=torch.float64, device=dev)
        ops.K('nero_meshpts_areas', v, V, t, T, None, None, area, None)
        chunk = torch.empty(ops.ceil_div(T, _BLOCK), dtype=torch.float64, device=dev)
        cdf = torch.empty(T, dtype=torch.float64, device=dev)
        ops.K('nero_meshpts_cdf', area, T, chunk, cdf, launches=3)
        total = float(cdf[-1])
        if not (total > 0 and np.isfinite(total)):
            raise ValueError(f'sample_surface: the mesh has no surface area (total {total})')
        out = torch.empty(int(n), 3, dtype=torch.float64, device=dev)
        ops.K('nero_meshpts_sample', v, V, t, T, cdf, int(seed), int(first), int(n), out)
    return out


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


def read_gt_image(root, img_id):
    """get_image: uint8 RGB [h,w,3] of the 8-bit <root>/<id>.png, alpha dropped."""
    import cv2
    path = os.path.join(root, f'{img_id}.png')
    raw = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if raw is None:
        raise FileNotFoundError(path)
    if raw.dtype != np.uint8 or raw.ndim != 3 or raw.shape[2] not in (3, 4):
        raise ValueError(f'{path}: expected an 8-bit RGB or RGBA image, got {raw.dtype} {raw.shape}')
    return np.ascontiguousarray(raw[..., 2::-1])


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
