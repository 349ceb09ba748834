"""numpy float64 oracle of the shape evaluation (nero_b200/evaluate.py, k_eval.cu).

Restates, independently of the kernels:
  * project_clip + rasterize: the reference's nvdiffrast call as rasterize_depth_map uses it (eval_synthetic_shape.py:39-60)
    -- clip-space vertices (x, y, z, w = 1), a scanline rasteriser sampling pixel (x, y) at NDC ((2x+1)/w - 1, (2y+1)/h - 1),
    screen-space barycentrics (with w = 1 perspective correction is the identity), near/far clipping as -1 <= z <= 1, the
    smallest z wins.  It does not cast rays, so its agreement with the ray-cast kernel checks rule 1 of evaluate.py.
  * raycast_depth: brute-force Moeller-Trumbore through the pixel centres with depth sum b z^2 / sum b z, for the CPU check
    that the two formulations agree.
  * depth_to_points: mask_depth_to_pts + pose_apply(pose_inverse(pose)) (utils/base_utils.py:44-52, 562-565, 583-584).
  * voxel_down_sample: Open3D's VoxelDownSample (min bound - voxel/2, floor index, mean summed in input order), output in
    ascending key order.
  * nearest_dist: brute force.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np

NEAR, FAR = 0.5, 100.0
KEY_BITS = 21


def project_clip(verts, pose, K, h, w, near=NEAR, far=FAR):
    """Clip-space vertices [V,4] of rasterize_depth_map: project_points, NDC (2p - size)/size, z = 2(depth-near)/(far-near)-1,
    w = 1."""
    verts = np.asarray(verts, np.float64)
    pose = np.asarray(pose, np.float64)
    K = np.asarray(K, np.float64)
    xc = verts @ pose[:, :3].T + pose[:, 3]
    p = xc @ K.T
    d = p[:, 2]
    out = np.ones((verts.shape[0], 4))
    out[:, 0] = (2 * p[:, 0] / d - w) / w
    out[:, 1] = (2 * p[:, 1] / d - h) / h
    out[:, 2] = 2 * (d - near) / (far - near) - 1
    return out


def rasterize(clip, tris, h, w):
    """nvdiffrast-style output [h,w,4] float64: (b0, b1, z, triangle id + 1), 0 where no triangle covers the pixel centre."""
    clip = np.asarray(clip, np.float64)
    tris = np.asarray(tris, np.int64)
    sx = (clip[:, 0] + 1) * w / 2            # pixel-unit screen coordinates; pixel (x, y) is sampled at (x + 1/2, y + 1/2)
    sy = (clip[:, 1] + 1) * h / 2
    z = clip[:, 2]
    rast = np.zeros((h, w, 4))
    zbuf = np.full((h, w), np.inf)
    for t, (a, b, c) in enumerate(tris):
        xa, xb, xc_ = sx[a], sx[b], sx[c]
        ya, yb, yc = sy[a], sy[b], sy[c]
        area = (xb - xa) * (yc - ya) - (xc_ - xa) * (yb - ya)
        if area == 0 or not np.isfinite(area):
            continue
        x0 = max(int(np.ceil(min(xa, xb, xc_) - 0.5)), 0)
        x1 = min(int(np.floor(max(xa, xb, xc_) - 0.5)), w - 1)
        y0 = max(int(np.ceil(min(ya, yb, yc) - 0.5)), 0)
        y1 = min(int(np.floor(max(ya, yb, yc) - 0.5)), h - 1)
        if x0 > x1 or y0 > y1:
            continue
        px, py = np.meshgrid(np.arange(x0, x1 + 1) + 0.5, np.arange(y0, y1 + 1) + 0.5)
        b0 = ((xb - px) * (yc - py) - (xc_ - px) * (yb - py)) / area
        b1 = ((xc_ - px) * (ya - py) - (xa - px) * (yc - py)) / area
        b2 = 1.0 - b0 - b1
        zz = b0 * z[a] + b1 * z[b] + b2 * z[c]
        sub = zbuf[y0:y1 + 1, x0:x1 + 1]
        win = (b0 >= 0) & (b1 >= 0) & (b2 >= 0) & (zz >= -1) & (zz <= 1) & (zz < sub)
        if not win.any():
            continue
        sub[win] = zz[win]
        r = rast[y0:y1 + 1, x0:x1 + 1]
        r[win] = np.stack([b0[win], b1[win], zz[win], np.full(int(win.sum()), t + 1.0)], -1)
    return rast


def render_depth(verts, tris, pose, K, h, w, near=NEAR, far=FAR):
    """(depth [h,w], mask [h,w]) as rasterize_depth_map returns them, depth 0 where the mask is false."""
    rast = rasterize(project_clip(verts, pose, K, h, w, near, far), tris, h, w)
    mask = rast[..., 3] != 0
    return np.where(mask, (rast[..., 2] + 1) / 2 * (far - near) + near, 0.0), mask


def pixel_rays(pose, K, h, w):
    """World-space origin [3] and directions [h*w,3] (camera z component 1) through the pixel centres (x + 1/2, y + 1/2)."""
    pose = np.asarray(pose, np.float64)
    K = np.asarray(K, np.float64)
    ys, xs = np.mgrid[0:h, 0:w]
    dc = np.stack([(xs.ravel() + 0.5 - K[0, 2]) / K[0, 0], (ys.ravel() + 0.5 - K[1, 2]) / K[1, 1], np.ones(h * w)], -1)
    R, t = pose[:, :3], pose[:, 3]
    return -R.T @ t, dc @ R


def raycast_depth(verts, tris, pose, K, h, w, near=NEAR, far=FAR):
    """Closest hit of the pixel-centre rays (all triangles, both orientations) and depth sum b_i z_i^2 / sum b_i z_i from its
    3-D barycentrics.  Returns (depth [h,w], triangle id [h,w] or -1)."""
    verts = np.asarray(verts, np.float64)
    tris = np.asarray(tris, np.int64)
    pose = np.asarray(pose, np.float64)
    o, d = pixel_rays(pose, K, h, w)
    v0, v1, v2 = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    e1, e2 = v1 - v0, v2 - v0
    zc = verts @ pose[2, :3] + pose[2, 3]
    pv = np.cross(d[:, None, :], e2[None])
    det = np.einsum('tk,ntk->nt', e1, pv)
    ok = np.abs(det) > 1e-300
    inv = 1.0 / np.where(ok, det, 1.0)
    tv = o[None, None, :] - v0[None]
    u = np.einsum('ntk,ntk->nt', tv, pv) * inv
    qv = np.cross(tv, e1[None])
    v = np.einsum('nk,ntk->nt', d, qv) * inv
    t = np.einsum('tk,ntk->nt', e2, qv) * inv
    hit = ok & (u >= 0) & (v >= 0) & (u + v <= 1) & (t > 0)
    t = np.where(hit, t, np.inf)
    best = np.argmin(t, 1)
    n = np.arange(d.shape[0])
    covered = np.isfinite(t[n, best])
    bu, bv = u[n, best], v[n, best]
    z = zc[tris[best]]
    b = np.stack([1 - bu - bv, bu, bv], -1)
    depth = (b * z * z).sum(-1) / (b * z).sum(-1)
    keep = covered & (depth >= near) & (depth <= far)
    return np.where(keep, depth, 0.0).reshape(h, w), np.where(keep, best, -1).reshape(h, w)


def depth_to_points(depth, mask, K, pose):
    """mask_depth_to_pts at integer pixel coordinates, then pose_apply(pose_inverse(pose)): world points [n,3] float64 in
    row-major pixel order."""
    hs, ws = np.nonzero(mask)
    d = np.asarray(depth, np.float64)[hs, ws]
    pts = np.stack([ws * d, hs * d, d], -1) @ np.linalg.inv(np.asarray(K, np.float64)).T
    pose = np.asarray(pose, np.float64)
    R, t = pose[:, :3], pose[:, 3]
    return (pts - t) @ R


def voxel_down_sample(points, voxel):
    """Open3D VoxelDownSample in float64 -> [m,3] voxel means in ascending key order (i << 42 | j << 21 | k)."""
    p = np.asarray(points, np.float64).reshape(-1, 3)
    if p.shape[0] == 0:
        return np.zeros((0, 3))
    lo = p.min(0) - voxel * 0.5
    idx = np.floor((p - lo) / voxel).astype(np.int64)
    if idx.max() >= 1 << KEY_BITS:
        raise ValueError(f'voxel grid of {idx.max(0) + 1} cells exceeds {1 << KEY_BITS} along an axis')
    key = (idx[:, 0] << 2 * KEY_BITS) | (idx[:, 1] << KEY_BITS) | idx[:, 2]
    uniq, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    sums = np.zeros((uniq.shape[0], 3))
    np.add.at(sums, inv.ravel(), p)          # sequential, in input order
    return sums / cnt[:, None]


def nearest_dist(q, t, chunk=2048):
    """Exact nearest distance from each q [n,3] to the set t [m,3], float64."""
    q = np.asarray(q, np.float64)
    t = np.asarray(t, np.float64)
    out = np.empty(q.shape[0])
    for i in range(0, q.shape[0], chunk):
        out[i:i + chunk] = np.sqrt((((q[i:i + chunk, None, :] - t[None]) ** 2).sum(-1)).min(1))
    return out


def chamfer(pts_gt, pts_pr):
    dg, dp = nearest_dist(pts_gt, pts_pr), nearest_dist(pts_pr, pts_gt)
    return (dg.mean() + dp.mean()) / 2, dg, dp

