"""numpy / fp64 restatement of the custom-object preparation kernels of k_objprep.cu (include/nero_objprep.h), in the GPU's
arithmetic order, so the kernels must match it bit for bit; plus a COLMAP model writer and a synthetic scene for the tests.

There is no reference code to pin the kernels against: the reference workflow (custom_object.md) crops the object and fits
the table plane by hand in CloudCompare.  This file states what the kernels compute instead:
  crop        a point is kept iff it lies inside the sphere and / or the box (fp64 tests)
  compaction  the flagged points in their original order
  hypotheses  three kept points per hypothesis from a counter-based hash; unit normal c / |c| of c = e1 x e2, offset -n.p0
  counts      |((nx x + ny y) + nz z) + d| <= tol per plane, counted exactly
  moments     inlier count, sum of d = p - center and of d d^T: per-thread sequential sums over 16 points, a 256-wide
              shared-memory tree, block partials added in block order
  isolation   height over the plane >= above, packed voxel keys, 26-connected voxel components labelled by their smallest
              voxel index, point counts per component, selection by a fraction of the largest, compaction
Elementwise numpy fp64 arithmetic rounds every operation, as the kernels' __d*_rn intrinsics do.
"""
import os
import struct

import numpy as np

CHUNK = 4096         # NERO_OBJPREP_CHUNK: points per block of the refit sums
BLOCK = 256          # threads per block (and compaction block)
NOKEY = np.int64(0x7fffffffffffffff)
VOX_MAX = 1 << 21


# ------------------------------------------------------------------------------------------------ kernels
def _mix(x):
    x = x ^ (x >> np.uint32(16))
    x = x * np.uint32(0x85ebca6b)
    x = x ^ (x >> np.uint32(13))
    x = x * np.uint32(0xc2b2ae35)
    return x ^ (x >> np.uint32(16))


def bits(seed, k, d):
    """uint32 hash(seed, k, d) = mix(mix(mix(seed 0x9e3779b9 + 0x7f4a7c15) ^ k) ^ d) of hypotheses k (array)."""
    k = np.asarray(k, np.uint32)
    with np.errstate(over='ignore'):
        h = _mix(np.full(k.shape, np.uint32(seed), np.uint32) * np.uint32(0x9e3779b9) + np.uint32(0x7f4a7c15))
        return _mix(_mix(h ^ k) ^ np.uint32(d))


def crop(pts, sphere=None, box=None):
    """bool [n]: inside the sphere (cx, cy, cz, r) and / or the box (x0, y0, z0, x1, y1, z1)."""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    inside = np.ones(p.shape[0], bool)
    if sphere is not None:
        c = np.asarray(sphere, np.float64)
        d = p - c[:3]
        inside &= (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= c[3] * c[3]
    if box is not None:
        b = np.asarray(box, np.float64)
        inside &= ((p >= b[:3]) & (p <= b[3:])).all(1)
    return inside


def _sq3(x, y, z):
    return (x * x + y * y) + z * z


def hypotheses(kept, H, seed):
    """(planes [H,4], sample [H,3] int32, valid [H] bool) of the kept points [n,3]."""
    p = np.asarray(kept, np.float64).reshape(-1, 3)
    n = p.shape[0]
    k = np.arange(H, dtype=np.uint32)
    sample = np.stack([((bits(seed, k, d).astype(np.uint64) * np.uint64(n)) >> np.uint64(32)).astype(np.int64) for d in range(3)], 1)
    p0, p1, p2 = p[sample[:, 0]], p[sample[:, 1]], p[sample[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    c2 = _sq3(cx, cy, cz)
    valid = c2 > 1e-20 * (_sq3(e1[:, 0], e1[:, 1], e1[:, 2]) * _sq3(e2[:, 0], e2[:, 1], e2[:, 2]))
    with np.errstate(invalid='ignore', divide='ignore'):
        nrm = np.sqrt(c2)
        nx, ny, nz = cx / nrm, cy / nrm, cz / nrm
        d = -((nx * p0[:, 0] + ny * p0[:, 1]) + nz * p0[:, 2])
    planes = np.stack([nx, ny, nz, d], 1)
    planes[~valid] = np.nan
    return planes, sample.astype(np.int32), valid


def residual(pts, plane):
    """((nx x + ny y) + nz z) + d for every point."""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    return ((plane[0] * p[:, 0] + plane[1] * p[:, 1]) + plane[2] * p[:, 2]) + plane[3]


def counts(kept, planes, tol, batch=64):
    """int64 [H]: points with |r| <= tol per plane (0 for a NaN plane)."""
    p = np.asarray(kept, np.float64).reshape(-1, 3)
    out = np.zeros(planes.shape[0], np.int64)
    for k0 in range(0, planes.shape[0], batch):
        pl = planes[k0:k0 + batch]
        r = ((pl[:, 0:1] * p[None, :, 0] + pl[:, 1:2] * p[None, :, 1]) + pl[:, 2:3] * p[None, :, 2]) + pl[:, 3:4]
        with np.errstate(invalid='ignore'):
            out[k0:k0 + batch] = (np.abs(r) <= tol).sum(1)
    return out


def moments(kept, plane, tol, center):
    """(partial [ceil(n/4096), 10], out [10]) as nero_objprep_moments sums them."""
    p = np.asarray(kept, np.float64).reshape(-1, 3)
    n = p.shape[0]
    nblk = (n + CHUNK - 1) // CHUNK
    q = np.zeros((nblk * CHUNK, 3))
    q[:n] = p
    inl = np.zeros(nblk * CHUNK, bool)
    inl[:n] = np.abs(residual(p, plane)) <= tol
    c = np.asarray(center, np.float64)
    d = q - c
    terms = [np.ones(q.shape[0]), d[:, 0], d[:, 1], d[:, 2], d[:, 0] * d[:, 0], d[:, 0] * d[:, 1], d[:, 0] * d[:, 2], d[:, 1] * d[:, 1],
             d[:, 1] * d[:, 2], d[:, 2] * d[:, 2]]
    partial = np.empty((nblk, 10))
    for m, t in enumerate(terms):
        t = np.where(inl, t, 0.0).reshape(nblk, CHUNK // BLOCK, BLOCK)    # [block, j, thread]
        s = np.zeros((nblk, BLOCK))
        for j in range(CHUNK // BLOCK):
            s = s + t[:, j]
        w = BLOCK // 2
        while w > 0:
            s = np.concatenate([s[:, :w] + s[:, w:2 * w], s[:, w:]], 1)
            w //= 2
        partial[:, m] = s[:, 0]
    out = partial[0].copy()
    for b in range(1, nblk):
        out = out + partial[b]
    return partial, out


def voxel_keys(pts, origin, voxel):
    """int64 [n] packed keys (a << 42) | (b << 21) | c, a = floor((x - origin_x) / voxel)."""
    p = np.asarray(pts, np.float64).reshape(-1, 3)
    a = np.floor((p - np.asarray(origin, np.float64)) / voxel).astype(np.int64)
    return (a[:, 0] << 42) | (a[:, 1] << 21) | a[:, 2]


def above(pts, keep, plane, height, origin, voxel):
    """(flag [n] bool, keys [n] int64; NOKEY where not flagged)."""
    flag = np.asarray(keep, bool) & (residual(pts, plane) >= height)
    keys = np.full(flag.shape[0], NOKEY, np.int64)
    keys[flag] = voxel_keys(np.asarray(pts, np.float64).reshape(-1, 3)[flag], origin, voxel)
    return flag, keys


def voxel_components(ukeys):
    """int64 [m]: 26-connected components of the occupied voxels (ascending keys), labelled by their smallest index."""
    u = np.asarray(ukeys, np.int64)
    m = u.shape[0]
    a, b, c = u >> 42, (u >> 21) & (VOX_MAX - 1), u & (VOX_MAX - 1)
    ea, eb = [], []
    for da in (-1, 0, 1):
        for db in (-1, 0, 1):
            for dc in (-1, 0, 1):
                if (da, db, dc) <= (0, 0, 0):
                    continue
                na, nb, nc = a + da, b + db, c + dc
                ok = (na >= 0) & (na < VOX_MAX) & (nb >= 0) & (nb < VOX_MAX) & (nc >= 0) & (nc < VOX_MAX)
                nk = (na << 42) | (nb << 21) | nc
                j = np.minimum(np.searchsorted(u, nk), m - 1)
                hit = ok & (u[j] == nk)
                ea.append(np.nonzero(hit)[0])
                eb.append(j[hit])
    ea, eb = np.concatenate(ea), np.concatenate(eb)
    parent = np.arange(m, dtype=np.int64)
    while True:
        ra, rb = parent[ea], parent[eb]
        lo, hi = np.minimum(ra, rb), np.maximum(ra, rb)
        mk = lo != hi
        if not mk.any():
            break
        np.minimum.at(parent, hi[mk], lo[mk])
        while True:
            g = parent[parent]
            if (g == parent).all():
                break
            parent = g
    return parent


def component_select(label, vcount, frac):
    """(comp_count [m] int64 indexed by root label, voxel_keep [m] bool)."""
    m = label.shape[0]
    cc = np.zeros(m, np.int64)
    np.add.at(cc, label, np.asarray(vcount, np.int64))
    return cc, cc[label].astype(np.float64) >= frac * float(cc.max())


def isolate(pts, keep, plane, height, origin, voxel, frac):
    """Everything isolate_object computes: dict of flag, keys, ukeys, vcount, label, comp_count, voxel_keep, point_keep, index."""
    flag, keys = above(pts, keep, plane, height, origin, voxel)
    ukeys, vcount = np.unique(keys[flag], return_counts=True)
    label = voxel_components(ukeys)
    cc, vk = component_select(label, vcount, frac)
    pk = np.zeros(flag.shape[0], bool)
    pk[flag] = vk[np.searchsorted(ukeys, keys[flag])]
    return dict(flag=flag, keys=keys, ukeys=ukeys, vcount=vcount, label=label, comp_count=cc, voxel_keep=vk, point_keep=pk,
                index=np.nonzero(pk)[0])


# ------------------------------------------------------------------------------------------------ COLMAP writer
# the published model format (colmap.github.io/format.html): model name -> (model id, number of parameters)
CAMERA_MODELS = {'SIMPLE_PINHOLE': (0, 3), 'PINHOLE': (1, 4), 'SIMPLE_RADIAL': (2, 4), 'RADIAL': (3, 5), 'OPENCV': (4, 8)}


def rotmat2qvec(R):
    """A unit quaternion (w, x, y, z), w >= 0, of the rotation matrix R."""
    R = np.asarray(R, np.float64)
    w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    x = np.sqrt(max(0.0, 1.0 + R[0, 0] - R[1, 1] - R[2, 2])) / 2
    y = np.sqrt(max(0.0, 1.0 - R[0, 0] + R[1, 1] - R[2, 2])) / 2
    z = np.sqrt(max(0.0, 1.0 - R[0, 0] - R[1, 1] + R[2, 2])) / 2
    x = np.copysign(x, R[2, 1] - R[1, 2])
    y = np.copysign(y, R[0, 2] - R[2, 0])
    z = np.copysign(z, R[1, 0] - R[0, 1])
    q = np.asarray([w, x, y, z])
    return q / np.linalg.norm(q)


def write_colmap_model(path, cameras, images, points, fmt):
    """cameras: {id: (model, width, height, params)}; images: {id: (qvec, tvec, camera_id, name, xys [k,2], point3D_ids [k])};
    points: {id: (xyz, rgb, error, image_ids, point2D_idxs)}.  fmt 'bin' or 'txt'; writes cameras, images and points3D."""
    os.makedirs(path, exist_ok=True)
    if fmt == 'bin':
        with open(os.path.join(path, 'cameras.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(cameras)))
            for cid, (model, w, h, params) in cameras.items():
                mid, npar = CAMERA_MODELS[model]
                assert len(params) == npar
                f.write(struct.pack('<iiQQ', cid, mid, w, h) + struct.pack(f'<{npar}d', *params))
        with open(os.path.join(path, 'images.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(images)))
            for iid, (q, t, cid, name, xys, p3d) in images.items():
                f.write(struct.pack('<i4d3di', iid, *q, *t, cid) + name.encode() + b'\x00')
                f.write(struct.pack('<Q', len(p3d)))
                for (x, y), pid in zip(xys, p3d):
                    f.write(struct.pack('<ddq', x, y, pid))
        with open(os.path.join(path, 'points3D.bin'), 'wb') as f:
            f.write(struct.pack('<Q', len(points)))
            for pid, (xyz, rgb, err, iids, p2d) in points.items():
                f.write(struct.pack('<Q3d3Bd', pid, *xyz, *rgb, err) + struct.pack('<Q', len(iids)))
                for a, b in zip(iids, p2d):
                    f.write(struct.pack('<ii', a, b))
    else:
        r = repr
        with open(os.path.join(path, 'cameras.txt'), 'w') as f:
            f.write('# Camera list with one line of data per camera:\n#   CAMERA_ID, MODEL, WIDTH, HEIGHT, PARAMS[]\n')
            f.write(f'# Number of cameras: {len(cameras)}\n')
            for cid, (model, w, h, params) in cameras.items():
                f.write(' '.join([str(cid), model, str(w), str(h)] + [r(float(p)) for p in params]) + '\n')
        with open(os.path.join(path, 'images.txt'), 'w') as f:
            f.write('# Image list with two lines of data per image:\n#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME\n'
                    '#   POINTS2D[] as (X, Y, POINT3D_ID)\n')
            for iid, (q, t, cid, name, xys, p3d) in images.items():
                f.write(' '.join([str(iid)] + [r(float(v)) for v in list(q) + list(t)] + [str(cid), name]) + '\n')
                f.write(' '.join(f'{r(float(x))} {r(float(y))} {int(pid)}' for (x, y), pid in zip(xys, p3d)) + '\n')
        with open(os.path.join(path, 'points3D.txt'), 'w') as f:
            f.write('# 3D point list with one line of data per point:\n'
                    '#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[] as (IMAGE_ID, POINT2D_IDX)\n')
            for pid, (xyz, rgb, err, iids, p2d) in points.items():
                f.write(' '.join([str(pid)] + [r(float(v)) for v in xyz] + [str(int(c)) for c in rgb] + [r(float(err))] +
                                 [f'{a} {b}' for a, b in zip(iids, p2d)]) + '\n')


# ------------------------------------------------------------------------------------------------ synthetic scene
def look_at(c, target, up):
    """COLMAP pose [3,4] (world -> camera, x right, y down, z forward) of a camera at c looking at target."""
    c, target = np.asarray(c, np.float64), np.asarray(target, np.float64)
    z = target - c
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z], 0)
    return np.concatenate([R, (-R @ c)[:, None]], 1)


def scene(n_table=120000, n_obj=80000, outlier_frac=0.1, n_cams=40, seed=0, sigma=0.0005):
    """A table plane tilted and offset in space, a box (0.3 x 0.3 x 1.0) standing on it with a sphere (r 0.3) on top, and
    outlier_frac of the cloud as uniform outliers in a 4 x 4 x 4 cube; 40 cameras on a hemisphere of radius 3 around the
    object looking at its centre.  -> dict(points [n,3] (shuffled), label [n] (0 table, 1 object, 2 outlier), up [3],
    origin [3] (table point under the object), center [3], poses [n_cams,3,4])."""
    rng = np.random.RandomState(seed)
    up = np.asarray([0.21, -0.33, 0.92])
    up /= np.linalg.norm(up)
    e1 = np.cross(up, [1.0, 0.0, 0.0])
    e1 /= np.linalg.norm(e1)
    e2 = np.cross(up, e1)
    o = np.asarray([1.3, -0.7, 2.1])
    frame = lambda a, b, h: o + a[:, None] * e1 + b[:, None] * e2 + h[:, None] * up
    # table: a disc of radius 1.8 around the object
    r, t = 1.8 * np.sqrt(rng.rand(n_table)), 2 * np.pi * rng.rand(n_table)
    table = frame(r * np.cos(t), r * np.sin(t), sigma * rng.randn(n_table))
    # object surface, area-uniform: 4 box sides + box top + sphere
    areas = np.asarray([0.3, 0.3, 0.3, 0.3, 0.09, 4 * np.pi * 0.09])
    k = rng.choice(6, n_obj, p=areas / areas.sum())
    u, w, v = 0.3 * (rng.rand(n_obj) - 0.5), 0.3 * (rng.rand(n_obj) - 0.5), rng.rand(n_obj)
    side = np.asarray([0.15, -0.15, 0.15, -0.15, 0.0, 0.0])[k]
    a = np.where(k < 2, side, u)                       # sides 0, 1 at a = +-0.15; sides 2, 3 at b = +-0.15; top at h = 1
    b = np.where((k == 2) | (k == 3), side, w)
    h = np.where(k < 4, v, 1.0)
    s = rng.randn(n_obj, 3)
    s /= np.linalg.norm(s, axis=1, keepdims=True)
    a = np.where(k == 5, 0.3 * s[:, 0], a)
    b = np.where(k == 5, 0.3 * s[:, 1], b)
    h = np.where(k == 5, 1.3 + 0.3 * s[:, 2], h)
    obj = frame(a, b, h) + sigma * rng.randn(n_obj, 3)
    n_out = int(round(outlier_frac * (n_table + n_obj) / (1 - outlier_frac)))
    c3 = rng.rand(n_out, 3) * 4 - 2
    outl = frame(c3[:, 0], c3[:, 1], c3[:, 2] + 1.0)
    pts = np.concatenate([table, obj, outl], 0)
    lab = np.concatenate([np.zeros(n_table, np.int64), np.ones(n_obj, np.int64), np.full(n_out, 2, np.int64)])
    perm = rng.permutation(pts.shape[0])
    center = o + 0.8 * up
    poses = []
    for i in range(n_cams):
        az, el = 2 * np.pi * i / n_cams + 0.1 * rng.rand(), np.radians(15 + 45 * rng.rand())
        d = np.cos(el) * (np.cos(az) * e1 + np.sin(az) * e2) + np.sin(el) * up
        poses.append(look_at(center + 3.0 * d, center, -up))
    return dict(points=pts[perm], label=lab[perm], up=up, origin=o, center=center, poses=np.stack(poses))


def scene_model(sc, width=640, height=480):
    """A COLMAP model of the scene's cameras with all three camera models the custom workflow accepts, and a few hundred
    sparse points -> (cameras, images, points) for write_colmap_model."""
    cams = {1: ('PINHOLE', width, height, [500.0, 510.0, width / 2, height / 2]),
            2: ('SIMPLE_RADIAL', width, height, [480.0, width / 2 + 3, height / 2 - 2, 0.01]),
            3: ('SIMPLE_PINHOLE', width, height, [520.0, width / 2, height / 2])}
    images = {}
    for i, P in enumerate(sc['poses']):
        iid = 100 - 2 * i                      # ids descend while names ascend
        images[iid] = (rotmat2qvec(P[:, :3]), P[:, 3], 1 + i % 3, f'img_{i:03d}.jpg', np.zeros((2, 2)), np.asarray([-1, 7]))
    rng = np.random.RandomState(1)
    sel = rng.choice(sc['points'].shape[0], 300, replace=False)
    points = {int(7 + 3 * j): (sc['points'][s], rng.randint(0, 256, 3), 0.5 + rng.rand(), [100, 98], [1, 0]) for j, s in enumerate(sel)}
    return cams, images, points
