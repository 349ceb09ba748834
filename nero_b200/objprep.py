"""Custom-object preparation on the GPU: the files CustomDatabase reads, from a COLMAP reconstruction, without CloudCompare.

Reference being replaced (paths relative to the reference repository):
  custom_object.md, steps 4-5      crop the object out of COLMAP's fused cloud by hand, fit a plane to the table (its normal
                                   is Z+), pick a point for X+, type both vectors into meta_info.txt
  dataset/database.py:293-323      CustomDatabase._parse_colmap: read_model(<root>/colmap/sparse/0), pose [R | t] from the
                                   image's qvec / tvec, K of SIMPLE_RADIAL (distortion ignored), SIMPLE_PINHOLE, PINHOLE
  dataset/database.py:331-368      _compute_rotation and _normalize: bounding-box centre and largest radius of
                                   object_point_cloud.ply, up and forward from rows 0 and 1 of meta_info.txt
COLMAP itself stays external: run_colmap.py only runs the COLMAP binary.

The protocol (k_objprep.cu, include/nero_objprep.h):
  * Scale.  COLMAP's units are arbitrary, so every default is a fraction of D, the median distance from the camera centres
    c = -R^T t to the object centre, the fp64 least-squares point closest to all optical axes (the third rows of R).  The
    default crop is the sphere of radius CROP_FRAC D around the object centre; tol = TOL_FRAC D, above = ABOVE_TOLS tol,
    voxel = VOXEL_FRAC D.
  * Crop.  A point is kept iff it lies inside the sphere and / or the box (fp64, inclusive).
  * Support plane.  RANSAC over the kept points: hypothesis k draws three of them from a counter-based hash of (seed, k),
    its plane is the unit normal of (p1 - p0) x (p2 - p0) through p0, and hypotheses whose three points are collinear or
    repeated are invalid.  Each plane counts the kept points with |n . p + d| <= tol; the best is the largest count, ties
    to the smallest k.  Two refit rounds follow: the least-squares plane (smallest eigenvector of the scatter about the
    centroid) of the previous plane's inliers.  The centroid and scatter are fp64 sums with a fixed order (per-block
    partials in block order), so the fit is the same on every run; the 3 x 3 eigen-solve runs on the host.
  * Up.  The normal's sign puts the majority of the camera centres on the positive side.
  * Object.  Points inside the crop and at least `above` over the plane are voxelised; 26-connected components of the
    occupied voxels are kept when their point count is >= min_component times the largest one's (1 keeps the largest);
    the kept points keep their original order.
  * Forward.  The direction from the object centre toward a camera centre (by default the first image in name order),
    projected onto the plane.
"""
import os
import struct

import numpy as np

CROP_FRAC = 0.5       # default crop radius / D
TOL_FRAC = 0.002      # default inlier tolerance / D
ABOVE_TOLS = 2.0      # default height over the plane, in tolerances
VOXEL_FRAC = 0.01     # default voxel size / D
HYPOTHESES = 1024
_BLOCK = 256          # NERO_OBJPREP_BLOCK (include/nero_objprep.h)
_CHUNK = 4096         # NERO_OBJPREP_CHUNK
_MOM = 10             # NERO_OBJPREP_MOMENTS
_KEY_LIMIT = 1 << 21  # voxel index bits per axis
_NOKEY = 0x7fffffffffffffff
_INT32_MAX = 2 ** 31 - 1


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ COLMAP model
# the published model format: id -> (name, number of parameters)
CAMERA_MODELS = {0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5), 4: ('OPENCV', 8),
                 5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5), 8: ('SIMPLE_RADIAL_FISHEYE', 4),
                 9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12), 11: ('RAD_TAN_THIN_PRISM_FISHEYE', 16)}


def qvec2rotmat(q):
    """Rotation of the unit quaternion (w, x, y, z), COLMAP's convention (world -> camera)."""
    w, x, y, z = (float(v) for v in q)
    return np.asarray([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                       [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                       [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def _intrinsics(model, params):
    """K float32 [3,3] as CustomDatabase._parse_colmap builds it; NotImplementedError for the models it refuses."""
    if model in ('SIMPLE_RADIAL', 'SIMPLE_PINHOLE'):
        f, cx, cy = params[:3]
        return np.asarray([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float32)
    if model == 'PINHOLE':
        fx, fy, cx, cy = params
        return np.asarray([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
    raise NotImplementedError(f'camera model {model}: the custom-object workflow accepts SIMPLE_RADIAL, SIMPLE_PINHOLE and PINHOLE')


def _read(f, fmt):
    n = struct.calcsize(fmt)
    b = f.read(n)
    if len(b) != n:
        raise ValueError(f'{f.name}: truncated COLMAP file')
    return struct.unpack(fmt, b)


def _read_bin(path, tracks=None):
    cameras, images, pts = {}, {}, []
    with open(os.path.join(path, 'cameras.bin'), 'rb') as f:
        for _ in range(_read(f, '<Q')[0]):
            cid, mid, w, h = _read(f, '<iiQQ')
            if mid not in CAMERA_MODELS:
                raise ValueError(f'{path}: unknown camera model id {mid}')
            name, npar = CAMERA_MODELS[mid]
            cameras[cid] = (name, w, h, _read(f, f'<{npar}d'))
    with open(os.path.join(path, 'images.bin'), 'rb') as f:
        for _ in range(_read(f, '<Q')[0]):
            iid, qw, qx, qy, qz, tx, ty, tz, cid = _read(f, '<i4d3di')
            name = bytearray()
            while True:
                c = f.read(1)
                if c in (b'\x00', b''):
                    break
                name += c
            f.seek(24 * _read(f, '<Q')[0], 1)                     # POINTS2D[] as (x, y double, point3D_id int64)
            images[iid] = (name.decode('utf-8'), (qw, qx, qy, qz), (tx, ty, tz), cid)
    with open(os.path.join(path, 'points3D.bin'), 'rb') as f:
        for _ in range(_read(f, '<Q')[0]):
            rec = _read(f, '<Q3d3BdQ')
            pts.append(rec[1:4])
            if tracks is None:
                f.seek(8 * rec[-1], 1)                             # TRACK[] as (image_id, point2D_idx int32)
            else:
                tracks.append(np.asarray(_read(f, f'<{2 * rec[-1]}i')[0::2], np.int64))
    return cameras, images, pts


def _data_lines(path):
    with open(path) as f:
        return [ln.rstrip('\r\n') for ln in f if not ln.startswith('#')]


def _read_txt(path, tracks=None):
    cameras, images, pts = {}, {}, []
    for ln in _data_lines(os.path.join(path, 'cameras.txt')):
        e = ln.split()
        if e:
            cameras[int(e[0])] = (e[1], int(e[2]), int(e[3]), tuple(float(v) for v in e[4:]))
    lines = _data_lines(os.path.join(path, 'images.txt'))
    i = 0
    while i < len(lines):
        e = lines[i].split()
        if not e:
            i += 1
            continue
        images[int(e[0])] = (' '.join(e[9:]), tuple(float(v) for v in e[1:5]), tuple(float(v) for v in e[5:8]), int(e[8]))
        i += 2                                                     # the POINTS2D line follows, possibly empty
    for ln in _data_lines(os.path.join(path, 'points3D.txt')):
        e = ln.split()
        if e:
            pts.append(tuple(float(v) for v in e[1:4]))
            if tracks is not None:                                 # TRACK[] as (IMAGE_ID, POINT2D_IDX) after ERROR
                tracks.append(np.asarray([int(v) for v in e[8::2]], np.int64))
    return cameras, images, pts


def read_colmap_model(path, tracks=False):
    """COLMAP sparse model in `path` (cameras, images, points3D as .bin, else .txt) -> (views, points), or with
    tracks=True (views, points, tracks).

    views = {image_id: (name, pose float32 [3,4] = [R | t] world -> camera, K float32 [3,3])} in file order, as
    CustomDatabase._parse_colmap builds them; points = the sparse points float64 [P,3] in file order; tracks = one int64
    array per point of the image ids of its track, in file order.  An image whose camera model is not SIMPLE_RADIAL
    (distortion ignored), SIMPLE_PINHOLE or PINHOLE raises NotImplementedError."""
    trk = [] if tracks else None
    if all(os.path.isfile(os.path.join(path, f'{n}.bin')) for n in ('cameras', 'images', 'points3D')):
        cameras, images, pts = _read_bin(path, trk)
    elif all(os.path.isfile(os.path.join(path, f'{n}.txt')) for n in ('cameras', 'images', 'points3D')):
        cameras, images, pts = _read_txt(path, trk)
    else:
        raise FileNotFoundError(f'{path}: no COLMAP model (cameras, images and points3D as .bin or .txt)')
    views = {}
    for iid, (name, q, t, cid) in images.items():
        if cid not in cameras:
            raise ValueError(f'{path}: image {iid} uses camera {cid}, which the model does not define')
        pose = np.concatenate([qvec2rotmat(q), np.asarray(t, np.float64)[:, None]], 1).astype(np.float32)
        views[iid] = (name, pose, _intrinsics(cameras[cid][0], cameras[cid][3]))
    if tracks:
        return views, np.asarray(pts, np.float64).reshape(-1, 3), trk
    return views, np.asarray(pts, np.float64).reshape(-1, 3)


# ------------------------------------------------------------------------------------------------ cameras and scale
def camera_centers(views):
    """(names [n] in name order, centres fp64 [n,3], optical axes fp64 [n,3]) of the views, from their float32 poses."""
    items = sorted(views.values(), key=lambda v: v[0])
    R = np.stack([v[1][:, :3] for v in items]).astype(np.float64)
    t = np.stack([v[1][:, 3] for v in items]).astype(np.float64)
    return [v[0] for v in items], -np.einsum('nji,nj->ni', R, t), R[:, 2]


def object_center(centers, axes):
    """The fp64 least-squares point closest to all optical axes: solves sum (I - a a^T) x = sum (I - a a^T) c."""
    a = np.asarray(axes, np.float64) / np.linalg.norm(axes, axis=1, keepdims=True)
    P = np.eye(3)[None] - a[:, :, None] * a[:, None, :]
    A, b = P.sum(0), np.einsum('nij,nj->i', P, centers)
    if np.linalg.eigvalsh(A)[0] <= 1e-6 * a.shape[0]:
        raise ValueError('the optical axes are (nearly) parallel: they do not define an object centre')
    return np.linalg.solve(A, b)


def scene_scale(views):
    """(object centre [3], D = median camera-to-centre distance, names in name order, camera centres [n,3])."""
    names, c, ax = camera_centers(views)
    o = object_center(c, ax)
    return o, float(np.median(np.linalg.norm(c - o, axis=1))), names, c


# ------------------------------------------------------------------------------------------------ GPU steps
def _cloud(points, what):
    torch = _torch()
    if torch.is_tensor(points):
        p = points.detach()
        if p.device.type != 'cuda':
            p = p.cuda()
        p = p.to(torch.float64)
    else:
        p = torch.from_numpy(np.ascontiguousarray(points, np.float64)).cuda()
    if p.dim() != 2 or p.shape[1] != 3:
        raise ValueError(f'{what} needs points [N,3], got {tuple(p.shape)}')
    if p.shape[0] < 3:
        raise ValueError(f'{what} needs at least 3 points, got {p.shape[0]}')
    if p.shape[0] > _INT32_MAX:
        raise ValueError(f'{what}: {p.shape[0]} points do not fit int32 indices')
    if not bool(torch.isfinite(p).all()):
        raise ValueError(f'{what}: point coordinates must be finite')
    _ops().require_cuda(p.device, what)
    return p.contiguous()


def _region(sphere, box):
    sph = bx = None
    if sphere is not None:
        sph = np.ascontiguousarray(sphere, np.float64).reshape(-1)
        if sph.shape != (4,) or not np.isfinite(sph).all() or not sph[3] > 0:
            raise ValueError(f'sphere must be 4 finite numbers (cx, cy, cz, r > 0), got {sphere}')
    if box is not None:
        bx = np.ascontiguousarray(box, np.float64).reshape(-1)
        if bx.shape != (6,) or not np.isfinite(bx).all() or not (bx[:3] <= bx[3:]).all():
            raise ValueError(f'box must be 6 finite numbers (x0, y0, z0, x1, y1, z1) with x0 <= x1, ..., got {box}')
    return sph, bx


def _compact(p, flag, with_points):
    """(indices int32 [m], points [m,3] or None) of the flagged points in their original order."""
    torch = _torch()
    ops = _ops()
    n = p.shape[0]
    nb = ops.ceil_div(n, _BLOCK)
    blk_cnt = torch.empty(nb, dtype=torch.int32, device=p.device)
    blk_off = torch.empty(nb, dtype=torch.int64, device=p.device)
    total = torch.empty(1, dtype=torch.int64, device=p.device)
    ops.K('nero_objprep_compact_count', flag, n, blk_cnt, blk_off, total, launches=2)
    m = int(total)
    idx = torch.empty(m, dtype=torch.int32, device=p.device)
    out = torch.empty(m, 3, dtype=torch.float64, device=p.device) if with_points else None
    ops.K('nero_objprep_compact_emit', p, flag, n, blk_off, m, idx, out)
    return idx, out


def crop_points(points, sphere=None, box=None):
    """(keep uint8 [N] CUDA, kept indices int32, kept points fp64 [m,3]) of the crop."""
    torch = _torch()
    sph, bx = _region(sphere, box)
    p = _cloud(points, 'crop_points')
    keep = torch.empty(p.shape[0], dtype=torch.uint8, device=p.device)
    _ops().K('nero_objprep_crop', p, p.shape[0], sph, bx, keep)
    idx, kept = _compact(p, keep, True)
    return keep, idx, kept


def _moments(kept, plane, tol, center):
    torch = _torch()
    n = kept.shape[0]
    partial = torch.empty(_ops().ceil_div(n, _CHUNK), _MOM, dtype=torch.float64, device=kept.device)
    out = torch.empty(_MOM, dtype=torch.float64, device=kept.device)
    _ops().K('nero_objprep_moments', kept, n, np.ascontiguousarray(plane, np.float64), float(tol), np.ascontiguousarray(center, np.float64),
             partial, out, launches=2)
    return partial, out.cpu().numpy()


def refit(kept, plane, tol):
    """One refit round: the least-squares plane of plane's inliers -> (plane [4], centroid [3], scatter [3,3], inliers).
    The normal keeps the side of the given one."""
    _, s = _moments(kept, plane, tol, np.zeros(3))
    cnt = int(s[0])
    if cnt < 3:
        raise ValueError(f'refit: only {cnt} points lie within tol = {tol} of the plane')
    centroid = s[1:4] / s[0]
    _, m = _moments(kept, plane, tol, centroid)
    S = np.asarray([[m[4], m[5], m[6]], [m[5], m[7], m[8]], [m[6], m[8], m[9]]])
    n = np.linalg.eigh(S)[1][:, 0]
    n = n / np.linalg.norm(n)
    if n @ np.asarray(plane[:3]) < 0:
        n = -n
    return np.concatenate([n, [-(n @ centroid)]]), centroid, S, cnt


def fit_support_plane(points, tol, sphere=None, box=None, hypotheses=HYPOTHESES, seed=0, centers=None, rounds=2):
    """RANSAC support plane of the cropped cloud (numpy array or CUDA tensor [N,3]) -> (plane fp64 [4] = (n, d) with a unit
    normal, info).  centers (optional, [n,3]): camera centres; the normal is turned toward the side holding most of them.

    info holds CUDA tensors keep [N] (uint8 crop), kept_index [m] (int32), planes [H,4], sample [H,3] (int32), valid [H]
    (uint8), counts [H] (int64); and on the host best (int), best_plane [4], refits (one (plane, centroid, scatter,
    inliers) per round), inliers (of the final plane), kept (m).  Raises ValueError for fewer than 3 points, a crop that
    keeps fewer than 3, or no valid hypothesis."""
    torch = _torch()
    ops = _ops()
    if not (np.isfinite(tol) and tol > 0):
        raise ValueError(f'tol must be positive, got {tol}')
    if int(hypotheses) != hypotheses or not 1 <= hypotheses <= _INT32_MAX:
        raise ValueError(f'hypotheses must be a positive integer, got {hypotheses}')
    if int(seed) != seed or not 0 <= seed < 2 ** 32:
        raise ValueError(f'seed must be an integer in [0, 2^32), got {seed}')
    keep, idx, kept = crop_points(points, sphere, box)
    m = kept.shape[0]
    if m < 3:
        raise ValueError(f'fit_support_plane: the crop keeps {m} points, at least 3 are needed')
    H = int(hypotheses)
    dev = kept.device
    with torch.cuda.device(dev):
        planes = torch.empty(H, 4, dtype=torch.float64, device=dev)
        sample = torch.empty(H, 3, dtype=torch.int32, device=dev)
        valid = torch.empty(H, dtype=torch.uint8, device=dev)
        ops.K('nero_objprep_hypotheses', kept, m, H, int(seed), planes, sample, valid)
        counts = torch.empty(H, dtype=torch.int64, device=dev)
        ops.K('nero_objprep_counts', kept, m, planes, H, float(tol), counts)
        c = counts.cpu().numpy()
        best = int(np.argmax(c))                                # the first maximum: ties go to the smallest k
        if not bool(valid.any()) or c[best] < 3:
            raise ValueError('fit_support_plane: no hypothesis has 3 inliers (are the kept points collinear or repeated?)')
        plane = planes[best].cpu().numpy()
        refits = []
        for _ in range(rounds):
            r = refit(kept, plane, tol)
            refits.append(r)
            plane = r[0]
        inliers = int(_moments(kept, plane, tol, np.zeros(3))[1][0])
    if centers is not None:
        r = np.asarray(centers, np.float64).reshape(-1, 3) @ plane[:3] + plane[3]
        if (r < 0).sum() > (r > 0).sum():
            plane = -plane
    info = dict(keep=keep, kept_index=idx, planes=planes, sample=sample, valid=valid, counts=counts, best=best,
                best_plane=planes[best].cpu().numpy(), refits=refits, inliers=inliers, kept=m)
    return plane, info


def isolate_object(points, plane, above, voxel, sphere=None, box=None, min_component=1.0):
    """The object: points inside the crop and at least `above` over the plane (its normal pointing up), in the 26-connected
    voxel components holding >= min_component times the largest component's points -> (points fp64 CUDA [k,3] in their
    original order, info).

    info holds CUDA tensors keep [N] (crop), flag [N] (crop and above), keys [N] (int64 voxel keys, 2^63 - 1 where not
    flagged), ukeys [m], vcount [m] (points per voxel), label [m] (int32 smallest voxel index of the component),
    comp_count [m] (points per component at its label), voxel_keep [m], point_keep [N], index [k] (int32); and the ints
    voxels, components, kept_components, kept."""
    torch = _torch()
    ops = _ops()
    plane = np.ascontiguousarray(plane, np.float64).reshape(-1)
    if plane.shape != (4,) or not np.isfinite(plane).all() or abs(plane[:3] @ plane[:3] - 1) > 1e-6:
        raise ValueError(f'plane must be (nx, ny, nz, d) with a unit normal, got {plane}')
    if not (np.isfinite(voxel) and voxel > 0) or not np.isfinite(above):
        raise ValueError(f'voxel must be positive and above finite, got {voxel}, {above}')
    if not 0.0 <= min_component <= 1.0:
        raise ValueError(f'min_component must lie in [0, 1], got {min_component}')
    p = _cloud(points, 'isolate_object')
    keep, _, kept = crop_points(p, sphere, box)
    if kept.shape[0] == 0:
        raise ValueError('isolate_object: no point lies inside the crop region')
    n, dev = p.shape[0], p.device
    lo, hi = kept.amin(0).cpu().numpy(), kept.amax(0).cpu().numpy()
    if (np.floor((hi - lo) / voxel) >= _KEY_LIMIT).any():
        raise ValueError(f'isolate_object: extent {hi - lo} at voxel {voxel} needs more than {_KEY_LIMIT} cells along an axis')
    with torch.cuda.device(dev):
        flag = torch.empty(n, dtype=torch.uint8, device=dev)
        keys = torch.empty(n, dtype=torch.int64, device=dev)
        ops.K('nero_objprep_above', p, n, keep, plane, float(above), np.ascontiguousarray(lo), float(voxel), flag, keys)
        skeys, _ = torch.sort(keys)                             # plumbing: the occupied voxels in key order
        ukeys, vcount = torch.unique_consecutive(skeys, return_counts=True)
        if int(ukeys[-1]) == _NOKEY:
            ukeys, vcount = ukeys[:-1], vcount[:-1]
        m = ukeys.shape[0]
        if m == 0:
            raise ValueError(f'isolate_object: no point of the crop lies {above} or more over the plane')
        ukeys, vcount = ukeys.contiguous(), vcount.contiguous()
        parent = torch.empty(m, dtype=torch.int32, device=dev)
        label = torch.empty(m, dtype=torch.int32, device=dev)
        ops.K('nero_objprep_voxel_components', ukeys, m, parent, label, launches=3 + (m - 1).bit_length() + 1)
        comp_count = torch.empty(m, dtype=torch.int64, device=dev)
        voxel_keep = torch.empty(m, dtype=torch.uint8, device=dev)
        ops.K('nero_objprep_component_select', label, vcount, m, float(min_component), comp_count, voxel_keep, launches=2)
        point_keep = torch.empty(n, dtype=torch.uint8, device=dev)
        ops.K('nero_objprep_point_keep', keys, flag, n, ukeys, m, voxel_keep, point_keep)
        idx, out = _compact(p, point_keep, True)
        roots = label == torch.arange(m, device=dev, dtype=torch.int32)
        kept_roots = roots & voxel_keep.bool()
    info = dict(keep=keep, flag=flag, keys=keys, ukeys=ukeys, vcount=vcount, label=label, comp_count=comp_count, voxel_keep=voxel_keep,
                point_keep=point_keep, index=idx, voxels=m, components=int(roots.sum()), kept_components=int(kept_roots.sum()),
                kept=int(idx.shape[0]))
    return out, info


# ------------------------------------------------------------------------------------------------ frame and normalisation
def forward_direction(center, camera, up):
    """Unit direction from the object centre toward the camera centre, projected onto the plane of normal `up`.  Raises
    ValueError when it is (nearly) parallel to up."""
    u = np.asarray(up, np.float64) / np.linalg.norm(up)
    v = np.asarray(camera, np.float64) - np.asarray(center, np.float64)
    return project_forward(v, u)


def project_forward(forward, up):
    """forward minus its component along up, normalised; ValueError if forward is (nearly) parallel to up."""
    u = np.asarray(up, np.float64) / np.linalg.norm(up)
    f = np.asarray(forward, np.float64)
    nf = np.linalg.norm(f)
    p = f - (f @ u) * u
    if not (nf > 0) or np.linalg.norm(p) <= 1e-6 * nf:
        raise ValueError(f'the forward direction {f} is parallel to up {u}')
    return p / np.linalg.norm(p)


def normalization(points, up, forward, centers=None):
    """What CustomDatabase._normalize does with object_point_cloud.ply = points and meta_info.txt = (up, forward):
    dict(center, offset, scale, R (R_rect), ref_points).  With camera centres [n,3]: camera_dist [n], their distances from
    the origin after normalisation, and inside [n], those below 1 (the renderer assumes cameras outside the unit sphere)."""
    ref_points = np.asarray(points, np.float64).reshape(-1, 3)
    max_pt, min_pt = np.max(ref_points, 0), np.min(ref_points, 0)
    center = (max_pt + min_pt) * 0.5
    offset = -center
    scale = 1 / np.max(np.linalg.norm(ref_points - center[None, :], 2, 1))
    directions = np.stack([np.asarray(up, np.float64), np.asarray(forward, np.float64)])
    up, forward = directions[0], directions[1]
    up, forward = up / np.linalg.norm(up), forward / np.linalg.norm(forward)
    y = np.cross(up, forward)
    x = np.cross(y, up)
    R = np.stack([x / np.linalg.norm(x), y / np.linalg.norm(y), up / np.linalg.norm(up)], 0)
    out = dict(center=center, offset=offset, scale=scale, R=R, ref_points=scale * (ref_points + offset) @ R.T)
    if centers is not None:
        c = scale * (np.asarray(centers, np.float64).reshape(-1, 3) + offset) @ R.T
        out['camera_dist'] = np.linalg.norm(c, axis=1)
        out['inside'] = out['camera_dist'] < 1.0
    return out


def write_meta_info(path, up, forward):
    """meta_info.txt: row 0 up, row 1 forward, as np.loadtxt reads them."""
    np.savetxt(path, np.stack([np.asarray(up, np.float64), np.asarray(forward, np.float64)]))
