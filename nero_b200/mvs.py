"""Dense multi-view stereo on the GPU: a fused point cloud from a COLMAP sparse model and its images, without COLMAP's CUDA
stages.

Reference being replaced (paths relative to the reference repository):
  run_colmap.py:66-90   image_undistorter, patch_match_stereo and stereo_fusion, which write <project>/points.ply, the cloud
                        custom_object.md crops by hand (and tools/prepare_custom_object.py crops here)
patch_match_stereo exists only in CUDA builds of COLMAP.  The workflow is tools/match_features.py (nero_b200.features)
-> tools/map_sparse.py (nero_b200.sfm; or colmap mapper) -> tools/dense_points.py -> tools/prepare_custom_object.py.  This module restates COLMAP's PatchMatch in spirit (a plane per
pixel, NCC over plane-induced homographies, red-black propagation, forward-backward geometric filtering); it is not pinned
to COLMAP's output (DESIGN.md section 2).

The protocol (k_mvs.cu, include/nero_mvs.h):
  * Inputs.  The model comes from objprep.read_colmap_model(tracks=True); K is the one CustomDatabase uses, so SIMPLE_RADIAL
    distortion is ignored, as training ignores it (a limitation: strongly distorted images match worse at their borders;
    undistort.py, tools/undistort_images.py, turns such a model into a pinhole project first).
    Views are taken in name order.  Pixel (x, y) is the image point (x + 1/2, y + 1/2).
  * Grey images.  From uint8 RGB, g = sum(299 R + 587 G + 114 B) / (255000 s^2) over each s x s block, the sum in integers
    and one fp32 division, s = ceil(max(w, h) / max_size); the image is (h // s) x (w // s) and K is scaled by 1 / s in x
    and y (fx, cx, fy, cy).
  * Sources and depth range (host, fp64).  Reference view i scores every other view j by the sparse points in both tracks
    whose triangulation angle at the point lies in [ANGLE_MIN, ANGLE_MAX] degrees; the best SOURCES views with a score >= 1
    are kept, ties in name order.  The depth range is [DEPTH_LO p1, DEPTH_HI p99] of the positive z-depths of i's track
    points (numpy's linear percentiles).  A view with fewer than MIN_SOURCES sources or MIN_TRACK track points is skipped
    and reported.
  * Matching cost.  A hypothesis is a z-depth d and a unit camera-frame normal n with n . r < 0 for the pixel's ray
    r = ((x + 1/2) ifx + ocx, (y + 1/2) ify + ocy, 1) (ifx = fp32(1/fx), ocx = fp32(-cx/fx)).  Against source j the
    window samples (x + k, y + l) for k, l in -RADIUS..RADIUS step STEP (l outer) map through H = A + b m^T, with the host's
    fp32 A = K_j R_ij K_i^-1, b = K_j t_ij and m = (n0 ifx, n1 ify, (n0 ocx + n1 ocy) + n2) / q, q = d ((n0 rx + n1 ry) + n2).
    Source samples are software-bilinear (texel centres at +1/2, clamped to the edge, coordinates first clamped to
    [-1, w + 1]); reference samples read the pixel, clamped to the edge.  cost = clamp(1 - NCC, 0, 2) with NCC =
    (E[rs] - E[r] E[s]) / sqrt(var r var s); 2 if the centre maps behind j or outside j, or either variance is below 1e-5.
    The reference mean and variance are computed once per pixel.  The aggregate is the mean of the BEST smallest source
    costs (of two when there are two sources).
  * Randomness.  u = (mix(key ^ dim) >> 8) 2^-24 with key = mix(mix(mix(mix(seed 0x9e3779b9 + 0x7f4a7c15) ^ view) ^ stage)
    ^ pixel), mix = rl_mix of hash.cuh, view = index in name order, stage 0 for the initialisation and 1 + 2 it + colour for
    a pass, pixel = y w + x.  A random hypothesis draws inverse depth 1/dmax + u0 (1/dmin - 1/dmax) and a normalised
    uniform vector in [-1, 1]^3 (dims 1-3), flipped to face the camera.
  * PatchMatch.  Random initial planes; then ITERATIONS times a red pass ((x + y) even) and a black pass.  In a pass each
    pixel of that colour tries, in order: its current plane (its stored cost); the planes of the pixels at distance 1 and 5
    along the axes, (-1, 0), (1, 0), (0, -1), (0, 1), then at 5, re-intersected with its ray (skipped when n . r >= 0 or the
    depth leaves the range); its depth perturbed in inverse depth by +- 2^-(it + 2) of the inverse-depth range (u dim 0);
    its normal perturbed by +- 2^-(it + 1) per component and renormalised (dims 1-3, skipped if it faces away); a fresh
    random plane (dims 4-7).  It keeps the lowest cost, ties to the earlier.  A pass reads only the other colour, and every
    fp32 operation is an uncontracted, correctly rounded one in the order above, so the result is the same on every run.
  * Filter (fp64).  A pixel with cost <= MAX_COST is projected from its centre at depth d into each source; the source
    pixel containing the projection (if its cost <= MAX_COST) is back-projected at its centre with its depth and
    reprojected into the reference.  The source agrees when the reprojection error is <= REPROJ px, |z - d| <= REL_DEPTH d
    and the cosine of the normals is >= cos(NORMAL_DEG) (computed on the host).  The pixel is kept with MIN_CONSISTENT
    agreeing sources; its depth goes to a map that is 0 where a pixel is rejected.
  * Fusion.  evaluate.depth_to_points_cuda unprojects each view's filtered map in fp64 with cx, cy lowered by 1/2 (it
    unprojects at (x, y)), in (view in name order, row, column) order; --voxel optionally thins the cloud with
    evaluate.voxel_down_sample_cuda.
  * Normals (normals=True).  Each kept pixel's plane normal n (camera frame) rotated to the world frame in fp64, R^T n with
    R the world -> camera rotation, in the same order as the points.  With --voxel, each voxel's normals are averaged with
    its points and the mean renormalised (a mean that cancels to zero stays zero).  They point towards the camera that saw
    the pixel, i.e. out of the surface.
"""
import os

import numpy as np

MAX_SIZE = 1600          # longest grey-image side
SOURCES = 8              # source views per reference view
MIN_SOURCES = 2
MIN_TRACK = 10           # sparse points a reference view must see
ANGLE_MIN, ANGLE_MAX = 2.0, 60.0    # triangulation angles (degrees) that score a source
DEPTH_LO, DEPTH_HI = 0.75, 1.25     # depth range = [DEPTH_LO p1, DEPTH_HI p99] of the track depths
RADIUS, STEP = 4, 2      # matching window offsets -RADIUS..RADIUS step STEP (25 samples)
BEST = 3                 # the aggregate cost is the mean of the BEST smallest source costs
ITERATIONS = 8           # red + black passes
MAX_COST = 0.5
REPROJ = 1.0             # px
REL_DEPTH = 0.01
NORMAL_DEG = 10.0
MIN_CONSISTENT = 2
SEED = 0
_MAX_SRC = 16            # NERO_MVS_MAX_SOURCES (include/nero_mvs.h)


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ host geometry
def grey_scale(w, h, max_size=MAX_SIZE):
    """s = ceil(max(w, h) / max_size): the block side of the grey image."""
    if not max_size >= 1:
        raise ValueError(f'max_size must be >= 1, got {max_size}')
    return max(1, -(-max(int(w), int(h)) // int(max_size)))


def scale_K(K, s):
    """fp64 K of the grey image: fx, cx, fy, cy divided by s."""
    K = np.asarray(K, np.float64).copy()
    K[:2] /= s
    return K


def kinv32(K):
    """(ifx, ify, ocx, ocy) as fp32: the ray of image point (u, v) is (u ifx + ocx, v ify + ocy, 1)."""
    K = np.asarray(K, np.float64)
    return tuple(float(np.float32(v)) for v in (1 / K[0, 0], 1 / K[1, 1], -K[0, 2] / K[0, 0], -K[1, 2] / K[1, 1]))


def _Rt(pose):
    P = np.asarray(pose, np.float64)
    return P[:, :3], P[:, 3]


def relative(pose_i, pose_j):
    """(R_ij, t_ij): camera i -> camera j, fp64."""
    Ri, ti = _Rt(pose_i)
    Rj, tj = _Rt(pose_j)
    R = Rj @ Ri.T
    return R, tj - R @ ti


def pm_table(K_i, pose_i, Ks, poses):
    """src_geo fp32 [S,12]: A = K_j R_ij K_i^-1 (row-major), b = K_j t_ij for the sources (Ks, poses)."""
    Ki_inv = np.linalg.inv(np.asarray(K_i, np.float64))
    rows = []
    for K_j, pose_j in zip(Ks, poses):
        R, t = relative(pose_i, pose_j)
        K_j = np.asarray(K_j, np.float64)
        rows.append(np.concatenate([(K_j @ R @ Ki_inv).reshape(9), K_j @ t]))
    return np.asarray(rows, np.float64).reshape(-1, 12).astype(np.float32)


def filter_table(pose_i, Ks, poses):
    """geo fp64 [S,28]: R_ij, t_ij, R_ji, t_ji, fx_j, fy_j, cx_j, cy_j."""
    rows = []
    for K_j, pose_j in zip(Ks, poses):
        Rij, tij = relative(pose_i, pose_j)
        Rji, tji = relative(pose_j, pose_i)
        K_j = np.asarray(K_j, np.float64)
        rows.append(np.concatenate([Rij.reshape(9), tij, Rji.reshape(9), tji, [K_j[0, 0], K_j[1, 1], K_j[0, 2], K_j[1, 2]]]))
    return np.asarray(rows, np.float64).reshape(-1, 28)


def select_sources(points, tracks, poses, image_ids, sources=SOURCES, angles=(ANGLE_MIN, ANGLE_MAX), depth=(DEPTH_LO, DEPTH_HI),
                   min_sources=MIN_SOURCES, min_track=MIN_TRACK):
    """Source views and depth ranges of the views (poses [n,3,4], image_ids [n], both in name order) from the sparse points
    [P,3] and their tracks (image ids per point).  -> (score int64 [n,n], plan), plan[i] = dict(sources: view indices,
    range: (dmin, dmax) or None, track: the number of track points, skip: None or the reason the view is skipped)."""
    pts = np.asarray(points, np.float64).reshape(-1, 3)
    poses = np.asarray(poses, np.float64).reshape(-1, 3, 4)
    n = poses.shape[0]
    index = {int(iid): k for k, iid in enumerate(image_ids)}
    R, t = poses[:, :, :3], poses[:, :, 3]
    centers = -np.einsum('nji,nj->ni', R, t)
    lo_c, hi_c = np.cos(np.radians(angles[1])), np.cos(np.radians(angles[0]))
    score = np.zeros((n, n), np.int64)
    members = [[] for _ in range(n)]
    for p, (x, tr) in enumerate(zip(pts, tracks)):
        mem = np.unique([index[int(i)] for i in tr if int(i) in index]).astype(np.int64)
        for k in mem:
            members[k].append(p)
        if mem.shape[0] < 2:
            continue
        v = centers[mem] - x
        v = v / np.linalg.norm(v, axis=1, keepdims=True)
        c = v @ v.T
        score[np.ix_(mem, mem)] += ((c >= lo_c) & (c <= hi_c)).astype(np.int64)
    np.fill_diagonal(score, 0)
    plan = []
    for i in range(n):
        cand = [j for j in range(n) if j != i and score[i, j] >= 1]
        src = sorted(cand, key=lambda j: (-score[i, j], j))[:sources]
        mem = np.asarray(members[i], np.int64)
        z = (pts[mem] @ R[i][2] + t[i][2]) if mem.shape[0] else np.zeros(0)
        z = z[z > 0]
        entry = dict(sources=src, range=None, track=int(z.shape[0]), skip=None)
        if len(src) < min_sources:
            entry['skip'] = f'{len(src)} source views (need {min_sources})'
        elif z.shape[0] < min_track:
            entry['skip'] = f'{z.shape[0]} sparse points in front of the camera (need {min_track})'
        else:
            p1, p99 = np.percentile(z, [1, 99])
            entry['range'] = (depth[0] * p1, depth[1] * p99)
        plan.append(entry)
    return score, plan


def read_rgb(path):
    """uint8 RGB [h,w,3] of an image file, in its stored pixel order: an EXIF orientation is ignored, as COLMAP and
    run_colmap.py's skimage reader ignore it, so the pixels are in the frame of the COLMAP model's cameras."""
    import cv2
    img = cv2.imread(path, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)
    if img is None:
        raise FileNotFoundError(f'{path}: cannot read the image')
    return np.ascontiguousarray(img[..., ::-1])


# ------------------------------------------------------------------------------------------------ GPU steps
def prepare_grey(rgb, s):
    """CUDA fp32 [h // s, w // s] grey image of uint8 RGB [h,w,3] (numpy array or tensor)."""
    torch = _torch()
    x = rgb if torch.is_tensor(rgb) else torch.from_numpy(np.ascontiguousarray(rgb, np.uint8))
    if x.dtype != torch.uint8 or x.dim() != 3 or x.shape[2] != 3:
        raise ValueError(f'prepare_grey needs uint8 RGB [h,w,3], got {x.dtype} {tuple(x.shape)}')
    x = x.cuda().contiguous()
    h, w = x.shape[:2]
    if h // s < 1 or w // s < 1:
        raise ValueError(f'image {w} x {h} is smaller than one {s} x {s} block')
    out = torch.empty(h // s, w // s, dtype=torch.float32, device=x.device)
    _ops().K('nero_mvs_grey', x, w, h, int(s), out)
    return out


class _Ref:
    """Device tables of one reference view."""

    def __init__(self, grey, K, stats, src_greys, src_geo):
        torch = _torch()
        dev = grey.device
        self.grey, self.h, self.w = grey, grey.shape[0], grey.shape[1]
        self.kinv = kinv32(K)
        self.stats = stats
        self.S = len(src_greys)
        self.src_img = torch.tensor([g.data_ptr() for g in src_greys], dtype=torch.int64, device=dev)
        self.src_wh = torch.tensor([[g.shape[1], g.shape[0]] for g in src_greys], dtype=torch.int32, device=dev)
        self.src_geo = torch.from_numpy(np.ascontiguousarray(src_geo, np.float32)).to(dev)
        self.keep = src_greys


def ref_stats(grey, radius=RADIUS, step=STEP):
    torch = _torch()
    h, w = grey.shape
    stats = torch.empty(h, w, 2, dtype=torch.float32, device=grey.device)
    _ops().K('nero_mvs_ref_stats', grey, w, h, int(radius), int(step), stats)
    return stats


def patchmatch(grey, K, src_greys, src_geo, drange, view, iterations=ITERATIONS, radius=RADIUS, step=STEP, seed=SEED, trace=None):
    """PatchMatch of one reference view -> (planes CUDA fp32 [h,w,4] (depth, normal), cost [h,w]).  grey: its CUDA grey
    image, K its fp64 intrinsics (scaled), src_greys the sources' grey images, src_geo their pm_table, drange (dmin, dmax),
    view its index in name order.  trace: a list that receives (planes, cost) copies after the initialisation and after
    every pass."""
    torch = _torch()
    ops = _ops()
    if not 2 <= len(src_greys) <= _MAX_SRC:
        raise ValueError(f'patchmatch needs 2 to {_MAX_SRC} sources, got {len(src_greys)}')
    dmin, dmax = float(np.float32(drange[0])), float(np.float32(drange[1]))
    if not (0 < dmin <= dmax < np.inf):
        raise ValueError(f'depth range must satisfy 0 < dmin <= dmax, got {drange}')
    stats = ref_stats(grey, radius, step)
    r = _Ref(grey, K, stats, src_greys, src_geo)
    planes = torch.empty(r.h, r.w, 4, dtype=torch.float32, device=grey.device)
    cost = torch.empty(r.h, r.w, dtype=torch.float32, device=grey.device)
    common = (grey, r.w, r.h) + r.kinv + (stats, r.src_img, r.src_wh, r.src_geo, r.S, int(radius), int(step), dmin, dmax, int(seed), int(view))
    ops.K('nero_mvs_init', *common, planes, cost)
    if trace is not None:
        trace.append((planes.clone(), cost.clone()))
    for it in range(iterations):
        for colour in (0, 1):
            ops.K('nero_mvs_pass', *common, it, colour, planes, cost)
            if trace is not None:
                trace.append((planes.clone(), cost.clone()))
    return planes, cost


def geometric_filter(K, pose, planes, cost, src, max_cost=MAX_COST, reproj=REPROJ, rel_depth=REL_DEPTH, normal_deg=NORMAL_DEG,
                     min_consistent=MIN_CONSISTENT):
    """(depth CUDA fp32 [h,w], 0 where rejected; count int32 [h,w] of agreeing sources) of a reference view.  src: list of
    (K_j, pose_j, planes_j, cost_j) of its sources that have hypotheses."""
    torch = _torch()
    h, w = cost.shape
    dev = cost.device
    S = len(src)
    if S > _MAX_SRC:
        raise ValueError(f'geometric_filter takes at most {_MAX_SRC} sources, got {S}')
    K = np.asarray(K, np.float64)
    depth = torch.empty(h, w, dtype=torch.float32, device=dev)
    count = torch.empty(h, w, dtype=torch.int32, device=dev)
    geo = torch.from_numpy(filter_table(pose, [s[0] for s in src], [s[1] for s in src])).to(dev)
    sp = torch.tensor([s[2].data_ptr() for s in src], dtype=torch.int64, device=dev)
    sc = torch.tensor([s[3].data_ptr() for s in src], dtype=torch.int64, device=dev)
    wh = torch.tensor([[s[3].shape[1], s[3].shape[0]] for s in src], dtype=torch.int32, device=dev).reshape(-1, 2)
    _ops().K('nero_mvs_filter', w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], planes, cost, sp if S else None, sc if S else None,
             wh if S else None, geo if S else None, S, float(max_cost), float(reproj) ** 2, float(rel_depth),
             float(np.cos(np.radians(normal_deg))), int(min_consistent), depth, count)
    return depth, count


def centre_K(K):
    """K with cx, cy lowered by 1/2: depth_to_points_cuda then unprojects pixel (x, y) at its centre."""
    K = np.asarray(K, np.float64).copy()
    K[0, 2] -= 0.5
    K[1, 2] -= 0.5
    return K


def reconstruct(views, points, tracks, images, max_size=MAX_SIZE, sources=SOURCES, iterations=ITERATIONS, radius=RADIUS, step=STEP,
                seed=SEED, voxel=None, trace=None, log=None, normals=False):
    """The dense cloud of a COLMAP model: views, points and tracks from objprep.read_colmap_model(path, tracks=True);
    images: a callable name -> uint8 RGB [h,w,3].  -> (points CUDA fp64 [n,3], info), or with normals=True (points, normals
    CUDA fp64 [n,3], info).  info holds, per view in name order, names, Ks (fp64, scaled), poses, greys, plan
    (select_sources), planes, cost, depth (filtered), count; and the ints fused (points before --voxel) and views_used.
    trace: dict view index -> list, filled by patchmatch."""
    torch = _torch()
    from .evaluate import depth_to_points_cuda, voxel_down_sample_cuda
    if not 1 <= sources <= _MAX_SRC:
        raise ValueError(f'sources must lie in [1, {_MAX_SRC}], got {sources}')
    if iterations < 0 or radius < 0 or step < 1:
        raise ValueError(f'need iterations >= 0, radius >= 0 and step >= 1, got {iterations}, {radius}, {step}')
    items = sorted(views.items(), key=lambda kv: kv[1][0])
    ids = [iid for iid, _ in items]
    names = [v[0] for _, v in items]
    poses = np.stack([np.asarray(v[1], np.float32) for _, v in items]) if items else np.zeros((0, 3, 4), np.float32)
    score, plan = select_sources(points, tracks, poses, ids, sources)
    greys, Ks = [], []
    for (_, (name, _, K)) in items:
        rgb = images(name)
        s = grey_scale(rgb.shape[1], rgb.shape[0], max_size)
        greys.append(prepare_grey(rgb, s))
        Ks.append(scale_K(K, s))
    n = len(items)
    planes, cost = [None] * n, [None] * n
    for i in range(n):
        e = plan[i]
        if e['skip']:
            if log:
                log(f'{names[i]}: skipped, {e["skip"]}')
            continue
        src = e['sources']
        geo = pm_table(Ks[i], poses[i], [Ks[j] for j in src], [poses[j] for j in src])
        tr = None
        if trace is not None:
            tr = trace.setdefault(i, [])
        planes[i], cost[i] = patchmatch(greys[i], Ks[i], [greys[j] for j in src], geo, e['range'], i, iterations, radius, step, seed, tr)
    depth, count, clouds, nclouds = [None] * n, [None] * n, [], []
    for i in range(n):
        if planes[i] is None:
            continue
        src = [(Ks[j], poses[j], planes[j], cost[j]) for j in plan[i]['sources'] if planes[j] is not None]
        depth[i], count[i] = geometric_filter(Ks[i], poses[i], planes[i], cost[i], src)
        clouds.append(depth_to_points_cuda(depth[i], poses[i].astype(np.float64), centre_K(Ks[i])))
        if normals:
            # the kept pixels in row-major order, as depth_to_points_cuda emits them; n^T R = (R^T n)^T
            d = depth[i].reshape(-1)
            keep = (d > 0) & torch.isfinite(d)
            R = torch.from_numpy(poses[i][:, :3].astype(np.float64)).to(d.device)
            nclouds.append(planes[i].reshape(-1, 4)[keep, 1:4].to(torch.float64) @ R)
    dev = torch.device('cuda')
    cloud = torch.cat(clouds, 0).to(torch.float64) if clouds else torch.zeros(0, 3, dtype=torch.float64, device=dev)
    nrm = torch.cat(nclouds, 0) if nclouds else torch.zeros(0, 3, dtype=torch.float64, device=dev)
    fused = int(cloud.shape[0])
    if voxel is not None and fused:
        if normals:
            cloud, nrm = voxel_down_sample_cuda(cloud, voxel, nrm)
            length = torch.linalg.norm(nrm, dim=1, keepdim=True)
            nrm = torch.where(length > 0, nrm / torch.where(length > 0, length, torch.ones_like(length)), nrm)
        else:
            cloud = voxel_down_sample_cuda(cloud, voxel)
    info = dict(names=names, ids=ids, Ks=Ks, poses=poses, greys=greys, score=score, plan=plan, planes=planes, cost=cost, depth=depth,
                count=count, fused=fused, views_used=sum(p is not None for p in planes))
    if normals:
        return cloud, nrm, info
    return cloud, info


def image_reader(image_dir):
    """A callable name -> uint8 RGB of <image_dir>/<name>."""
    return lambda name: read_rgb(os.path.join(image_dir, name))
