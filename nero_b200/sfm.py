"""Incremental structure from motion on the GPU: cameras, poses and sparse points from the COLMAP database that
features.py writes, saved as the COLMAP model that dense_points.py and prepare_custom_object.py read, without COLMAP's
mapper.

Reference being replaced (paths relative to the reference repository):
  run_colmap.py:54-58   colmap mapper --database_path <root>/database.db --image_path <images> --output_path <root>/sparse
What the later steps read is the same: <root>/sparse/0 with cameras.bin, images.bin and points3D.bin.  The mapper is
COLMAP's incremental scheme in spirit and is not pinned to COLMAP's (DESIGN.md section 2).

The protocol (k_sfm.cu, include/nero_sfm.h):
  * Input.  Cameras, images, keypoints and two_view_geometries of the database (sqlite3); only the stored inlier matches
    of verified pairs (rows > 0) are used.  Every camera must have the camera model the mapper estimates: SIMPLE_PINHOLE
    (the default, what features.py writes by default) or SIMPLE_RADIAL (camera_model='SIMPLE_RADIAL').  Camera
    ids, image ids and names carry through to the model.  The images of the largest connected component of the verified
    pair graph (most images, ties to the lower smallest id) are reconstructed, at most MAX_IMAGES of them; the others are
    reported as not registered.
  * Tracks.  Nodes are the (image, keypoint) pairs of any verified match in (image id, keypoint) order, edges the inlier
    matches.  Union-find labels each node with the smallest node of its component, the roots are compacted in node order
    (block_offsets), so track ids follow the smallest node.  A track with two keypoints in one image is dropped.
  * Initial pair.  Verified pairs by inlier count descending, ties to the lower pair id, at most INIT_TRIES of them.
    E = K2^T F K1 from the prior K; of its four (R, t) the one with most tracks in front of both cameras.  The tracks
    seen by both images are triangulated, then a two-view bundle adjustment (focal held at the prior, INIT_BA_ITERS
    iterations) and the filter below.  The pair is accepted with >= INIT_MIN_POINTS points and a median triangulation
    angle >= INIT_MIN_TRI_ANGLE; otherwise the next pair is tried, and no accepted pair is an error.
  * Registration.  The next image is the unregistered, not yet failed one that sees the most points (ties to the lower
    image id).  P3P RANSAC over its 2D-3D correspondences: P3P_HYPOTHESES Lambda Twist solves of 3 hashed draws (seed
    SEED, the image id), inliers within ABS_POSE_MAX_ERROR px, the largest integer count wins (ties to the lower
    hypothesis).  The image is accepted with >= ABS_POSE_MIN_INLIERS inliers that are >= ABS_POSE_MIN_RATIO of its
    correspondences, else it is marked failed (a later registration clears the marks).  Its pose, and its camera's focal
    once >= FOCAL_MIN_IMAGES images are registered, are refined on the inliers with the points held (REFINE_ITERS).
  * Triangulation.  Each track seen by the new image with no point and >= 2 registered observations is triangulated
    from all of them (multi-view DLT, k_sfm.cu) and kept when it is in front of every camera, every reprojection is
    <= MAX_REPROJ px and its largest ray angle is >= MIN_TRI_ANGLE.  A track that has a point gains the new image's
    observation when it reprojects within MAX_REPROJ px.
  * Bundle adjustment.  Levenberg-Marquardt in fp64 after every registration (GLOBAL_BA_ITERS iterations) and once at
    the end to convergence (FINAL_BA_ITERS at most): per image an axis-angle update of R and t, per camera the focal
    (free once FOCAL_MIN_IMAGES images are registered), per point its position; the principal point is fixed.  Gauge: the
    first initial image's pose and the largest |component| of the second's translation are fixed.  Squared loss.  The
    points are eliminated by the Schur complement; the dense reduced system (6 per image + 1 per camera) is solved by
    torch.linalg.cholesky_ex.  Its entries are summed over segments of an (o, o') list cut into chunks of CHUNK (one
    block per chunk, then the chunks of a segment in a fixed shape), so a shared camera's focal segments, which hold
    every pair, are spread over the GPU.  Marquardt damping diag * (1 + lambda), lambda from LAMBDA0, / 10 on a step that lowers the
    cost, * 10 and retried otherwise.  Sums have a fixed order: per point in observation order, per system entry over a
    segment of an (o, o') list sorted once per adjustment, block partials in block order.
  * Filter.  After every adjustment observations reprojecting beyond MAX_REPROJ px are dropped, then points with fewer
    than two observations or a largest ray angle < MIN_TRI_ANGLE.
  * SIMPLE_RADIAL (include/nero_sfm_radial.h).  Each camera has two free parameters, f and k; the principal point stays
    fixed.  k starts at the database's value (0 from features.py) and follows the focal's rule: held during the initial
    pair and while fewer than FOCAL_MIN_IMAGES images are registered, free after that in the registration refinement and
    in every global adjustment.  Every reprojection error compared with a pixel threshold is measured in the distorted
    image, where the keypoints are: the adjustment's cost, the filter, a new track's acceptance, track continuation and
    the model's per-point error.  P3P and the DLT work on rays, so they take the keypoints undistorted with the camera's
    current (f, k) (undistort.points) as pinhole pixels f x + (cx, cy) of the same camera; a keypoint that is invalid at
    the current k is left out of that registration or triangulation.  P3P's inlier threshold ABS_POSE_MAX_ERROR is
    therefore in undistorted pixels.  A DLT point is judged by the distorted reprojection (nero_sfm_radial_filter), not
    by the DLT's own pixel statistic.  After an adjustment the undistorted keypoints of the cameras whose (f, k) it
    changed are recomputed.
  * Model.  One model of the registered images: SIMPLE_PINHOLE (f, cx, cy) or SIMPLE_RADIAL (f, cx, cy, k) per camera,
    every keypoint of an image as a POINTS2D entry (point3D id -1 without a point), points numbered 1.. in track order,
    RGB the rounded mean of the pixels (mvs.read_rgb, stored order) under its observations, error the mean reprojection
    error of its track.  The same input gives the same bytes.
"""
import math
import os
import sqlite3
import time

import numpy as np

from . import features as Ft
from . import objprep

MAX_IMAGES = 500                  # NERO_SFM_MAX_IMAGES: the reduced camera system is dense
CHUNK = 256                       # NERO_SFM_CHUNK: entries one block of the reduced-system kernels sums
INIT_MIN_POINTS = 100             # COLMAP init_min_num_inliers
INIT_MIN_TRI_ANGLE = 16.0         # degrees, COLMAP init_min_tri_angle
INIT_TRIES = 50
INIT_BA_ITERS = 30
ABS_POSE_MAX_ERROR = 12.0         # px, COLMAP abs_pose_max_error
ABS_POSE_MIN_INLIERS = 30         # COLMAP abs_pose_min_num_inliers
ABS_POSE_MIN_RATIO = 0.25         # COLMAP abs_pose_min_inlier_ratio
P3P_HYPOTHESES = 1024
REFINE_ITERS = 10
MAX_REPROJ = 4.0                  # px, COLMAP tri_complete_max_reproj_error / filter_max_reproj_error
MIN_TRI_ANGLE = 1.5               # degrees, COLMAP tri_min_angle / filter_min_tri_angle
FOCAL_MIN_IMAGES = 3
GLOBAL_BA_ITERS = 10
FINAL_BA_ITERS = 100
LAMBDA0 = 1e-4
BA_TOL = 1e-12                    # relative cost decrease that ends an adjustment
SEED = 0
CAMERA_MODELS = ('SIMPLE_PINHOLE', 'SIMPLE_RADIAL')   # what the mapper estimates (map_sparse.py --camera-model)


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ database
def read_database(path):
    """-> dict(cameras {id: (model, w, h, params fp64)}, images {id: (name, camera id)}, keypoints {id: fp64 [n, 2]},
    pairs {(id1, id2): (inlier matches int64 [m, 2], F [3, 3])} of the verified pairs, id1 < id2)."""
    if not os.path.isfile(path):
        raise FileNotFoundError(f'{path}: no database')
    con = sqlite3.connect(f'file:{path}?mode=ro', uri=True)
    try:
        cams = {int(c): (int(m), int(w), int(h), np.frombuffer(p, np.float64).copy())
                for c, m, w, h, p in con.execute('SELECT camera_id, model, width, height, params FROM cameras')}
        images = {int(i): (n, int(c)) for i, n, c in con.execute('SELECT image_id, name, camera_id FROM images')}
        kps = {int(i): np.frombuffer(b, np.float32).reshape(r, c)[:, :2].astype(np.float64)
               for i, r, c, b in con.execute('SELECT image_id, rows, cols, data FROM keypoints') if r > 0}
        pairs = {}
        for pid, r, d, F in con.execute('SELECT pair_id, rows, data, F FROM two_view_geometries WHERE rows > 0'):
            a, b = Ft.pair_ids(pid)
            m = np.frombuffer(d, np.uint32).reshape(r, 2).astype(np.int64)
            pairs[a, b] = (m, np.frombuffer(F, np.float64).reshape(3, 3).copy() if F else np.zeros((3, 3)))
    finally:
        con.close()
    return dict(cameras=cams, images=images, keypoints=kps, pairs=pairs)


def check_database(db, camera_model='SIMPLE_PINHOLE'):
    """The refusals that need no GPU: an unknown camera_model, a camera of another model than camera_model, or no
    verified pair."""
    if camera_model not in CAMERA_MODELS:
        raise ValueError(f'camera model {camera_model!r}: the mapper estimates {" or ".join(CAMERA_MODELS)} cameras')
    bad = sorted(c for c, (m, *_r) in db['cameras'].items() if m != Ft.CAMERA_MODELS[camera_model])
    if bad:
        name = objprep.CAMERA_MODELS.get(db['cameras'][bad[0]][0], ('unknown',))[0]
        if camera_model == 'SIMPLE_PINHOLE':
            raise ValueError(f'camera {bad[0]} is {name}: the mapper reconstructs SIMPLE_PINHOLE cameras only (the model '
                             'match_features.py writes by default); for SIMPLE_RADIAL cameras give --camera-model SIMPLE_RADIAL')
        raise ValueError(f'camera {bad[0]} is {name}: --camera-model SIMPLE_RADIAL estimates SIMPLE_RADIAL cameras only (write '
                         'the database with match_features.py --camera-model SIMPLE_RADIAL)')
    if camera_model == 'SIMPLE_RADIAL':
        bad = sorted(c for c, (_m, _w, _h, p) in db['cameras'].items() if p.shape[0] != 4 or not np.isfinite(p).all())
        if bad:
            raise ValueError(f'camera {bad[0]}: SIMPLE_RADIAL needs 4 finite parameters (f, cx, cy, k)')
    if not db['pairs']:
        raise ValueError('the database has no verified image pair (two_view_geometries with inlier matches)')


def largest_component(image_ids, pairs):
    """Image ids of the largest connected component of the verified pair graph (most images, ties to the lower smallest
    id), sorted."""
    parent = {i: i for i in image_ids}

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b in sorted(pairs):
        ra, rb = find(a), find(b)
        if ra != rb:
            parent[max(ra, rb)] = min(ra, rb)
    comps = {}
    for i in sorted(image_ids):
        comps.setdefault(find(i), []).append(i)
    return max(comps.values(), key=lambda c: (len(c), -c[0]))


# ------------------------------------------------------------------------------------------------ GPU steps
def _dev(a, dtype):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype)).cuda()


def build_tracks(edges, n):
    """Union-find tracks of n nodes under the edges [E, 2] -> (label [n], track [n], number of tracks), numpy."""
    torch = _torch()
    nb = -(-n // 256)
    label = torch.empty(n, dtype=torch.int32, device='cuda')
    track = torch.empty(n, dtype=torch.int32, device='cuda')
    cnt = torch.empty(nb, dtype=torch.int32, device='cuda')
    off = torch.empty(nb, dtype=torch.int64, device='cuda')
    total = torch.empty(1, dtype=torch.int64, device='cuda')
    e = _dev(np.asarray(edges).reshape(-1, 2), np.int32)
    rounds = 1 + int(math.ceil(math.log2(max(n, 1))))         # uf_flatten's pointer-jumping rounds
    _ops().K('nero_sfm_tracks', e, e.shape[0], n, label, cnt, off, total, track, launches=5 + rounds + int(e.shape[0] > 0))
    return label.cpu().numpy(), track.cpu().numpy(), int(total.item())


def p3p_ransac(xy, X, f, cx, cy, image, hypotheses=P3P_HYPOTHESES, seed=SEED, max_err=ABS_POSE_MAX_ERROR):
    """-> (pose [12], winning hypothesis, count, inlier bool [n], counts [H]) of the correspondences xy [n, 2] -> X [n, 3]."""
    torch = _torch()
    n = xy.shape[0]
    counts = torch.empty(hypotheses, dtype=torch.int32, device='cuda')
    poses = torch.empty(hypotheses, 12, dtype=torch.float64, device='cuda')
    best = torch.empty(2, dtype=torch.int32, device='cuda')
    pose = torch.empty(12, dtype=torch.float64, device='cuda')
    inl = torch.empty(n, dtype=torch.uint8, device='cuda')
    _ops().K('nero_sfm_p3p', _dev(xy, np.float64), _dev(X, np.float64), n, float(f), float(cx), float(cy), int(image), int(hypotheses),
             int(seed), float(max_err) ** 2, counts, poses, best, pose, inl, launches=2)
    b = best.cpu().numpy()
    return pose.cpu().numpy(), int(b[0]), int(b[1]), inl.cpu().numpy().astype(bool), counts.cpu().numpy()


def _cams(pose, img_cam, focal, pp):
    return _dev(pose, np.float64), _dev(img_cam, np.int32), _dev(focal, np.float64), _dev(pp, np.float64)


def triangulate(off, obs_img, obs_xy, pose, img_cam, focal, pp):
    """DLT points of the tracks off [T + 1] over the observations -> (X [T, 3], stat [T, 3] = smallest depth, largest
    error px, largest angle rad)."""
    torch = _torch()
    T = off.shape[0] - 1
    X = torch.empty(max(T, 1), 3, dtype=torch.float64, device='cuda')
    st = torch.empty(max(T, 1), 3, dtype=torch.float64, device='cuda')
    if T:
        _ops().K('nero_sfm_triangulate', _dev(off, np.int64), T, _dev(obs_img, np.int32), _dev(obs_xy, np.float64),
                 *_cams(pose, img_cam, focal, pp), X, st)
    return X[:T].cpu().numpy(), st[:T].cpu().numpy()


def reprojection(pt_off, obs_img, obs_xy, pose, img_cam, focal, pp, X, radial=None):
    """-> (err [n, 2] = depth, reprojection error px per observation, angle [P] rad per point).  With radial (k per
    camera) the error is measured through SIMPLE_RADIAL, in the distorted image."""
    torch = _torch()
    P = pt_off.shape[0] - 1
    err = torch.empty(max(obs_img.shape[0], 1), 2, dtype=torch.float64, device='cuda')
    ang = torch.empty(max(P, 1), dtype=torch.float64, device='cuda')
    if P and radial is None:
        _ops().K('nero_sfm_filter', _dev(pt_off, np.int64), P, _dev(obs_img, np.int32), _dev(obs_xy, np.float64),
                 *_cams(pose, img_cam, focal, pp), _dev(X, np.float64), err, ang)
    elif P:
        _ops().K('nero_sfm_radial_filter', _dev(pt_off, np.int64), P, _dev(obs_img, np.int32), _dev(obs_xy, np.float64),
                 *_cams(pose, img_cam, focal, pp), _dev(radial, np.float64), _dev(X, np.float64), err, ang)
    return err[:obs_img.shape[0]].cpu().numpy(), ang[:P].cpu().numpy()


def _chunks(counts, key):
    """Cut consecutive segments of `counts` entries into chunks of at most CHUNK -> (chunk [C, 2] int64 (begin, end),
    chunk key (the segment's key row), seg_chunk [S + 1] int64: segment s owns chunks seg_chunk[s] .. seg_chunk[s + 1] - 1)."""
    torch = _torch()
    dev = counts.device
    seg_off = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(counts, 0)])
    per = (counts + CHUNK - 1) // CHUNK
    seg_chunk = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev), torch.cumsum(per, 0)])
    seg = torch.repeat_interleave(torch.arange(counts.shape[0], device=dev), per)
    begin = seg_off[seg] + CHUNK * (torch.arange(seg.shape[0], device=dev) - seg_chunk[seg])
    end = torch.minimum(begin + CHUNK, seg_off[seg + 1])
    return torch.stack([begin, end], 1).contiguous(), key[seg].contiguous(), seg_chunk


class Problem:
    """One bundle adjustment on the device: the point-ordered observations, the parameters and the reduced-system layout
    (the (o, o') entry list sorted by (row block, column block) once).  radial (k per camera) makes the cameras
    SIMPLE_RADIAL (include/nero_sfm_radial.h): each camera then has the two columns (f, k), fixed [6 nimg + 2 ncam]; with
    None the cameras are SIMPLE_PINHOLE and fixed is [6 nimg + ncam]."""

    def __init__(self, pose, focal, pp, img_cam, X, pt_off, obs_img, obs_xy, fixed, fix_points=False, radial=None):
        torch = _torch()
        self.nimg, self.ncam, self.P, self.n = pose.shape[0], focal.shape[0], X.shape[0], obs_img.shape[0]
        if self.nimg > MAX_IMAGES:
            raise ValueError(f'{self.nimg} images: the bundle adjustment takes at most {MAX_IMAGES}')
        self.pose, self.img_cam, self.focal, self.pp = _cams(pose, img_cam, focal, pp)
        self.X = _dev(X, np.float64)
        self.pt_off = _dev(pt_off, np.int64)
        self.obs_img = _dev(obs_img, np.int32)
        self.obs_xy = _dev(obs_xy, np.float64)
        self.fixed = _dev(fixed, np.uint8)
        self.fix_points = int(bool(fix_points))
        self.radial = None if radial is None else _dev(radial, np.float64)
        kc = 1 if radial is None else 2           # columns per camera
        self.ncol = 6 * self.nimg + kc * self.ncam
        dev = self.X.device
        cnt = self.pt_off[1:] - self.pt_off[:-1]
        obs_pt = torch.repeat_interleave(torch.arange(self.P, device=dev), cnt)
        self.obs_pt = obs_pt.int()
        # (o, o') of every point in (point, o, o') order
        rep = cnt[obs_pt]
        o1 = torch.repeat_interleave(torch.arange(self.n, device=dev), rep)
        first = torch.cumsum(rep, 0) - rep
        o2 = self.pt_off[obs_pt[o1]] + (torch.arange(o1.shape[0], device=dev) - first[o1])
        pb = self.obs_img.long()
        cb = self.nimg + self.img_cam.long()[pb]
        nblk = self.nimg + self.ncam
        keys = torch.cat([pb[o1] * nblk + pb[o2], pb[o1] * nblk + cb[o2], cb[o1] * nblk + pb[o2], cb[o1] * nblk + cb[o2]])
        ent = torch.stack([o1, o2], 1).repeat(4, 1)
        keys, order = torch.sort(keys, stable=True)
        self.ent = ent[order].int().contiguous()
        ukey, counts = torch.unique_consecutive(keys, return_counts=True)
        self.seg_key = torch.stack([ukey // nblk, ukey % nblk], 1).int().contiguous()
        self.chunk, self.chunk_key, self.seg_chunk = _chunks(counts, self.seg_key)
        oi = torch.arange(self.n, device=dev)
        rkeys = torch.cat([pb, cb])
        rkeys, rorder = torch.sort(rkeys, stable=True)
        self.obs_seg = torch.stack([torch.cat([oi, oi]), torch.cat([pb, cb])], 1)[rorder].int().contiguous()
        rblk, rcounts = torch.unique_consecutive(rkeys, return_counts=True)
        self.rseg_blk = rblk.int().contiguous()
        self.rchunk, self.rchunk_blk, self.rseg_chunk = _chunks(rcounts, self.rseg_blk)
        f64 = dict(dtype=torch.float64, device=dev)
        self.res = torch.empty(self.n, 2, **f64)
        self.Jc = torch.empty(self.n, 2, 6 + kc, **f64)
        self.Jp = torch.empty(self.n, 2, 3, **f64)
        self.Y = torch.empty(self.n, 6 + kc, 3, **f64)
        self.Vinv = torch.empty(self.P, 9, **f64)
        self.gp = torch.empty(self.P, 3, **f64)
        self.partial = torch.empty(-(-self.P // 256), **f64)
        self.cost_buf = torch.empty(1, **f64)
        self.spartial = torch.empty(max(self.chunk.shape[0], 1), 36, **f64)
        self.bpartial = torch.empty(max(self.rchunk.shape[0], 1), 6, **f64)

    def cost(self, pose=None, focal=None, X=None, radial=None):
        ops = _ops()
        pose, focal, X = self.pose if pose is None else pose, self.focal if focal is None else focal, self.X if X is None else X
        if self.radial is None:
            ops.K('nero_sfm_ba_cost', self.pt_off, self.P, self.obs_img, self.obs_xy, pose, self.img_cam, focal, self.pp, X, self.partial,
                  self.cost_buf, launches=2)
        else:
            ops.K('nero_sfm_radial_ba_cost', self.pt_off, self.P, self.obs_img, self.obs_xy, pose, self.img_cam, focal, self.pp,
                  self.radial if radial is None else radial, X, self.partial, self.cost_buf, launches=2)
        return float(self.cost_buf.item())

    def linearize(self):
        if self.radial is None:
            _ops().K('nero_sfm_ba_linearize', self.pt_off, self.P, self.obs_img, self.obs_xy, self.pose, self.img_cam, self.focal, self.pp,
                     self.X, self.res, self.Jc, self.Jp)
        else:
            _ops().K('nero_sfm_radial_ba_linearize', self.pt_off, self.P, self.obs_img, self.obs_xy, self.pose, self.img_cam, self.focal,
                     self.pp, self.radial, self.X, self.res, self.Jc, self.Jp)

    def eliminate(self, lam):
        _ops().K('nero_sfm_ba_points' if self.radial is None else 'nero_sfm_radial_ba_points', self.pt_off, self.P, self.res, self.Jc,
                 self.Jp, float(lam), self.fix_points, self.Vinv, self.gp, self.Y)

    def reduce(self, lam):
        torch = _torch()
        S = torch.zeros(self.ncol, self.ncol, dtype=torch.float64, device='cuda')
        b = torch.zeros(self.ncol, dtype=torch.float64, device='cuda')
        _ops().K('nero_sfm_ba_reduce' if self.radial is None else 'nero_sfm_radial_ba_reduce', self.ent, self.chunk, self.chunk_key,
                 self.chunk.shape[0], self.seg_chunk, self.seg_key, self.seg_key.shape[0], self.obs_seg, self.rchunk, self.rchunk_blk,
                 self.rchunk.shape[0], self.rseg_chunk, self.rseg_blk, self.rseg_blk.shape[0], self.obs_pt, self.img_cam, self.nimg, self.ncam, self.Jc, self.Jp, self.res, self.Y, self.gp,
                 float(lam), self.fixed, self.spartial, self.bpartial, S, b, launches=4)
        d = S.diagonal()
        d.copy_(torch.where(d == 0, torch.ones_like(d), d))       # a parameter no observation reaches stays put
        return S, b

    def backsub(self, dc):
        """-> candidate (pose, focal, X), and radial after them for SIMPLE_RADIAL cameras."""
        torch = _torch()
        pose = torch.empty_like(self.pose)
        focal = torch.empty_like(self.focal)
        X = torch.empty_like(self.X)
        if self.radial is None:
            _ops().K('nero_sfm_ba_backsub', self.pt_off, self.P, self.obs_img, self.img_cam, self.nimg, self.ncam, self.Jc, self.Jp, self.Vinv,
                     self.gp, dc.contiguous(), self.pose, self.focal, self.X, pose, focal, X)
            return pose, focal, X
        radial = torch.empty_like(self.radial)
        _ops().K('nero_sfm_radial_ba_backsub', self.pt_off, self.P, self.obs_img, self.img_cam, self.nimg, self.ncam, self.Jc, self.Jp,
                 self.Vinv, self.gp, dc.contiguous(), self.pose, self.focal, self.radial, self.X, pose, focal, radial, X)
        return pose, focal, X, radial

    def step(self, lam):
        """One damped step from the current linearisation -> the candidate of backsub or None when S is not positive
        definite."""
        torch = _torch()
        self.eliminate(lam)
        S, b = self.reduce(lam)
        L, info = torch.linalg.cholesky_ex(S)
        if int(info.item()) != 0:
            return None
        dc = torch.cholesky_solve(b[:, None], L)[:, 0]
        return self.backsub(dc)

    def solve(self, iterations, tol=BA_TOL, lam=LAMBDA0):
        """Levenberg-Marquardt: at most `iterations` linearisations -> dict(cost0, cost, iterations, accepted)."""
        c0 = cost = self.cost()
        it = acc = 0
        while it < iterations and cost > 0:
            it += 1
            self.linearize()
            while lam <= 1e12:
                cand = self.step(lam)
                new = self.cost(*cand) if cand is not None else math.inf
                if new < cost:
                    self.pose, self.focal, self.X = cand[:3]
                    if self.radial is not None:
                        self.radial = cand[3]
                    lam = max(lam / 10, 1e-12)
                    acc += 1
                    break
                lam *= 10
            else:
                break
            done = cost - new <= tol * cost
            cost = new
            if done:
                break
        return dict(cost0=c0, cost=cost, iterations=it, accepted=acc, lam=lam)

    def result(self):
        return self.pose.cpu().numpy(), self.focal.cpu().numpy(), self.X.cpu().numpy()


# ------------------------------------------------------------------------------------------------ the mapper
def _qvec(R):
    """Unit quaternion (w, x, y, z), w >= 0, of a rotation matrix (the largest of the four diagonal forms)."""
    t = np.trace(R)
    c = [t, R[0, 0], R[1, 1], R[2, 2]]
    k = int(np.argmax(c))
    if k == 0:
        s = 2.0 * math.sqrt(1.0 + t)
        q = np.array([s / 4, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    elif k == 1:
        s = 2.0 * math.sqrt(max(1.0 + R[0, 0] - R[1, 1] - R[2, 2], 1e-300))
        q = np.array([(R[2, 1] - R[1, 2]) / s, s / 4, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    elif k == 2:
        s = 2.0 * math.sqrt(max(1.0 + R[1, 1] - R[0, 0] - R[2, 2], 1e-300))
        q = np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, s / 4, (R[1, 2] + R[2, 1]) / s])
    else:
        s = 2.0 * math.sqrt(max(1.0 + R[2, 2] - R[0, 0] - R[1, 1], 1e-300))
        q = np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, s / 4])
    q = q / np.linalg.norm(q)
    return q if q[0] >= 0 else -q


def _orthonormal(R):
    U, _, Vt = np.linalg.svd(R)
    R = U @ Vt
    return R if np.linalg.det(R) > 0 else -R


def essential_poses(E):
    """The four (R, t) of an essential matrix (|t| = 1)."""
    U, _, Vt = np.linalg.svd(E)
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(Vt) < 0:
        Vt = -Vt
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    R1, R2, t = U @ W @ Vt, U @ W.T @ Vt, U[:, 2]
    return [(R1, t), (R1, -t), (R2, t), (R2, -t)]


class Mapper:
    """The state of one reconstruction: tracks, registered images, points."""

    def __init__(self, db, log=None, camera_model='SIMPLE_PINHOLE'):
        self.log = log or (lambda s: None)
        self.times = dict(tracks=0.0, init=0.0, register=0.0, triangulate=0.0, bundle=0.0)
        self.db = db
        self.ids = largest_component(sorted(db['images']), db['pairs'])
        if len(self.ids) > MAX_IMAGES:
            raise ValueError(f'{len(self.ids)} connected images: the mapper reconstructs at most {MAX_IMAGES}')
        slot = {iid: k for k, iid in enumerate(self.ids)}
        self.slot = slot
        n_img = len(self.ids)
        self.cam_ids = sorted({db['images'][i][1] for i in self.ids})
        cslot = {c: k for k, c in enumerate(self.cam_ids)}
        self.img_cam = np.array([cslot[db['images'][i][1]] for i in self.ids], np.int64)
        self.focal = np.array([db['cameras'][c][3][0] for c in self.cam_ids], np.float64)
        self.pp = np.array([db['cameras'][c][3][1:3] for c in self.cam_ids], np.float64)
        # k per camera for SIMPLE_RADIAL, None for the pinhole mapper
        self.radial = np.array([db['cameras'][c][3][3] for c in self.cam_ids], np.float64) if camera_model == 'SIMPLE_RADIAL' else None
        self.pairs = {(a, b): v for (a, b), v in db['pairs'].items() if a in slot and b in slot}
        t0 = time.time()
        self._tracks()
        self.node_und = self.node_xy if self.radial is None else self.node_xy.copy()
        self.node_ok = np.ones(self.N, bool)
        self._undistort(np.arange(len(self.cam_ids)))
        self.times['tracks'] = time.time() - t0
        self.pose = np.zeros((n_img, 12))
        self.reg = np.zeros(n_img, bool)
        self.order = []
        self.has_pt = np.zeros(self.T, bool)
        self.Xt = np.zeros((self.T, 3))
        self.active = np.zeros(self.N, bool)

    # -------------------------------------------------------------------------------------------- tracks
    def _tracks(self):
        kp = self.db['keypoints']
        used = {i: np.zeros(kp[i].shape[0] if i in kp else 0, bool) for i in self.ids}
        for (a, b), (m, _) in self.pairs.items():
            used[a][m[:, 0]] = True
            used[b][m[:, 1]] = True
        base, n = {}, 0
        rank = {}
        node_img, node_kp = [], []
        for i in self.ids:
            k = np.nonzero(used[i])[0]
            r = np.full(used[i].shape[0], -1, np.int64)
            r[k] = n + np.arange(k.shape[0])
            rank[i] = r
            node_img.append(np.full(k.shape[0], self.slot[i], np.int64))
            node_kp.append(k)
            n += k.shape[0]
        self.N = n
        self.node_img = np.concatenate(node_img)
        self.node_kp = np.concatenate(node_kp)
        self.node_xy = np.concatenate([kp[i][used[i]] for i in self.ids], 0).reshape(-1, 2)
        edges = np.concatenate([np.stack([rank[a][m[:, 0]], rank[b][m[:, 1]]], 1) for (a, b), (m, _) in sorted(self.pairs.items())], 0)
        self.node_of = rank
        _, track, T = build_tracks(edges, n)
        # a track with two keypoints in one image is dropped; nodes of a track are in node order, so in image order
        order = np.lexsort((np.arange(n), track))
        ts, im = track[order], self.node_img[order]
        dup = np.zeros(T, bool)
        same = (ts[1:] == ts[:-1]) & (im[1:] == im[:-1])
        dup[ts[1:][same]] = True
        self.dropped = int(dup.sum())
        keep_t = np.nonzero(~dup)[0]
        remap = np.full(T, -1, np.int64)
        remap[keep_t] = np.arange(keep_t.shape[0])
        self.track = remap[track]
        self.T = keep_t.shape[0]
        order = np.lexsort((np.arange(n), self.track))
        order = order[self.track[order] >= 0]
        self.tnodes = order
        self.toff = np.concatenate([[0], np.cumsum(np.bincount(self.track[order], minlength=self.T))]).astype(np.int64)
        self.log(f'tracks: {n} nodes, {edges.shape[0]} edges, {self.T} tracks ({self.dropped} dropped: two keypoints in one image)')

    def _track_nodes(self, t):
        return self.tnodes[self.toff[t]:self.toff[t + 1]]

    # -------------------------------------------------------------------------------------------- camera model
    def _undistort(self, cams):
        """SIMPLE_RADIAL: the keypoints of cameras `cams` undistorted with their current (f, k) into pinhole pixels
        f x + (cx, cy) (node_und), and whether each is invertible (node_ok).  P3P and the DLT take these; the pinhole
        mapper gives them the keypoints as they are."""
        if self.radial is None:
            return
        from . import undistort
        node_cam = self.img_cam[self.node_img]
        for c in cams:
            sel = np.nonzero(node_cam == c)[0]
            if sel.shape[0]:
                xn, ok = undistort.points(self.node_xy[sel], self.focal[c], self.pp[c, 0], self.pp[c, 1], self.radial[c])
                self.node_und[sel] = self.focal[c] * xn.cpu().numpy() + self.pp[c]
                self.node_ok[sel] = ok.cpu().numpy()

    def _reprojection(self, off, nodes, X):
        """(depth, reprojection error px) of the nodes and the largest ray angle of each point, measured through the camera
        model in the image the keypoints come from."""
        return reprojection(off, self.node_img[nodes], self.node_xy[nodes], self.pose, self.img_cam, self.focal, self.pp, X, self.radial)

    # -------------------------------------------------------------------------------------------- helpers
    def _obs_lists(self, tracks, nodes_of):
        """(off [T + 1], nodes) of the given tracks with nodes_of(t) -> their selected nodes."""
        sel = [nodes_of(t) for t in tracks]
        off = np.concatenate([[0], np.cumsum([s.shape[0] for s in sel])]).astype(np.int64)
        nodes = np.concatenate(sel) if sel else np.zeros(0, np.int64)
        return off, nodes.astype(np.int64)

    def _points(self, registered_only=True):
        """Point-ordered observation list of the current model: (tracks, pt_off, nodes)."""
        ok = self.active & self.reg[self.node_img] if registered_only else self.active
        nodes = self.tnodes[ok[self.tnodes] & self.has_pt[self.track[self.tnodes]]]
        tr = self.track[nodes]
        tracks, cnt = np.unique(tr, return_counts=True)
        off = np.concatenate([[0], np.cumsum(cnt)]).astype(np.int64)
        return tracks, off, nodes

    def problem(self, images=None, fix_points=False, nodes_pt=None):
        """The bundle-adjustment Problem of the registered images (or `images`) and the points, with the mapper's gauge
        and focal rule -> (problem, image slots, camera slots, tracks), or None without observations."""
        imgs = np.nonzero(self.reg)[0] if images is None else np.asarray(images)
        if nodes_pt is None:
            tracks, off, nodes = self._points()
        else:
            tracks, off, nodes = nodes_pt
        if nodes.shape[0] == 0:
            return None
        islot = np.full(self.reg.shape[0], -1, np.int64)
        islot[imgs] = np.arange(imgs.shape[0])
        cams = np.unique(self.img_cam[imgs])
        cslot = np.full(self.focal.shape[0], -1, np.int64)
        cslot[cams] = np.arange(cams.shape[0])
        nimg, ncam = imgs.shape[0], cams.shape[0]
        fixed = np.zeros(6 * nimg + (1 if self.radial is None else 2) * ncam, np.uint8)
        if images is None:
            g0, g1 = self.order[0], self.order[1]
            fixed[6 * islot[g0]:6 * islot[g0] + 6] = 1
            fixed[6 * islot[g1] + 3 + int(np.argmax(np.abs(self.pose[g1, 9:])))] = 1
        if self.reg.sum() < FOCAL_MIN_IMAGES:
            fixed[6 * nimg:] = 1                                  # the focal, and k of SIMPLE_RADIAL
        pr = Problem(self.pose[imgs], self.focal[cams], self.pp[cams], cslot[self.img_cam[imgs]], self.Xt[tracks], off,
                     islot[self.node_img[nodes]], self.node_xy[nodes], fixed, fix_points,
                     None if self.radial is None else self.radial[cams])
        return pr, imgs, cams, tracks

    def _bundle(self, iterations, images=None, fix_points=False, nodes_pt=None):
        """Adjust the registered images (or `images`) and the points; with fix_points the points stay put."""
        t0 = time.time()
        built = self.problem(images, fix_points, nodes_pt)
        if built is None:
            return None
        pr, imgs, cams, tracks = built
        nimg = imgs.shape[0]
        info = pr.solve(iterations)
        pose, focal, X = pr.result()
        for k in range(nimg):
            pose[k, :9] = _orthonormal(pose[k, :9].reshape(3, 3)).reshape(-1)
        self.pose[imgs] = pose
        if self.radial is not None:
            k = pr.radial.cpu().numpy()
            changed = cams[(focal != self.focal[cams]) | (k != self.radial[cams])]
            self.radial[cams] = k
        self.focal[cams] = focal
        if self.radial is not None:
            self._undistort(changed)
        if not fix_points:
            self.Xt[tracks] = X
        self.times['bundle'] += time.time() - t0
        info.update(observations=int(pr.n), points=int(tracks.shape[0]), images=int(nimg))
        return info

    def _filter(self):
        """Drop observations beyond MAX_REPROJ px (or behind the camera), then points with < 2 observations or a largest
        ray angle < MIN_TRI_ANGLE."""
        tracks, off, nodes = self._points()
        if nodes.shape[0] == 0:
            return
        err, _ = self._reprojection(off, nodes, self.Xt[tracks])
        bad = (err[:, 0] <= 0) | (err[:, 1] > MAX_REPROJ)
        self.active[nodes[bad]] = False
        tracks, off, nodes = self._points()
        _, ang = self._reprojection(off, nodes, self.Xt[tracks])
        drop = (np.diff(off) < 2) | (ang < math.radians(MIN_TRI_ANGLE))
        for t in tracks[drop]:
            self.has_pt[t] = False
            self.active[self._track_nodes(t)] = False

    def _triangulate(self, tracks, min_angle=MIN_TRI_ANGLE, max_err=MAX_REPROJ):
        """Triangulate the tracks from their registered observations (SIMPLE_RADIAL: the invertible ones, undistorted);
        keep the good ones.  -> number kept."""
        t0 = time.time()
        tracks = [t for t in tracks if not self.has_pt[t]]
        sel = lambda t: (lambda nd: nd[self.reg[self.node_img[nd]] & self.node_ok[nd]])(self._track_nodes(t))
        tracks = [t for t in tracks if sel(t).shape[0] >= 2]
        off, nodes = self._obs_lists(tracks, sel)
        X, st = triangulate(off, self.node_img[nodes], self.node_und[nodes], self.pose, self.img_cam, self.focal, self.pp)
        if self.radial is not None and tracks:        # judged in the distorted image, not by the DLT's pinhole pixels
            err, ang = self._reprojection(off, nodes, X)
            st = np.stack([np.minimum.reduceat(err[:, 0], off[:-1]), np.maximum.reduceat(err[:, 1], off[:-1]), ang], 1)
        ok = (st[:, 0] > 0) & (st[:, 1] <= max_err) & (st[:, 2] >= math.radians(min_angle)) & np.isfinite(X).all(1)
        for k in np.nonzero(ok)[0]:
            t = tracks[k]
            self.has_pt[t] = True
            self.Xt[t] = X[k]
            self.active[nodes[off[k]:off[k + 1]]] = True
        self.times['triangulate'] += time.time() - t0
        return int(ok.sum())

    def _tracks_of_image(self, i):
        nd = np.nonzero(self.node_img == i)[0]
        t = self.track[nd]
        return nd[t >= 0], t[t >= 0]

    # -------------------------------------------------------------------------------------------- initial pair
    def _reset(self):
        self.reg[:] = False
        self.order = []
        self.has_pt[:] = False
        self.active[:] = False
        self.pose[:] = 0

    def initialize(self):
        t0 = time.time()
        K = lambda i: np.array([[self.focal[self.img_cam[i]], 0, self.pp[self.img_cam[i], 0]],
                                [0, self.focal[self.img_cam[i]], self.pp[self.img_cam[i], 1]], [0, 0, 1]])
        cands = sorted(self.pairs, key=lambda ab: (-self.pairs[ab][0].shape[0], Ft.pair_id(*ab)))[:INIT_TRIES]
        for a, b in cands:
            i, j = self.slot[a], self.slot[b]
            ni, ti = self._tracks_of_image(i)
            nj, tj = self._tracks_of_image(j)
            common = np.intersect1d(ti, tj)
            if common.shape[0] < INIT_MIN_POINTS:
                continue
            E = K(j).T @ self.pairs[a, b][1] @ K(i)
            self._reset()
            self.reg[[i, j]] = True
            self.order = [i, j]
            sel = lambda t: (lambda nd: nd[((self.node_img[nd] == i) | (self.node_img[nd] == j)) & self.node_ok[nd]])(self._track_nodes(t))
            if self.radial is not None:
                common = np.asarray([t for t in common if sel(t).shape[0] == 2], np.int64)
            off, nodes = self._obs_lists(common, sel)
            best = None
            for R, t in essential_poses(E):
                self.pose[i] = np.concatenate([np.eye(3).reshape(-1), np.zeros(3)])
                self.pose[j] = np.concatenate([R.reshape(-1), t])
                _, st = triangulate(off, self.node_img[nodes], self.node_und[nodes], self.pose, self.img_cam, self.focal, self.pp)
                front = int((st[:, 0] > 0).sum())
                if best is None or front > best[0]:
                    best = (front, R, t)
            self.pose[j] = np.concatenate([best[1].reshape(-1), best[2]])
            n0 = self._triangulate(common, min_angle=0.0, max_err=np.inf)
            self._bundle(INIT_BA_ITERS)
            self._filter()
            tracks, off, nodes = self._points()
            ang = self._reprojection(off, nodes, self.Xt[tracks])[1]
            med = math.degrees(float(np.median(ang))) if ang.shape[0] else 0.0
            self.log(f'initial pair {a}, {b}: {self.pairs[a, b][0].shape[0]} inliers, {n0} triangulated, {tracks.shape[0]} points after '
                     f'the two-view adjustment, median angle {med:.1f} deg')
            if tracks.shape[0] >= INIT_MIN_POINTS and med >= INIT_MIN_TRI_ANGLE:
                self.times['init'] = time.time() - t0
                return a, b
        self._reset()
        raise RuntimeError(f'no initial pair: none of the {len(cands)} best verified pairs gives {INIT_MIN_POINTS} points with a '
                           f'median triangulation angle >= {INIT_MIN_TRI_ANGLE} deg')

    # -------------------------------------------------------------------------------------------- registration
    def _correspondences(self, i):
        nd, t = self._tracks_of_image(i)
        ok = self.has_pt[t] & self.node_ok[nd]
        return nd[ok], t[ok]

    def register(self, i):
        """P3P RANSAC, then pose (and focal) refinement on the inliers.  -> (accepted, inliers, correspondences)."""
        t0 = time.time()
        nd, t = self._correspondences(i)
        n = nd.shape[0]
        if n < max(3, ABS_POSE_MIN_INLIERS):
            self.times['register'] += time.time() - t0
            return False, 0, n
        c = self.img_cam[i]
        pose, _, cnt, inl, _ = p3p_ransac(self.node_und[nd], self.Xt[t], self.focal[c], self.pp[c, 0], self.pp[c, 1], self.ids[i])
        if cnt < ABS_POSE_MIN_INLIERS or cnt < ABS_POSE_MIN_RATIO * n:
            self.times['register'] += time.time() - t0
            return False, cnt, n
        pose[:9] = _orthonormal(pose[:9].reshape(3, 3)).reshape(-1)
        self.pose[i] = pose
        self.reg[i] = True
        self.order.append(i)
        # pose (and focal) refinement with the points held: each inlier its own one-observation point
        nin = nd[inl]
        self._bundle(REFINE_ITERS, images=[i], fix_points=True,
                     nodes_pt=(t[inl], np.arange(nin.shape[0] + 1, dtype=np.int64), nin))
        self.times['register'] += time.time() - t0
        return True, cnt, n

    def extend(self, i):
        """After registering image i: continue its tracks that have points, triangulate the others."""
        t0 = time.time()
        nd, t = self._tracks_of_image(i)
        hp = self.has_pt[t]
        cont = 0
        if hp.any():
            nd1, t1 = nd[hp], t[hp]
            off = np.arange(nd1.shape[0] + 1, dtype=np.int64)
            err, _ = self._reprojection(off, nd1, self.Xt[t1])
            good = (err[:, 0] > 0) & (err[:, 1] <= MAX_REPROJ)
            self.active[nd1[good]] = True
            cont = int(good.sum())
        self.times['triangulate'] += time.time() - t0
        new = self._triangulate(t[~hp])
        return cont, new

    def run(self):
        a, b = self.initialize()
        self.log(f'initial pair: images {a} and {b}, {int(self.has_pt.sum())} points')
        failed = np.zeros(self.reg.shape[0], bool)
        while True:
            cand = np.nonzero(~self.reg & ~failed)[0]
            if cand.shape[0] == 0:
                break
            vis = np.zeros(self.reg.shape[0], np.int64)
            sel = self.has_pt[np.maximum(self.track, 0)] & (self.track >= 0)
            np.add.at(vis, self.node_img[sel], 1)
            i = int(cand[np.argmax(vis[cand])])               # the first of the most: lower slot = lower image id
            ok, cnt, n = self.register(i)
            if not ok:
                failed[i] = True
                self.log(f'image {self.ids[i]}: not registered ({cnt} of {n} correspondences are P3P inliers)')
                continue
            cont, new = self.extend(i)
            info = self._bundle(GLOBAL_BA_ITERS)
            self._filter()
            failed[:] = False
            self.log(f'image {self.ids[i]}: registered with {cnt} of {n} inliers, {cont} observations added, {new} new points; '
                     f'{int(self.reg.sum())} images, {int(self.has_pt.sum())} points, rms {math.sqrt(info["cost"] / max(info["observations"], 1)):.3f} px')
        info = self._bundle(FINAL_BA_ITERS)
        self._filter()
        self.final_ba = info
        return self

    # -------------------------------------------------------------------------------------------- model
    def model(self, image_dir=None):
        """(cameras, images, points, summary) of the reconstruction in the form objprep.write_colmap_model takes.  A
        SIMPLE_RADIAL camera that undistort.camera would refuse is still written; its message goes to summary['warnings']."""
        from . import mvs, undistort
        db = self.db
        tracks, off, nodes = self._points()
        err, _ = self._reprojection(off, nodes, self.Xt[tracks])
        regs = np.nonzero(self.reg)[0]
        cams = {}
        warnings = []
        for c in sorted({int(self.img_cam[i]) for i in regs}):
            cid = self.cam_ids[c]
            _, w, h, _ = db['cameras'][cid]
            par = [float(self.focal[c]), float(self.pp[c, 0]), float(self.pp[c, 1])]
            if self.radial is None:
                cams[cid] = ('SIMPLE_PINHOLE', w, h, par)
                continue
            cams[cid] = ('SIMPLE_RADIAL', w, h, par + [float(self.radial[c])])
            try:
                undistort.camera(w, h, *cams[cid][3], name=f'camera {cid}')
            except ValueError as e:                      # the model is still written; undistort_images.py will refuse it
                warnings.append(str(e))
        pid = np.full(self.T, -1, np.int64)
        pid[tracks] = np.arange(1, tracks.shape[0] + 1)
        rgb_sum = np.zeros((tracks.shape[0], 3), np.int64)
        pt_of_node = np.repeat(np.arange(tracks.shape[0]), np.diff(off))
        images = {}
        for i in regs:
            iid = self.ids[i]
            name, cid = db['images'][iid]
            xys = db['keypoints'].get(iid, np.zeros((0, 2)))
            p3d = np.full(xys.shape[0], -1, np.int64)
            mine = self.node_img[nodes] == i
            p3d[self.node_kp[nodes[mine]]] = pid[self.track[nodes[mine]]]
            R = self.pose[i, :9].reshape(3, 3)
            images[iid] = (_qvec(R), self.pose[i, 9:].copy(), cid, name, xys, p3d)
            if image_dir is not None and mine.any():
                rgb = mvs.read_rgb(os.path.join(image_dir, name))
                h, w = rgb.shape[:2]
                xy = self.node_xy[nodes[mine]]
                px = rgb[np.clip(np.floor(xy[:, 1]).astype(np.int64), 0, h - 1), np.clip(np.floor(xy[:, 0]).astype(np.int64), 0, w - 1)]
                np.add.at(rgb_sum, pt_of_node[mine], px.astype(np.int64))
        cnt = np.diff(off)
        rgb = np.floor(rgb_sum / np.maximum(cnt, 1)[:, None] + 0.5).astype(np.int64) if image_dir is not None else np.zeros_like(rgb_sum)
        perr = np.add.reduceat(err[:, 1], off[:-1]) / np.maximum(cnt, 1) if nodes.shape[0] else np.zeros(0)
        points = {}
        for k, t in enumerate(tracks):
            nd = nodes[off[k]:off[k + 1]]
            points[k + 1] = (self.Xt[t].copy(), [int(v) for v in rgb[k]], float(perr[k]),
                             [self.ids[i] for i in self.node_img[nd]], [int(v) for v in self.node_kp[nd]])
        summary = dict(registered=[self.ids[i] for i in regs], unregistered=[iid for iid in sorted(db['images']) if iid not in images],
                       points=int(tracks.shape[0]), mean_track=float(cnt.mean()) if cnt.shape[0] else 0.0,
                       mean_error=float(err[:, 1].mean()) if err.shape[0] else 0.0,
                       focals={cid: p[3][0] for cid, p in cams.items()}, dropped_tracks=self.dropped, times=dict(self.times))
        if self.radial is not None:
            summary.update(radial={cid: p[3][3] for cid, p in cams.items()}, warnings=warnings)
        return cams, images, points, summary


def map_sparse(db_path, output, image_dir=None, log=None, camera_model='SIMPLE_PINHOLE'):
    """The whole tool: read the database, reconstruct, write <output>/{cameras,images,points3D}.bin.  -> summary."""
    t0 = time.time()
    db = read_database(db_path)
    check_database(db, camera_model)
    t1 = time.time()
    mp = Mapper(db, log, camera_model).run()
    cams, images, points, summary = mp.model(image_dir)
    t2 = time.time()
    objprep.write_colmap_model(output, cams, images, points)
    summary['times'].update(read=t1 - t0, mapper=t2 - t1, write=time.time() - t2, total=time.time() - t0)
    summary['final_ba'] = mp.final_ba
    summary['names'] = {iid: db['images'][iid][0] for iid in db['images']}
    return summary
