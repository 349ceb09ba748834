"""Sparse features on the GPU: SIFT extraction, all-pair matching and two-view verification of a custom object's images,
written as the COLMAP database that nero_b200.sfm (tools/map_sparse.py) or `colmap mapper` reconstructs from, without
COLMAP's feature_extractor or exhaustive_matcher.

Reference being replaced (paths relative to the reference repository):
  run_colmap.py:12-39   database.db with one SIMPLE_PINHOLE camera per image (or one shared camera with --same_camera)
  run_colmap.py:41-53   colmap feature_extractor and colmap exhaustive_matcher
What the mapper then reads is the same: cameras, images, keypoints, descriptors, matches and two-view geometries in
COLMAP's schema.  The features are SIFT in spirit and are not pinned to COLMAP's (DESIGN.md section 2).

The protocol (k_sift.cu, k_match.cu, k_verify.cu, include/nero_features.h):
  * Images.  The files matching *.jpg, *.png, *.PNG, *.JPG of the image directory (in that pattern order, then sorted
    by path) get image ids 1..n.  Pixels are read in their stored order (mvs.read_rgb ignores an EXIF orientation), as
    run_colmap.py's skimage reader and COLMAP read them, so sizes, cameras and keypoints share COLMAP's frame.  Each image gets the camera SIMPLE_PINHOLE (f, w / 2, h / 2) with f = sqrt(w^2 + h^2)
    and prior_focal_length = 1; with same_camera the first image's camera (id 1) serves every image.  With
    camera_model='SIMPLE_RADIAL' the camera is SIMPLE_RADIAL (f, w / 2, h / 2, 0) with the same prior, for a mapper that
    estimates k (COLMAP's); undistort.py then resamples the images.
  * Grey image.  mvs.prepare_grey (nero_mvs_grey) with s = ceil(max(w, h) / max_size): integer luma block-averaged over
    s x s.  Grey pixel p has its centre at image point (p + 1/2) s.
  * Scale space.  OCTAVES octaves of SCALES + 3 Gaussian levels; octave 0 is the grey image itself (COLMAP upsamples
    first).  Level 0 of octave 0 is the grey image blurred by sqrt(SIGMA0^2 - CAMERA_BLUR^2); level l >= 1 is level l - 1
    blurred by SIGMA0 sqrt(k^(2l) - k^(2l - 2)), k = 2^(1 / SCALES); level 0 of octave o > 0 is level SCALES of octave
    o - 1 decimated (sample (x, y) = (2x, 2y)).  An octave smaller than 2 BORDER + 3 samples is not built.  A blur of sigma
    has radius r = min(ceil(4 sigma), 32) and the fp32 taps t_k = g_k / (g_0 + 2 sum g_k), g_k = exp(-k^2 / (2 sigma^2))
    in fp64; each pass (rows, then columns, clamp to edge) computes acc = t0 x0, then acc + t_k (x_-k + x_+k) for k = 1..r,
    every operation rounded.  DoG level l = G[l + 1] - G[l].
  * Candidates.  Samples of DoG levels 1..SCALES at least BORDER from the edges with |D| > PRE_PEAK PEAK and D strictly
    above or below its 26 neighbours, in (octave, level, row, column) order (count -> block_offsets -> emit).
  * Refinement (fp64).  Central differences give the gradient and Hessian in (x, y, level); the offset -H^-1 g moves the
    sample by one in x and y where it exceeds 0.6, at most 5 times.  A keypoint is kept when every offset is < 1.5, the
    interpolated |D| >= PEAK and tr^2 / det < (EDGE + 1)^2 / EDGE for the 2 x 2 spatial Hessian (det > 0).  Its sigma is
    SIGMA0 2^(level / SCALES) octave samples at the fractional level.
  * Selection.  The kept keypoints of all octaves are ordered by |D| descending, ties in candidate order; the first
    max_features are described.
  * Orientation.  A 36-bin histogram of the gradient angles (central differences) of Gaussian level l within radius
    3 (1.5 sigma), weighted by magnitude and a Gaussian of sigma 1.5 sigma, smoothed six times by a circular [1 1 1] / 3;
    up to 2 local peaks >= 0.8 of the maximum, highest first, each refined by a parabola.  Each one is a feature.
  * Descriptor.  A 4 x 4 spatial x 8 angular histogram over bins of 3 sigma rotated to the orientation, trilinear, with
    a Gaussian window of half the descriptor width; L2-normalised, clamped at 0.2, L2-normalised, then RootSIFT (L1
    normalise and square root) and uint8 = min(255, floor(512 v + 1/2)).  Layout (row bin, column bin, angle bin).
  * Features of an image.  In selection order, each keypoint's orientations in peak order, truncated to max_features.
    Keypoint rows are COLMAP's affine form (x, y, a11, a12, a21, a22) = (u s, v s, c cos t, -c sin t, c sin t, c cos t)
    with (u, v) the grey image point, c the scale in image pixels and t the orientation.
  * Matching.  For every pair i < j both directions run as tiles of one launch: each row's nearest and second-nearest
    descriptor of the other image by exact integer squared distance (ties to the lower index).  Row r of i matches
    column c of j when 25 d1 < 16 d2 (ratio 0.8), d1 <= MAX_D1 and r is also c's nearest row.  Matches of a pair are in
    row order.  |d|^2 of every descriptor is one int32 torch reduction.  The pairs run in batches of consecutive pairs
    whose row-best records fit MATCH_ROWS (match_batches), one matcher launch per batch, so every offset fits int32.
  * Verification (fp64).  Per pair with matches (x1, y1, x2, y2 in image pixels), HYPOTHESES 8-point fundamental matrices
    on Hartley-normalised points (centroid, mean distance sqrt 2), each from 8 distinct matches: draw d of hypothesis h
    takes match mix(mix(mix(mix(SEED 0x9e3779b9 + 0x7f4a7c15) ^ pair) ^ h) ^ d) mod n (mix = rl_mix of hash.cuh; pair =
    the index in the list of pairs with matches), duplicates are redrawn, at most 64 draws.  The null vector comes from
    12 cyclic Jacobi sweeps of the 9 x 9 normal matrix (summed in draw order), the rank 2 from 8 sweeps on F^T F; F is
    denormalised, scaled to unit norm with its largest |entry| positive.  Inliers have (x2^T F x1)^2 <= MAX_ERROR^2
    ((F x1)_0^2 + (F x1)_1^2 + (F^T x2)_0^2 + (F^T x2)_1^2).  The largest count wins, ties to the lower hypothesis; it is
    refit once on its inliers (summed in match order), and the refit's inliers are final.  A pair with >= MIN_INLIERS
    of them is verified: config 3 (UNCALIBRATED), F, E = K_j^T F K_i from the guessed K, H = 0, qvec (1, 0, 0, 0), tvec 0.
  * Database.  COLMAP's schema; blobs are the arrays' bytes: params fp64, keypoints fp32 [n, 6], descriptors uint8
    [n, 128], matches uint32 [m, 2] under pair_id = id1 2147483647 + id2 (id1 < id2), geometries fp64.
"""
import math
import os
import sqlite3

import numpy as np

from . import mvs

MAX_SIZE = 3200
MAX_FEATURES = 8192
OCTAVES = 4
SCALES = 3
SIGMA0 = 1.6
CAMERA_BLUR = 0.5
PEAK = 0.02 / SCALES
PRE_PEAK = 0.8
EDGE = 10.0
BORDER = 5               # NERO_FEATURES_BORDER
RATIO = (16, 25)         # 25 d1 < 16 d2: distance ratio 0.8
MAX_D1 = 128450          # floor(0.49 512^2): distance 0.7 on unit descriptors
HYPOTHESES = 512
MAX_ERROR = 4.0          # px (Sampson)
MIN_INLIERS = 15
SEED = 0
TILE = 128               # NERO_FEATURES_TILE
MATCH_ROWS = 1 << 26     # row-best records (12 B each) per matcher launch
_INT32_MAX = 2 ** 31 - 1
PATTERNS = ('*.jpg', '*.png', '*.PNG', '*.JPG')
SIMPLE_PINHOLE = 0
SIMPLE_RADIAL = 2
CAMERA_MODELS = {'SIMPLE_PINHOLE': SIMPLE_PINHOLE, 'SIMPLE_RADIAL': SIMPLE_RADIAL}   # the models the database may get
UNCALIBRATED = 3
MAX_IMAGE_ID = 2147483647

_KP = 8


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


# ------------------------------------------------------------------------------------------------ host protocol
def pair_id(id1, id2):
    a, b = (int(id1), int(id2)) if id1 < id2 else (int(id2), int(id1))
    return a * MAX_IMAGE_ID + b


def pair_ids(pid):
    b = int(pid) % MAX_IMAGE_ID
    return (int(pid) - b) // MAX_IMAGE_ID, b


def gaussian_taps(sigma):
    """fp32 taps t[0..r] of a Gaussian of `sigma`, r = min(ceil(4 sigma), 32)."""
    r = min(max(1, int(math.ceil(4.0 * sigma))), 32)
    g = np.exp(-np.arange(r + 1, dtype=np.float64) ** 2 / (2.0 * sigma * sigma))
    return (g / (g[0] + 2.0 * g[1:].sum())).astype(np.float32)


def level_sigmas(scales=SCALES, sigma0=SIGMA0, camera_blur=CAMERA_BLUR):
    """The blur that makes each Gaussian level of an octave from the previous one (level 0: from the grey image)."""
    k = 2.0 ** (1.0 / scales)
    return [math.sqrt(sigma0 ** 2 - camera_blur ** 2)] + [sigma0 * math.sqrt(k ** (2 * l) - k ** (2 * l - 2)) for l in range(1, scales + 3)]


def octave_sizes(w, h, octaves=OCTAVES):
    sizes = []
    for _ in range(octaves):
        if min(w, h) < 2 * BORDER + 3:
            break
        sizes.append((w, h))
        w, h = w // 2, h // 2
    return sizes


def list_images(image_dir):
    """Image file names in id order (ids 1..n)."""
    from pathlib import Path
    d = Path(image_dir)
    fns = []
    for pat in PATTERNS:
        fns += list(d.glob(pat))
    return [f.name for f in sorted(fns)]


def image_size(path):
    """(w, h) of an image file as mvs.read_rgb decodes it: the stored pixel grid, EXIF orientation ignored."""
    h, w = mvs.read_rgb(path).shape[:2]
    return w, h


def image_table(image_dir, same_camera=False, camera_model='SIMPLE_PINHOLE'):
    """(names, cameras, camera id of each image) of an image directory, in id order."""
    if not os.path.isdir(image_dir):
        raise FileNotFoundError(f'{image_dir}: no image directory')
    names = list_images(image_dir)
    if not names:
        raise FileNotFoundError(f'{image_dir}: no *.jpg / *.png images')
    cams, cam_of = cameras_for([image_size(os.path.join(image_dir, n)) for n in names], same_camera, camera_model)
    return names, cams, cam_of


def cameras_for(sizes, same_camera=False, camera_model='SIMPLE_PINHOLE'):
    """(cameras, images camera ids) for images of sizes [(w, h)] in id order: camera rows (camera_id, model, width, height,
    params fp64, prior_focal_length).  camera_model: 'SIMPLE_PINHOLE' (f, cx, cy) or 'SIMPLE_RADIAL' (f, cx, cy, k = 0)."""
    if camera_model not in CAMERA_MODELS:
        raise ValueError(f'camera model {camera_model!r}: the database takes SIMPLE_PINHOLE or SIMPLE_RADIAL')
    model, extra = CAMERA_MODELS[camera_model], [0.0] if camera_model == 'SIMPLE_RADIAL' else []
    cams, cam_of = [], []
    for k, (w, h) in enumerate(sizes):
        if not same_camera or k == 0:
            focal = np.sqrt(h ** 2 + w ** 2)
            cams.append((len(cams) + 1, model, int(w), int(h), np.array([focal, w / 2, h / 2] + extra, np.float64), 1))
        cam_of.append(len(cams))
    return cams, cam_of


def camera_K(cam):
    f, cx, cy = cam[4][:3]
    return np.array([[f, 0, cx], [0, f, cy], [0, 0, 1]], np.float64)


_SCHEMA = [
    ('cameras', 'camera_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, model INTEGER NOT NULL, width INTEGER NOT NULL, '
                'height INTEGER NOT NULL, params BLOB, prior_focal_length INTEGER NOT NULL'),
    ('images', 'image_id INTEGER PRIMARY KEY AUTOINCREMENT NOT NULL, name TEXT NOT NULL UNIQUE, camera_id INTEGER NOT NULL, '
               'prior_qw REAL, prior_qx REAL, prior_qy REAL, prior_qz REAL, prior_tx REAL, prior_ty REAL, prior_tz REAL, '
               f'CONSTRAINT image_id_check CHECK(image_id >= 0 and image_id < {MAX_IMAGE_ID}), '
               'FOREIGN KEY(camera_id) REFERENCES cameras(camera_id)'),
    ('keypoints', 'image_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL, cols INTEGER NOT NULL, data BLOB, '
                  'FOREIGN KEY(image_id) REFERENCES images(image_id) ON DELETE CASCADE'),
    ('descriptors', 'image_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL, cols INTEGER NOT NULL, data BLOB, '
                    'FOREIGN KEY(image_id) REFERENCES images(image_id) ON DELETE CASCADE'),
    ('matches', 'pair_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL, cols INTEGER NOT NULL, data BLOB'),
    ('two_view_geometries', 'pair_id INTEGER PRIMARY KEY NOT NULL, rows INTEGER NOT NULL, cols INTEGER NOT NULL, data BLOB, '
                            'config INTEGER NOT NULL, F BLOB, E BLOB, H BLOB, qvec BLOB, tvec BLOB'),
]
TABLES = tuple(t for t, _ in _SCHEMA)


def _blob(a, dtype):
    return np.ascontiguousarray(a, dtype).tobytes()


def write_database(path, images, cameras, keypoints, descriptors, matches, geometries):
    """Write a COLMAP database at `path` (which must not exist).  cameras: rows of cameras_for; images: (image_id, name,
    camera_id); keypoints / descriptors: {image_id: [n, 6] fp32 / [n, 128] uint8}; matches: {(id1, id2): uint32 [m, 2]},
    id1 < id2; geometries: {(id1, id2): dict(matches, config, F, E, H, qvec, tvec)}."""
    if os.path.exists(path):
        raise FileExistsError(f'{path} exists')
    con = sqlite3.connect(path)
    try:
        con.executescript('; '.join(f'CREATE TABLE IF NOT EXISTS {t} ({cols})' for t, cols in _SCHEMA) +
                          '; CREATE UNIQUE INDEX IF NOT EXISTS index_name ON images(name)')
        for cid, model, w, h, params, prior in cameras:
            con.execute('INSERT INTO cameras VALUES (?, ?, ?, ?, ?, ?)', (cid, model, w, h, _blob(params, np.float64), prior))
        for iid, name, cid in images:
            con.execute('INSERT INTO images VALUES (?, ?, ?, ?, ?, ?, ?, ?, ?, ?)', (iid, name, cid) + (None,) * 7)
        for iid in sorted(keypoints):
            k = np.asarray(keypoints[iid], np.float32)
            con.execute('INSERT INTO keypoints VALUES (?, ?, ?, ?)', (iid,) + k.shape + (_blob(k, np.float32),))
        for iid in sorted(descriptors):
            d = np.asarray(descriptors[iid], np.uint8)
            con.execute('INSERT INTO descriptors VALUES (?, ?, ?, ?)', (iid,) + d.shape + (_blob(d, np.uint8),))
        for (a, b) in sorted(matches):
            m = np.asarray(matches[a, b], np.uint32).reshape(-1, 2)
            con.execute('INSERT INTO matches VALUES (?, ?, ?, ?)', (pair_id(a, b),) + m.shape + (_blob(m, np.uint32),))
        for (a, b) in sorted(geometries):
            g = geometries[a, b]
            m = np.asarray(g['matches'], np.uint32).reshape(-1, 2)
            con.execute('INSERT INTO two_view_geometries VALUES (?, ?, ?, ?, ?, ?, ?, ?, ?, ?)',
                        (pair_id(a, b),) + m.shape + (_blob(m, np.uint32), int(g['config'])) +
                        tuple(_blob(g[k], np.float64) for k in ('F', 'E', 'H', 'qvec', 'tvec')))
        con.commit()
    finally:
        con.close()


# ------------------------------------------------------------------------------------------------ GPU steps
def scale_space(grey, octaves=OCTAVES, scales=SCALES):
    """(gauss, dog): per octave CUDA fp32 stacks [scales + 3, h, w] and [scales + 2, h, w] of a CUDA grey image."""
    torch = _torch()
    ops = _ops()
    dev = grey.device
    sig = level_sigmas(scales)
    taps = [torch.from_numpy(gaussian_taps(s)).to(dev) for s in sig]
    h0, w0 = grey.shape
    gauss, dog = [], []
    for o, (w, h) in enumerate(octave_sizes(w0, h0, octaves)):
        G = torch.empty(scales + 3, h, w, dtype=torch.float32, device=dev)
        tmp = torch.empty(h, w, dtype=torch.float32, device=dev)
        if o == 0:
            ops.K('nero_features_blur', grey.contiguous(), w, h, taps[0], taps[0].shape[0] - 1, tmp, G[0], launches=2)
        else:
            P = gauss[-1]
            ops.K('nero_features_decimate', P[scales], P.shape[2], P.shape[1], G[0])
        for l in range(1, scales + 3):
            ops.K('nero_features_blur', G[l - 1], w, h, taps[l], taps[l].shape[0] - 1, tmp, G[l], launches=2)
        D = torch.empty(scales + 2, h, w, dtype=torch.float32, device=dev)
        ops.K('nero_features_dog', G[:-1], G[1:], D.numel(), D)
        gauss.append(G)
        dog.append(D)
    return gauss, dog


def candidates(D, threshold):
    """CUDA int32 [n, 3] (x, y, level) of one octave's DoG stack."""
    torch = _torch()
    ops = _ops()
    L, h, w = D.shape
    nblk = -(-(L - 2) * h * w // 128)
    dev = D.device
    cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
    off = torch.empty(nblk, dtype=torch.int64, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    cap = 1 << 16
    while True:
        cand = torch.empty(cap, 3, dtype=torch.int32, device=dev)
        ops.K('nero_features_extrema', D, w, h, L, float(threshold), cnt, off, total, cand, cap, launches=3)
        n = int(total.item())
        if n <= cap:
            return cand[:n]
        cap = n


def detect(dog, peak=PEAK, edge=EDGE, sigma0=SIGMA0):
    """(cand, kp): per octave the candidates and their refined records [n, 8] (x, y, sigma, response, octave, level,
    fractional level, ok)."""
    torch = _torch()
    ops = _ops()
    cands, kps = [], []
    for o, D in enumerate(dog):
        L, h, w = D.shape
        c = candidates(D, np.float32(PRE_PEAK * peak))
        kp = torch.empty(c.shape[0], _KP, dtype=torch.float32, device=D.device)
        ops.K('nero_features_refine', D, w, h, L, c, c.shape[0], o, float(sigma0), float(peak), float(edge), kp)
        cands.append(c)
        kps.append(kp)
    return cands, kps


def select(kps, max_features=MAX_FEATURES):
    """The kept keypoint records of all octaves by |response| descending (ties in candidate order), at most max_features."""
    torch = _torch()
    kp = torch.cat(kps, 0)
    kp = kp[kp[:, 7] > 0]
    order = torch.sort(-kp[:, 3].abs(), stable=True).indices
    return kp[order[:max_features]].contiguous()


def describe(kp, gauss):
    """(angle [n, 2], desc [n, 2, 128] uint8, nori [n]) of keypoint records kp on the octaves' Gaussian stacks."""
    torch = _torch()
    dev = kp.device
    n = kp.shape[0]
    angle = torch.zeros(n, 2, dtype=torch.float32, device=dev)
    desc = torch.zeros(n, 2, 128, dtype=torch.uint8, device=dev)
    nori = torch.zeros(n, dtype=torch.int32, device=dev)
    ptrs = torch.tensor([g.data_ptr() for g in gauss], dtype=torch.int64, device=dev)
    wh = torch.tensor([[g.shape[2], g.shape[1]] for g in gauss], dtype=torch.int32, device=dev)
    _ops().K('nero_features_describe', kp, n, ptrs, wh, len(gauss), gauss[0].shape[0], angle, desc, nori)
    return angle, desc, nori


def extract(rgb, max_size=MAX_SIZE, max_features=MAX_FEATURES):
    """SIFT features of one uint8 RGB image [h, w, 3] -> (keypoints fp32 [n, 6] numpy, descriptors uint8 [n, 128] CUDA,
    info dict with s, grey, gauss, dog, cand, kp (all refined records per octave), sel (the described records), angle,
    nori)."""
    torch = _torch()
    h, w = rgb.shape[:2]
    s = mvs.grey_scale(w, h, max_size)
    grey = mvs.prepare_grey(rgb, s)
    gauss, dog = scale_space(grey)
    cand, kps = detect(dog)
    sel = select(kps, max_features)
    angle, desc, nori = describe(sel, gauss) if sel.shape[0] else (torch.zeros(0, 2, device=grey.device),
                                                                    torch.zeros(0, 2, 128, dtype=torch.uint8, device=grey.device),
                                                                    torch.zeros(0, dtype=torch.int32, device=grey.device))
    keep = (torch.arange(2, device=grey.device)[None, :] < nori[:, None].long()).reshape(-1)
    src = torch.arange(sel.shape[0], device=grey.device).repeat_interleave(2)[keep][:max_features]
    th = angle.reshape(-1)[keep][:max_features].double().cpu().numpy()
    d = desc.reshape(-1, 128)[keep][:max_features].contiguous()
    k = sel[src].double().cpu().numpy()
    f = 2.0 ** k[:, 4]
    u, v, c = (f * k[:, 0] + 0.5) * s, (f * k[:, 1] + 0.5) * s, f * k[:, 2] * s
    kp6 = np.stack([u, v, c * np.cos(th), -c * np.sin(th), c * np.sin(th), c * np.cos(th)], 1).astype(np.float32)
    return kp6, d, dict(s=s, grey=grey, gauss=gauss, dog=dog, cand=cand, kp=kps, sel=sel, angle=angle, nori=nori, src=src)


def pairs_of(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


def match_batches(pad, limit=MATCH_ROWS):
    """The pairs i < j of images with pad[i] padded descriptor rows, as runs of consecutive pairs whose row-best records
    (pad[i] + pad[j] per pair) fit in `limit`: one matcher launch each, so every record offset fits the kernels' int32 and
    the records' memory stays bounded whatever the number of images."""
    if int(np.sum(pad, dtype=np.int64)) + TILE > _INT32_MAX:
        raise ValueError(f'{int(np.sum(pad, dtype=np.int64))} descriptor rows do not fit int32 offsets')
    batches, cur, rows = [], [], 0
    for i, j in pairs_of(len(pad)):
        need = int(pad[i]) + int(pad[j])
        if need > limit:
            raise ValueError(f'pair {i}, {j} needs {need} row-best records, more than {limit}')
        if cur and rows + need > limit:
            batches.append(cur)
            cur, rows = [], 0
        cur.append((i, j))
        rows += need
    if cur:
        batches.append(cur)
    return batches


def _batch_tables(batch, n, pad, off):
    """(tiles [T, 5], fwd [T', 4], the pair of each forward tile, row-best records) of one batch, int64."""
    tiles, fwd, fwd_pair, o = [], [], [], 0
    for i, j in batch:
        base = {(i, j): o, (j, i): o + pad[i]}
        o += pad[i] + pad[j]
        for a, b in ((i, j), (j, i)):
            if n[a] == 0 or n[b] == 0:
                continue
            t = np.arange(0, n[a], TILE, dtype=np.int64)
            rows = np.minimum(TILE, n[a] - t)
            tiles.append(np.stack([off[a] + t, rows, np.full_like(t, off[b]), np.full_like(t, n[b]), base[a, b] + t], 1))
            if a == i:
                fwd.append(np.stack([base[i, j] + t, np.full_like(t, base[j, i]), rows, t], 1))
                fwd_pair += [(i, j)] * t.shape[0]
    cat = lambda x, k: np.concatenate(x, 0) if x else np.zeros((0, k), np.int64)
    return cat(tiles, 5), cat(fwd, 4), fwd_pair, o


def match_all(descs, ratio=RATIO, max_d1=MAX_D1, batch_rows=MATCH_ROWS):
    """Mutual matches of every pair i < j of the CUDA uint8 descriptor sets descs [n_i, 128] -> {(i, j): CUDA int64 [m, 2]
    (index in i, index in j)} for the pairs with matches, and info (tiles: every directed tile, batches: launches)."""
    torch = _torch()
    ops = _ops()
    dev = torch.device('cuda')
    n = [int(d.shape[0]) for d in descs]
    pad = [-(-k // TILE) * TILE for k in n]
    batches = match_batches(pad, batch_rows)
    off = np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)
    buf = torch.zeros(max(int(off[-1]), TILE), 128, dtype=torch.uint8, device=dev)
    for i, d in enumerate(descs):
        if n[i]:
            buf[off[i]:off[i] + n[i]] = d
    norms = (buf.to(torch.int32) ** 2).sum(1, dtype=torch.int32)
    out, all_tiles = {}, []
    for batch in batches:
        tiles, fwd, fwd_pair, o = _batch_tables(batch, n, pad, off)
        all_tiles.append(tiles)
        T = fwd.shape[0]
        if T == 0:
            continue
        best = torch.empty(o, 3, dtype=torch.int32, device=dev)
        tt = torch.from_numpy(tiles.astype(np.int32)).to(dev)
        ops.K('nero_features_match', buf, norms, tt, tiles.shape[0], best)
        ft = torch.from_numpy(fwd.astype(np.int32)).to(dev)
        cnt = torch.empty(T, dtype=torch.int32, device=dev)
        boff = torch.empty(T, dtype=torch.int64, device=dev)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        cap = int(fwd[:, 2].sum())
        m = torch.empty(cap, 2, dtype=torch.int32, device=dev)
        ops.K('nero_features_mutual', best, ft, T, int(ratio[0]), int(ratio[1]), int(max_d1), cnt, boff, total, m, cap, launches=3)
        starts, counts = boff.cpu().numpy(), cnt.cpu().numpy()
        res = {}
        for t, pr in enumerate(fwd_pair):
            if counts[t]:
                r = res.setdefault(pr, [int(starts[t]), 0])
                r[1] = int(starts[t] + counts[t])
        for pr, (s0, s1) in res.items():
            out[pr] = m[s0:s1].long()
        assert sum(int(v.shape[0]) for pr, v in out.items() if pr in res) == int(total.item())
    return out, dict(tiles=np.concatenate(all_tiles, 0) if all_tiles else np.zeros((0, 5), np.int64), batches=len(batches), norms=norms)


def verify(points, hypotheses=HYPOTHESES, max_error=MAX_ERROR, seed=SEED):
    """RANSAC of each pair's correspondences points[k] = fp64 [m_k, 4] (x1, y1, x2, y2) -> (F [P, 9], best [P, 2]
    (hypothesis, count), count [P], inliers: list of bool arrays), all numpy."""
    torch = _torch()
    dev = torch.device('cuda')
    P = len(points)
    sizes = [int(np.asarray(p).shape[0]) for p in points]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    pts = torch.from_numpy(np.ascontiguousarray(np.concatenate([np.asarray(p, np.float64).reshape(-1, 4) for p in points], 0)
                                                if P else np.zeros((0, 4)))).to(dev)
    F = torch.empty(max(P, 1), 9, dtype=torch.float64, device=dev)
    best = torch.empty(max(P, 1), 2, dtype=torch.int32, device=dev)
    count = torch.empty(max(P, 1), dtype=torch.int32, device=dev)
    inl = torch.empty(max(int(off[-1]), 1), dtype=torch.uint8, device=dev)
    if P:
        _ops().K('nero_features_verify', pts, torch.from_numpy(off).to(dev), P, int(hypotheses), int(seed), float(max_error) ** 2, F, best,
                 count, inl)
    inl = inl.cpu().numpy().astype(bool)
    return F[:P].cpu().numpy(), best[:P].cpu().numpy(), count[:P].cpu().numpy(), [inl[off[k]:off[k + 1]] for k in range(P)]


def build_database(image_dir, db_path, same_camera=False, max_size=MAX_SIZE, max_features=MAX_FEATURES, log=None,
                   camera_model='SIMPLE_PINHOLE'):
    """The whole tool: features of every image, all-pair matches and verified geometries written to db_path.  -> info.
    Two-view verification fits F on the raw keypoints whatever the camera model."""
    import time
    names, cams, cam_of = image_table(image_dir, same_camera, camera_model)
    t0 = time.time()
    kps, descs = [], []
    for name in names:
        rgb = mvs.read_rgb(os.path.join(image_dir, name))
        k, d, _ = extract(rgb, max_size, max_features)
        kps.append(k)
        descs.append(d)
        if log:
            log(f'{name}: {k.shape[0]} features')
    t1 = time.time()
    matches, _ = match_all(descs)
    t2 = time.time()
    keys = sorted(matches)
    pts = [np.concatenate([kps[i][matches[i, j][:, 0].cpu().numpy(), :2], kps[j][matches[i, j][:, 1].cpu().numpy(), :2]], 1)
           .astype(np.float64) for i, j in keys]
    F, best, count, inl = verify(pts)
    t3 = time.time()
    geos = {}
    for k, (i, j) in enumerate(keys):
        if count[k] >= MIN_INLIERS:
            Fm = F[k].reshape(3, 3)
            E = camera_K(cams[cam_of[j] - 1]).T @ Fm @ camera_K(cams[cam_of[i] - 1])
            geos[i + 1, j + 1] = dict(matches=matches[i, j].cpu().numpy()[inl[k]], config=UNCALIBRATED, F=Fm, E=E, H=np.zeros((3, 3)),
                                      qvec=np.array([1.0, 0.0, 0.0, 0.0]), tvec=np.zeros(3))
    write_database(db_path, [(k + 1, nm, cam_of[k]) for k, nm in enumerate(names)], cams,
                   {k + 1: kp for k, kp in enumerate(kps)}, {k + 1: d.cpu().numpy() for k, d in enumerate(descs)},
                   {(i + 1, j + 1): matches[i, j].cpu().numpy() for i, j in keys}, geos)
    t4 = time.time()
    return dict(names=names, features=[k.shape[0] for k in kps], pairs=len(keys), verified=len(geos),
                times=dict(extract=t1 - t0, match=t2 - t1, verify=t3 - t2, write=t4 - t3))
