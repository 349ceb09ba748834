"""Sparse features on the GPU: the scale space and candidates of k_sift.cu bit for bit against
oracle/nero_oracle_features.py, refinement, orientations and descriptors to rounding, the tensor-core matcher exactly
against the int64 oracle, RANSAC against the fp64 oracle, run-to-run identity of the database, and accuracy on the
synthetic table / box / sphere project."""
import importlib.util
import os
import shutil
import sqlite3

import numpy as np
import pytest
import torch

import nero_oracle_features as OF
import nero_oracle_mvs as OM
from nero_b200 import features as Ft
from nero_b200 import mvs

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture(scope='module')
def small(tmp_path_factory):
    root = str(tmp_path_factory.mktemp('feat_small'))
    pr = OM.project(root, 4, 480, 360, per_view=10)
    out = []
    for name in pr['names']:
        rgb = mvs.read_rgb(os.path.join(root, 'images', name))
        out.append(Ft.extract(rgb, max_features=1000))
    return root, pr, out


def _taps():
    return [Ft.gaussian_taps(s) for s in Ft.level_sigmas()]


def test_scale_space_and_candidates_match_the_oracle_bit_for_bit(small):
    _, _, out = small
    for _, _, info in out:
        grey = info['grey'].cpu().numpy()
        sizes = [(g.shape[2], g.shape[1]) for g in info['gauss']]
        assert sizes == Ft.octave_sizes(grey.shape[1], grey.shape[0])
        og, od = OF.scale_space(grey, _taps(), sizes, Ft.SCALES)
        for o in range(len(sizes)):
            assert np.array_equal(info['gauss'][o].cpu().numpy(), og[o]), f'octave {o}: Gaussian levels differ'
            assert np.array_equal(info['dog'][o].cpu().numpy(), od[o]), f'octave {o}: DoG levels differ'
            oc = OF.extrema(od[o], np.float32(Ft.PRE_PEAK * Ft.PEAK))
            assert np.array_equal(info['cand'][o].cpu().numpy(), oc), f'octave {o}: candidates differ'
        assert sum(c.shape[0] for c in info['cand']) > 50


def test_refinement_orientation_and_descriptors_match_the_oracle(small):
    _, _, out = small
    for _, _, info in out:
        for o, (c, kp) in enumerate(zip(info['cand'], info['kp'])):
            ok = OF.refine(info['dog'][o].cpu().numpy(), c.cpu().numpy(), o, Ft.SIGMA0, Ft.PEAK, Ft.EDGE)
            g = kp.cpu().numpy().astype(np.float64)
            agree = g[:, 7] == ok[:, 7]
            assert agree.mean() >= 0.99
            both = agree & (ok[:, 7] > 0)
            assert np.abs(g[both, :2] - ok[both, :2]).max(initial=0.0) <= 1e-4
            assert np.allclose(g[both, 2], ok[both, 2], rtol=1e-5)
        sel = info['sel'].cpu().numpy()
        gauss = [g.cpu().numpy() for g in info['gauss']]
        oa, odesc, onori, _ = OF.describe(sel, gauss)
        nori = info['nori'].cpu().numpy()
        same = nori == onori
        assert same.mean() >= 0.97
        a = info['angle'].cpu().numpy()
        desc = Ft.describe(info['sel'], info['gauss'])[1].cpu().numpy().astype(np.int64)
        first = same & (nori > 0)
        close_ang = np.abs(np.angle(np.exp(1j * (a[first, 0] - oa[first, 0])))) <= 1e-3
        assert close_ang.mean() >= 0.97
        good = (np.abs(desc[first, 0] - odesc[first, 0].astype(np.int64)).max(1) <= 1)[close_ang]
        assert good.mean() >= 0.99, f'{(~good).sum()} descriptors differ by more than 1'


def test_matcher_equals_the_int64_oracle():
    rng = np.random.RandomState(3)
    sizes = [1, 127, 128, 129, 300, 0]
    base = rng.randint(0, 256, (64, 128))
    descs = []
    for n in sizes:
        # perturbed copies of a shared pool so that ratio and mutual tests both pass and fail
        d = np.clip(base[rng.randint(0, 64, n)] + rng.randint(-40, 41, (n, 128)), 0, 255).astype(np.uint8)
        descs.append(d)
    gm, info = Ft.match_all([torch.from_numpy(d).cuda() for d in descs])
    # the same pairs in launches of at most 1024 row-best records each
    bm, binfo = Ft.match_all([torch.from_numpy(d).cuda() for d in descs], batch_rows=1024)
    assert info['batches'] == 1 and binfo['batches'] > 3
    total = 0
    for i, j in Ft.pairs_of(len(sizes)):
        om = OF.match(descs[i], descs[j])
        for m in (gm, bm):
            got = m[i, j].cpu().numpy() if (i, j) in m else np.zeros((0, 2), np.int64)
            assert np.array_equal(got, om), f'pair {i}, {j}'
        total += om.shape[0]
    assert total > 20


def test_matcher_and_ransac_equal_the_oracle_on_extracted_features(small):
    _, _, out = small
    descs = [d for _, d, _ in out]
    gm, _ = Ft.match_all(descs)
    npd = [d.cpu().numpy() for d in descs]
    keys = sorted(gm)
    for i, j in Ft.pairs_of(len(descs)):
        om = OF.match(npd[i], npd[j])
        assert np.array_equal(gm[i, j].cpu().numpy() if (i, j) in gm else np.zeros((0, 2), np.int64), om)
    pts = [np.concatenate([out[i][0][gm[i, j][:, 0].cpu().numpy(), :2], out[j][0][gm[i, j][:, 1].cpu().numpy(), :2]], 1).astype(np.float64)
           for i, j in keys]
    F, best, count, inl = Ft.verify(pts)
    checked = 0
    for p, P in enumerate(pts):
        oF, oh, oc, oin = OF.ransac(P, p, Ft.HYPOTHESES, Ft.SEED, Ft.MAX_ERROR ** 2)
        if oc < Ft.MIN_INLIERS:
            continue
        checked += 1
        print(f'pair {keys[p]}: {P.shape[0]} matches, hypothesis {tuple(best[p])} vs oracle {(oh, oc)}, inliers {count[p]} vs {oin.sum()}, '
              f'|F - oracle| {np.abs(F[p] - oF).max():.3e}')
        assert best[p, 0] == oh and best[p, 1] == oc
        assert np.array_equal(inl[p], oin) and count[p] == oin.sum()
        assert np.abs(F[p] - oF).max() <= 1e-9 * np.abs(oF).max()
    assert checked >= 2


def test_database_is_identical_across_runs(small, tmp_path):
    root, _, _ = small
    rows = []
    for k in range(2):
        db = str(tmp_path / f'db{k}.db')
        info = Ft.build_database(os.path.join(root, 'images'), db)
        con = sqlite3.connect(db)
        rows.append({t: con.execute(f'SELECT * FROM {t}').fetchall() for t in Ft.TABLES})
        con.close()
    assert rows[0] == rows[1]
    assert len(rows[0]['keypoints']) == 4 and len(rows[0]['matches']) >= 1


def _rotation_deg(R):
    return np.degrees(np.arccos(np.clip((np.trace(R) - 1) / 2, -1, 1)))


def test_accuracy_on_twelve_views(tmp_path):
    root = str(tmp_path)
    pr = OM.project(root, 12, 640, 480, per_view=10, workers=4)
    db = os.path.join(root, 'database.db')
    info = Ft.build_database(os.path.join(root, 'images'), db)
    con = sqlite3.connect(db)
    kps = {i: np.frombuffer(b, np.float32).reshape(r, c) for i, r, c, b in con.execute('SELECT image_id, rows, cols, data FROM keypoints')}
    geos = {Ft.pair_ids(p): (np.frombuffer(d, np.uint32).reshape(r, 2), np.frombuffer(F, np.float64).reshape(3, 3))
            for p, r, d, F in con.execute('SELECT pair_id, rows, data, F FROM two_view_geometries')}
    con.close()
    K = pr['K']
    poses, truth = pr['poses'], pr['truth']
    good = tot = 0
    errs = []
    for (a, b), (m, F) in geos.items():
        i, j = a - 1, b - 1
        x1, x2 = kps[a][m[:, 0], :2].astype(np.float64), kps[b][m[:, 1], :2].astype(np.float64)
        d = truth[i]['depth'][np.clip(x1[:, 1].astype(int), 0, 479), np.clip(x1[:, 0].astype(int), 0, 639)]
        X = np.stack([(x1[:, 0] - K[0, 2]) / K[0, 0] * d, (x1[:, 1] - K[1, 2]) / K[1, 1] * d, d], 1)
        R, t = mvs.relative(poses[i], poses[j])
        Y = X @ R.T + t
        y = Y[:, :2] / Y[:, 2:] * K[0, 0] + K[:2, 2]
        ok = (d > 0) & (np.linalg.norm(y - x2, axis=1) <= 2.0)
        good += ok.sum()
        tot += m.shape[0]
        if m.shape[0] >= 100:
            # E from the true K; of its two rotations the one closer to the truth must be within 1 degree
            U, _, Vt = np.linalg.svd(K.T @ F @ K)
            Wm = np.array([[0, -1, 0], [1, 0, 0], [0, 0, 1]])
            cands = [U @ W @ Vt for W in (Wm, Wm.T)]
            cands = [Rc * np.sign(np.linalg.det(Rc)) for Rc in cands]
            errs.append(min(_rotation_deg(Rc @ R.T) for Rc in cands))
    errs = np.asarray(errs)
    print(f'{len(geos)} verified pairs, {good} of {tot} inliers within 2 px; rotation errors (deg) of {errs.shape[0]} pairs with >= 100 '
          f'inliers: median {np.median(errs):.3f}, max {errs.max():.3f}, {(errs <= 1.0).mean():.3f} within 1 deg')
    assert tot > 0 and good / tot >= 0.95, f'{good} of {tot} inliers within 2 px'
    # the pairs whose views overlap (half of view i's surface samples project into view j) are verified
    overlap = verified = 0
    for i, j in Ft.pairs_of(12):
        ys, xs = np.nonzero(truth[i]['depth'] > 0)
        sel = np.arange(0, ys.shape[0], 97)
        d = truth[i]['depth'][ys[sel], xs[sel]]
        X = np.stack([(xs[sel] + 0.5 - K[0, 2]) / K[0, 0] * d, (ys[sel] + 0.5 - K[1, 2]) / K[1, 1] * d, d], 1)
        R, t = mvs.relative(poses[i], poses[j])
        Y = X @ R.T + t
        y = Y[:, :2] / Y[:, 2:] * K[0, 0] + K[:2, 2]
        vis = (Y[:, 2] > 0) & (y[:, 0] >= 0) & (y[:, 0] < 640) & (y[:, 1] >= 0) & (y[:, 1] < 480)
        if vis.mean() >= 0.5:
            overlap += 1
            verified += (i + 1, j + 1) in geos
    print(f'{verified} of {overlap} overlapping pairs verified')
    assert verified >= 0.9 * overlap


def _triangulate(K, P1, P2, x1, x2):
    """DLT points [n, 3] of correspondences x1, x2 [n, 2] between world-to-camera poses P1, P2 [3, 4]."""
    A1, A2 = K @ P1, K @ P2
    out = []
    for a, b in zip(x1, x2):
        M = np.stack([a[0] * A1[2] - A1[0], a[1] * A1[2] - A1[1], b[0] * A2[2] - A2[0], b[1] * A2[2] - A2[1]])
        X = np.linalg.svd(M)[2][-1]
        out.append(X[:3] / X[3])
    return np.asarray(out).reshape(-1, 3)


def test_match_features_database_feeds_dense_points_and_prepare_custom_object(tmp_path, capsys):
    """The database's image ids, names and keypoints make the model the mapper would write (here with the true poses and
    K, tracks triangulated from the verified inliers), and the rest of the workflow accepts it."""
    import nero_oracle_objprep as OOp
    from nero_b200 import objprep as OP
    from nero_b200.evaluate import read_points_ply
    root = str(tmp_path)
    pr = OM.project(root, 12, 640, 480, seed=3, workers=4)
    shutil.rmtree(os.path.join(root, 'sparse'))          # the model below comes from the database alone
    tool('match_features').main(['--root', root])
    con = sqlite3.connect(os.path.join(root, 'database.db'))
    images = con.execute('SELECT image_id, name, camera_id FROM images ORDER BY image_id').fetchall()
    cam_ids = sorted({c for _, _, c in images})
    kps = {i: np.frombuffer(b, np.float32).reshape(r, c).astype(np.float64)
           for i, r, c, b in con.execute('SELECT image_id, rows, cols, data FROM keypoints')}
    geos = [(Ft.pair_ids(p), np.frombuffer(d, np.uint32).reshape(r, 2)) for p, r, d in
            con.execute('SELECT pair_id, rows, data FROM two_view_geometries ORDER BY pair_id')]
    con.close()
    assert [n for _, n, _ in images] == pr['names']
    K = pr['K']
    pose = {iid: pr['poses'][pr['names'].index(name)] for iid, name, _ in images}
    p3d = {iid: np.full(kps[iid].shape[0], -1, np.int64) for iid in kps}
    points = {}
    for (a, b), m in geos:
        m = m[(p3d[a][m[:, 0]] < 0) & (p3d[b][m[:, 1]] < 0)]
        X = _triangulate(K, pose[a], pose[b], kps[a][m[:, 0], :2], kps[b][m[:, 1], :2])
        for (k1, k2), x in zip(m, X):
            ok = True
            for iid, k in ((a, k1), (b, k2)):
                y = K @ (pose[iid][:, :3] @ x + pose[iid][:, 3])
                ok = ok and y[2] > 0 and np.hypot(*(y[:2] / y[2] - kps[iid][k, :2])) <= 2.0
            if ok and p3d[a][k1] < 0 and p3d[b][k2] < 0:
                pid = len(points) + 1
                points[pid] = (x, [128, 128, 128], 0.5, [a, b], [int(k1), int(k2)])
                p3d[a][k1], p3d[b][k2] = pid, pid
    cams = {c: ('PINHOLE', 640, 480, [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]) for c in cam_ids}
    imgs = {iid: (OOp.rotmat2qvec(pose[iid][:, :3]), pose[iid][:, 3], cid, name, kps[iid][:, :2], p3d[iid]) for iid, name, cid in images}
    OOp.write_colmap_model(os.path.join(root, 'sparse', '0'), cams, imgs, points, 'bin')
    tool('dense_points').main(['--root', root])
    assert os.path.isfile(os.path.join(root, 'points.ply'))
    tool('prepare_custom_object').main(['--root', root, '--min-component', '0.1'])
    up = np.loadtxt(os.path.join(root, 'meta_info.txt'))[0]
    ang = np.degrees(np.arccos(np.clip(up @ pr['up'] / np.linalg.norm(up), -1, 1)))
    obj = read_points_ply(os.path.join(root, 'object_point_cloud.ply'))
    _, D, _, _ = OP.scene_scale(OP.read_colmap_model(os.path.join(root, 'sparse', '0'))[0])
    lo, hi = OM.object_bbox()
    err = max(np.abs(obj.min(0) - lo).max(), np.abs(obj.max(0) - hi).max())
    print(capsys.readouterr().out)
    print(f'{len(points)} triangulated points; up error {ang:.4f} deg, bounding-box error {err / (OP.VOXEL_FRAC * D):.2f} voxels, '
          f'{obj.shape[0]} object points')
    assert len(points) >= 12 * 10 and ang <= 1.0 and err <= 2 * OP.VOXEL_FRAC * D
