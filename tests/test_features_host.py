"""Sparse features without a GPU: the database writer against the golden database made by the reference's own set-up
(oracle/make_golden_colmapdb.py), the pair ids, the header's symbols, the tool's argument checks, and the numpy oracle's
detector on synthetic images."""
import importlib.util
import os
import re
import sqlite3
import subprocess

import numpy as np
import pytest

import nero_oracle_features as OF
from nero_b200 import features as Ft

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'colmap_database.npz')


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _dump(path):
    con = sqlite3.connect(path)
    try:
        tables = [r[0] for r in con.execute("SELECT name FROM sqlite_master WHERE type = 'table' AND name != 'sqlite_sequence' ORDER BY name")]
        info = {t: con.execute(f'PRAGMA table_info({t})').fetchall() for t in tables}
        rows = {t: sorted(con.execute(f'SELECT * FROM {t}').fetchall(), key=repr) for t in tables}
        index = con.execute('PRAGMA index_list(images)').fetchall()
    finally:
        con.close()
    return tables, info, rows, index


@pytest.mark.parametrize('same', [False, True])
def test_database_equals_the_golden_one(tmp_path, same):
    g = np.load(GOLD)
    img_dir = tmp_path / 'images'
    img_dir.mkdir()
    for k, name in enumerate(g['image_names']):
        (img_dir / str(name)).write_bytes(g[f'image_{k}'].tobytes())
    names = Ft.list_images(str(img_dir))
    cams, cam_of = Ft.cameras_for([Ft.image_size(str(img_dir / n)) for n in names], same)
    geo = dict(matches=g['m12'][:2], config=3, F=g['F'], E=g['E'], H=np.zeros((3, 3)), qvec=np.array([1.0, 0, 0, 0]), tvec=np.zeros(3))
    db = str(tmp_path / 'database.db')
    Ft.write_database(db, [(k + 1, n, cam_of[k]) for k, n in enumerate(names)], cams, {1: g['kp_1'], 2: g['kp_2']},
                      {1: g['desc_1'], 2: g['desc_2']}, {(1, 2): g['m12'], (2, 3): g['m32'][:, ::-1]}, {(1, 2): geo})
    ref = str(tmp_path / 'golden.db')
    with open(ref, 'wb') as f:
        f.write(g[f'database_same{int(same)}'].tobytes())
    got, want = _dump(db), _dump(ref)
    assert got[0] == want[0] and set(Ft.TABLES) <= set(got[0])
    assert got[1] == want[1], 'PRAGMA table_info differs'
    assert got[2] == want[2], 'rows differ'
    assert got[3] == want[3]
    assert len(want[2]['cameras']) == (1 if same else len(names))


def test_pair_id_round_trip():
    for a, b in [(1, 2), (7, 3), (1, 2147483646), (123456, 654321)]:
        pid = Ft.pair_id(a, b)
        assert pid == min(a, b) * 2147483647 + max(a, b)
        assert Ft.pair_ids(pid) == (min(a, b), max(a, b))


def test_library_exports_every_features_symbol():
    from nero_b200 import ops
    header = open(os.path.join(ROOT, 'include', 'nero_features.h')).read()
    names = set(re.findall(r'\bint\s+(nero_features_\w+)\s*\(', header))
    assert names == set(ops.FEATURES_PROTOS) and len(names) == 9
    out = subprocess.run(['nm', '-D', '--defined-only', ops._LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r'\bT\s+(nero_features_\w+)', out))
    assert names <= exported, f'not exported: {names - exported}'


def test_tool_refuses_an_existing_database_and_a_missing_image_directory(tmp_path):
    mf = tool('match_features')
    with pytest.raises(SystemExit):
        mf.parse_args(['--root', str(tmp_path)])            # no images/
    (tmp_path / 'images').mkdir()
    assert mf.parse_args(['--root', str(tmp_path)]).database == str(tmp_path / 'database.db')
    (tmp_path / 'database.db').write_bytes(b'')
    with pytest.raises(SystemExit):
        mf.parse_args(['--root', str(tmp_path)])
    assert mf.parse_args(['--root', str(tmp_path), '--force']).force
    with pytest.raises(FileExistsError):
        Ft.write_database(str(tmp_path / 'database.db'), [], [], {}, {}, {}, {})


def _blobs(w, h, centres, sigmas):
    ys, xs = np.mgrid[0:h, 0:w] + 0.5
    img = np.full((h, w), 0.2)
    for (cx, cy), s in zip(centres, sigmas):
        img += 0.6 * np.exp(-((xs - cx) ** 2 + (ys - cy) ** 2) / (2 * s * s))
    return img.astype(np.float32)


def _oracle_keypoints(grey):
    taps = [Ft.gaussian_taps(s) for s in Ft.level_sigmas()]
    sizes = Ft.octave_sizes(grey.shape[1], grey.shape[0])
    G, D = OF.scale_space(grey, taps, sizes, Ft.SCALES)
    out = []
    for o in range(len(sizes)):
        r = OF.refine(D[o], OF.extrema(D[o], np.float32(Ft.PRE_PEAK * Ft.PEAK)), o, Ft.SIGMA0, Ft.PEAK, Ft.EDGE)
        r = r[r[:, 7] > 0]
        f = 2.0 ** o
        out.append(np.stack([f * r[:, 0] + 0.5, f * r[:, 1] + 0.5, f * r[:, 2]], 1))
    return np.concatenate(out, 0)


def test_oracle_finds_blob_centres_and_scales():
    centres = [(40.2, 40.7), (120.3, 52.7), (70.6, 110.2), (150.0, 130.0)]
    sigmas = [5.0, 4.5, 6.0, 8.0]
    kp = _oracle_keypoints(_blobs(192, 160, centres, sigmas))
    for (cx, cy), s in zip(centres, sigmas):
        d = np.hypot(kp[:, 0] - cx, kp[:, 1] - cy)
        k = int(np.argmin(d))
        # the scale-normalised Laplacian of a Gaussian blob of sigma s peaks at scale s; the DoG lands a little below
        assert d[k] <= 0.5, f'blob at {(cx, cy)}: nearest keypoint {d[k]:.2f} px away'
        assert abs(np.log(kp[k, 2] / s)) <= np.log(1.25), f'blob of sigma {s}: scale {kp[k, 2]:.2f}'


def test_oracle_keypoints_repeat_opencv_sift():
    cv2 = pytest.importorskip('cv2')
    import nero_oracle_mvs as OM
    pr = OM.render(OM.OOp.scene(n_table=10, n_obj=10, outlier_frac=0.0, n_cams=1, seed=0)['poses'][0],
                   np.array([[288.0, 0, 160], [0, 288.0, 120], [0, 0, 1]]), 320, 240)
    grey = OM.grey(pr['rgb'], 1)
    kp = _oracle_keypoints(grey)
    sift = cv2.SIFT_create(contrastThreshold=0.02)
    ck = np.array([k.pt for k in sift.detect((grey * 255).astype(np.uint8), None)]) + 0.5
    near = np.array([np.hypot(ck[:, 0] - x, ck[:, 1] - y).min() for x, y in kp[:, :2]])
    # OpenCV upsamples first and differs in thresholds: a sanity check on position repeatability only
    assert kp.shape[0] >= 50 and (near <= 2.0).mean() >= 0.5, f'{(near <= 2.0).mean():.2f} of {kp.shape[0]} within 2 px'


def _jpeg_with_orientation(path, w, h, orientation):
    """A w x h JPEG whose EXIF block says `orientation` (6: display rotated by 90 degrees)."""
    import struct
    import cv2
    ok, enc = cv2.imencode('.jpg', np.random.RandomState(0).randint(0, 256, (h, w, 3)).astype(np.uint8))
    data = enc.tobytes()
    ifd = b'II*\x00' + struct.pack('<I', 8) + struct.pack('<H', 1) + struct.pack('<HHIHH', 0x0112, 3, 1, orientation, 0) + \
        struct.pack('<I', 0)
    app1 = b'Exif\x00\x00' + ifd
    with open(path, 'wb') as f:
        f.write(data[:2] + b'\xff\xe1' + struct.pack('>H', len(app1) + 2) + app1 + data[2:])


def test_images_keep_their_stored_frame_whatever_the_exif_orientation(tmp_path):
    """COLMAP and run_colmap.py's reader ignore EXIF orientation; the cameras, the pixels the features come from and the
    dense stage's pixels must all be in that stored frame."""
    import cv2
    from nero_b200 import mvs
    img_dir = tmp_path / 'images'
    img_dir.mkdir()
    path = str(img_dir / 'phone.jpg')
    _jpeg_with_orientation(path, 40, 20, 6)
    assert cv2.imread(path, cv2.IMREAD_COLOR).shape[:2] == (40, 20)     # a reader that applies the orientation
    assert mvs.read_rgb(path).shape == (20, 40, 3)
    assert Ft.image_size(path) == (40, 20)
    names, cams, cam_of = Ft.image_table(str(img_dir))
    assert names == ['phone.jpg'] and cam_of == [1]
    assert cams[0][2:4] == (40, 20) and np.array_equal(cams[0][4], [np.sqrt(40 ** 2 + 20 ** 2), 20.0, 10.0])


def test_match_batches_keep_every_offset_in_int32():
    pad = [8192] * 600                       # one launch for every pair would need 600 * 599 * 8192 > 2^31 records
    assert sum(2 * p for p in pad[:2]) * len(Ft.pairs_of(600)) > 2 ** 31
    batches = Ft.match_batches(pad)
    assert [pr for b in batches for pr in b] == Ft.pairs_of(600) and len(batches) > 1
    off = np.concatenate([[0], np.cumsum(pad)]).astype(np.int64)
    for b in (batches[0], batches[-1]):
        tiles, fwd, _, rows = Ft._batch_tables(b, pad, pad, off)
        assert rows <= Ft.MATCH_ROWS and tiles.max() < 2 ** 31 and fwd.max() < 2 ** 31
        assert (tiles[:, 4] + tiles[:, 1]).max() <= rows
    small = Ft.match_batches([128, 256, 128, 384], limit=640)
    for b in small:
        assert sum([128, 256, 128, 384][i] + [128, 256, 128, 384][j] for i, j in b) <= 640
    with pytest.raises(ValueError):
        Ft.match_batches([128, 1024], limit=640)              # one pair alone exceeds the limit
    with pytest.raises(ValueError):
        Ft.match_batches([2 ** 30, 2 ** 30])                  # the descriptor rows themselves exceed int32
