"""Structure from motion without a GPU: the model writer against the golden model written by the reference's own writer
(oracle/make_golden_sfm.py), the header's symbols, the oracle's P3P, the host protocol's small pieces and the tool's
refusals, which all come before any GPU work."""
import importlib.util
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import make_golden_sfm as MG
import nero_oracle_sfm as OS
from nero_b200 import features as Ft
from nero_b200 import objprep as OP
from nero_b200 import sfm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'colmap_model.npz')


def tool(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, 'tools', f'{name}.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_model_writer_reproduces_the_reference_bytes_and_reads_back(tmp_path):
    g = np.load(GOLD)
    cams, images, points = MG.model()
    OP.write_colmap_model(str(tmp_path), cams, images, points)
    for n in ('cameras', 'images', 'points3D'):
        assert (tmp_path / f'{n}.bin').read_bytes() == g[f'{n}_bin'].tobytes(), f'{n}.bin differs from the reference writer'
    views, pts, tracks = OP.read_colmap_model(str(tmp_path), tracks=True)
    assert sorted(views) == sorted(images) and pts.shape == (len(points), 3)
    for (pid, p), X, tr in zip(points.items(), pts, tracks):
        assert np.array_equal(X, p[0]) and list(tr) == p[3]
    for iid, (q, t, cid, name, _, _) in images.items():
        assert views[iid][0] == name
        assert np.allclose(views[iid][1][:, 3], t, rtol=1e-6) and np.allclose(views[iid][1][:, :3], OP.qvec2rotmat(q), atol=1e-6)


def test_library_exports_every_sfm_symbol():
    from nero_b200 import ops
    header = open(os.path.join(ROOT, 'include', 'nero_sfm.h')).read()
    names = set(re.findall(r'\bint\s+(nero_sfm_\w+)\s*\(', header))
    assert names == set(ops.SFM_PROTOS) and len(names) == 9
    out = subprocess.run(['nm', '-D', '--defined-only', ops._LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(re.findall(r'\bT\s+(nero_sfm_\w+)', out))
    assert names <= exported, f'not exported: {names - exported}'


def test_sizes_agree_with_the_header():
    header = open(os.path.join(ROOT, 'include', 'nero_sfm.h')).read()
    val = lambda k: int(re.search(rf'#define {k}\s+(\d+)', header).group(1))
    assert val('NERO_SFM_MAX_IMAGES') == sfm.MAX_IMAGES and val('NERO_SFM_CHUNK') == sfm.CHUNK
    assert sfm.P3P_HYPOTHESES <= val('NERO_SFM_MAX_HYP') and val('NERO_SFM_BLOCK') == 256


def test_chunks_cover_each_segment_in_order():
    import torch
    counts = torch.tensor([1, 256, 257, 1000, 3], dtype=torch.int64)
    key = torch.arange(10, dtype=torch.int32).reshape(5, 2)
    chunk, ckey, seg_chunk = sfm._chunks(counts, key)
    off = np.concatenate([[0], np.cumsum(counts.numpy())])
    assert seg_chunk.tolist() == [0, 1, 2, 4, 8, 9]
    for s in range(5):
        c = chunk[seg_chunk[s]:seg_chunk[s + 1]].numpy()
        assert c[0, 0] == off[s] and c[-1, 1] == off[s + 1] and (c[1:, 0] == c[:-1, 1]).all()
        assert ((c[:, 1] - c[:, 0]) <= sfm.CHUNK).all() and ((c[:, 1] - c[:, 0]) > 0).all()
        assert (ckey[seg_chunk[s]:seg_chunk[s + 1]] == key[s]).all()


def test_oracle_p3p_recovers_known_poses():
    rng = np.random.RandomState(5)
    worst = 0.0
    for _ in range(200):
        R = OS.rodrigues(rng.randn(3))
        t = rng.randn(3) * 0.5 + [0, 0, 5]
        Xc = np.stack([rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3), rng.uniform(3, 7, 3)], 1)
        X = (Xc - t) @ R
        sols = OS.p3p(Xc / np.linalg.norm(Xc, axis=1, keepdims=True), X)
        assert 1 <= len(sols) <= 4
        worst = max(worst, min(max(np.abs(Rs - R).max(), np.abs(ts - t).max()) for Rs, ts in sols))
    assert worst <= 1e-9, worst


def test_essential_decomposition_contains_the_true_pose():
    rng = np.random.RandomState(2)
    R = OS.rodrigues(0.3 * rng.randn(3))
    t = rng.randn(3)
    t /= np.linalg.norm(t)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    cands = sfm.essential_poses(5.0 * tx @ R)
    assert min(np.abs(Rc - R).max() + np.abs(tc - t).max() for Rc, tc in cands) <= 1e-12


def test_quaternions_round_trip():
    rng = np.random.RandomState(3)
    for k in range(100):
        R = OS.rodrigues(rng.randn(3) * (3.0 if k % 2 else 0.1))
        q = sfm._qvec(R)
        assert q[0] >= 0 and abs(np.linalg.norm(q) - 1) <= 1e-14
        assert np.abs(OP.qvec2rotmat(q) - R).max() <= 1e-12


def test_largest_component_and_its_ties():
    pairs = {(1, 2): None, (2, 3): None, (5, 6): None, (6, 7): None, (8, 9): None}
    assert sfm.largest_component(list(range(1, 10)), pairs) == [1, 2, 3]      # ties to the lower smallest id
    pairs[(7, 8)] = None
    assert sfm.largest_component(list(range(1, 10)), pairs) == [5, 6, 7, 8, 9]


def _database(path, model=Ft.SIMPLE_PINHOLE, verified=True):
    cams, cam_of = Ft.cameras_for([(64, 48)] * 3)
    cams = [(c, model, w, h, np.append(p, 0.0) if model != Ft.SIMPLE_PINHOLE else p, pr) for c, _, w, h, p, pr in cams]
    kp = {i: np.random.RandomState(i).rand(10, 6).astype(np.float32) * 40 for i in (1, 2, 3)}
    m = np.stack([np.arange(10), np.arange(10)], 1).astype(np.uint32)
    geos = {(1, 2): dict(matches=m, config=3, F=np.eye(3), E=np.eye(3), H=np.zeros((3, 3)), qvec=np.array([1.0, 0, 0, 0]),
                         tvec=np.zeros(3))} if verified else {}
    Ft.write_database(str(path), [(k + 1, f'img_{k}.png', cam_of[k]) for k in range(3)], cams, kp, {}, {(1, 2): m}, geos)


def _refusal(root, *extra):
    """Exit code and stderr of map_sparse.py in a process that sees no GPU."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'map_sparse.py'), '--root', str(root), *extra], env=env,
                       capture_output=True, text=True, timeout=300)
    return r.returncode, r.stderr


def test_tool_refusals_come_before_any_gpu_work(tmp_path):
    ms = tool('map_sparse')
    root = tmp_path / 'obj'
    root.mkdir()
    (root / 'images').mkdir()
    rc, err = _refusal(root)
    assert rc == 2 and 'no database' in err
    _database(root / 'database.db', verified=False)
    rc, err = _refusal(root)
    assert rc == 2 and 'no verified image pair' in err
    os.remove(root / 'database.db')
    _database(root / 'database.db', model=2)
    rc, err = _refusal(root)
    assert rc == 2 and 'SIMPLE_PINHOLE cameras only' in err and 'SIMPLE_RADIAL' in err
    os.remove(root / 'database.db')
    _database(root / 'database.db')
    flags, db = ms.parse_args(['--root', str(root)])
    assert flags.output == str(root / 'sparse' / '0') and flags.database == str(root / 'database.db')
    assert sorted(db['pairs']) == [(1, 2)] and db['pairs'][1, 2][0].shape == (10, 2)
    os.makedirs(root / 'sparse' / '0')
    (root / 'sparse' / '0' / 'images.bin').write_bytes(b'')
    rc, err = _refusal(root)
    assert rc == 2 and 'holds a model' in err
    assert ms.parse_args(['--root', str(root), '--force'])[0].force
