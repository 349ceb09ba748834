"""CPU: the occlusion sampler's strata, the byte formula, the occlusion map file, the glTF container with and without an
occlusion texture, the argument errors of gltf.export and tools/bake_occlusion.py, and the library's exports of
include/nero_occlusion.h."""
import ctypes
import json
import os
import re
import struct
import subprocess
import sys
from fractions import Fraction

import numpy as np
import pytest

import nero_oracle_occlusion as OO
from nero_b200 import gltf as GL
from nero_b200 import occlusion as OC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools')


@pytest.mark.parametrize('seed', [0, 1, 7])
def test_sampler_is_in_the_unit_square_with_one_sample_per_stratum(seed):
    """r1, r2 in [0, 1); at N = 256 each r1-stratum of width 1/N holds one sample (checked for these seeds and keys: a
    wrapped value can round onto a stratum edge for others), and so does each r2-stratum."""
    keys = np.arange(512)
    r1, r2 = OO.sampler(seed, keys, 256)
    assert r1.dtype == np.float32 and r1.shape == (512, 256)
    assert (r1 >= 0).all() and (r1 < 1).all() and (r2 >= 0).all() and (r2 < 1).all()
    for r in (r1, r2):
        strata = np.sort(np.floor(r.astype(np.float64) * 256).astype(np.int64), axis=1)
        assert np.array_equal(strata, np.broadcast_to(np.arange(256), strata.shape))
    # a pure function of (seed, key, i, N): the same key gives the same row, another key another rotation
    a1, _ = OO.sampler(seed, [5, 5, 6], 256)
    assert np.array_equal(a1[0], a1[1]) and not np.array_equal(a1[0], a1[2])


def test_brev_is_the_bit_reversal():
    i = np.asarray([0, 1, 2, 3, 0x80000000, 0x12345678], np.uint64)
    ref = [int(f'{int(x):032b}'[::-1], 2) for x in i]
    assert [int(x) for x in OO.brev32(i)] == ref


@pytest.mark.parametrize('rays', [1, 2, 3, 7, 64, 255, 256, 1000, 4096])
def test_byte_is_round_half_up_of_255_c_over_n(rays):
    c = np.arange(rays + 1)
    ref = np.asarray([int(Fraction(255 * int(k), rays) + Fraction(1, 2)) for k in c])
    assert np.array_equal(OC.encode(c, rays), ref) and np.array_equal(OO.encode(c, rays), ref)
    assert OC.encode(rays, rays) == 255 and OC.encode(0, rays) == 0


def test_byte_at_the_largest_ray_count():
    c = np.asarray([0, 1, 128, 32767, 32768, 65535, 65536])
    ref = np.asarray([int(Fraction(255 * int(k), 65536) + Fraction(1, 2)) for k in c])
    assert np.array_equal(OC.encode(c, 65536), ref)


def test_occlusion_map_file_round_trip(tmp_path):
    import cv2
    img = np.random.RandomState(3).randint(0, 256, (13, 21)).astype(np.uint8)
    path = str(tmp_path / 'occlusion_0.png')
    OC.write_occlusion_map(path, img)
    raw = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    assert raw.shape == (13, 21, 3) and (raw[..., 0] == raw[..., 1]).all() and (raw[..., 1] == raw[..., 2]).all()
    assert np.array_equal(OC.read_occlusion_map(path), img)
    OC.write_occlusion_map(path, np.repeat(img[..., None], 3, 2))       # the bake's [h,w,3] form writes the same file
    assert np.array_equal(OC.read_occlusion_map(path), img)
    grey = str(tmp_path / 'grey.png')
    cv2.imwrite(grey, img)
    with pytest.raises(ValueError, match='grey.png'):
        OC.read_occlusion_map(grey)
    sixteen = str(tmp_path / 'sixteen.png')
    cv2.imwrite(sixteen, np.zeros((4, 4, 3), np.uint16))
    with pytest.raises(ValueError, match='sixteen.png'):
        OC.read_occlusion_map(sixteen)
    with pytest.raises(ValueError, match='missing'):
        OC.read_occlusion_map(str(tmp_path / 'nope.png'))


def small_glb_arrays(seed=0):
    rng = np.random.RandomState(seed)
    pos = rng.rand(4, 3).astype(np.float32)
    nrm = np.tile(np.asarray([[0, 0, 1]], np.float32), (4, 1))
    uv = rng.rand(4, 2).astype(np.float32)
    idx = np.asarray([[0, 1, 2], [0, 2, 3]], np.uint32)
    images = {'base_color': rng.randint(0, 256, (6, 5, 3)).astype(np.uint8),
              'metallic_roughness': rng.randint(0, 256, (6, 5, 3)).astype(np.uint8)}
    return pos, nrm, uv, idx, images


def glb_json(data):
    jl = struct.unpack('<I', data[12:16])[0]
    return json.loads(data[20:20 + jl].decode())


def test_glb_container_with_and_without_occlusion():
    pos, nrm, uv, idx, images = small_glb_arrays()
    plain = GL.glb_bytes(pos, nrm, uv, idx, images)
    assert plain == GL.glb_bytes(pos, nrm, uv, idx, images, occlusion=False)
    assert 'occlusionTexture' not in glb_json(plain)['materials'][0]
    back = GL.read_glb(plain)
    assert back['occlusion'] is None and back['occlusion_strength'] is None
    with_occ = GL.glb_bytes(pos, nrm, uv, idx, images, occlusion=True)
    mat = glb_json(with_occ)['materials'][0]
    assert mat['occlusionTexture'] == {'index': 1} and mat['pbrMetallicRoughness']['metallicRoughnessTexture'] == {'index': 1}
    back = GL.read_glb(with_occ)
    assert np.array_equal(back['occlusion'], images['metallic_roughness'][..., 0]) and back['occlusion_strength'] == 1.0
    assert np.array_equal(back['images']['metallic_roughness'], images['metallic_roughness'])


def write_obj(tmp_path, size=8):
    from nero_b200 import synthetic
    from nero_b200.texmap import write_textured_obj
    verts, tris = synthetic.icosphere(0, 0.5)
    tris = np.ascontiguousarray(tris[:, [0, 2, 1]])
    rng = np.random.RandomState(0)
    vt, ft = rng.rand(3 * tris.shape[0], 2).astype(np.float32), np.arange(3 * tris.shape[0], dtype=np.int32).reshape(-1, 3)
    grey = np.full((size, size, 3), 128, np.uint8)
    write_textured_obj(str(tmp_path / 'n2m'), verts, tris, vt, ft, (grey, grey, grey))
    return str(tmp_path / 'n2m' / 'mesh_0.obj')


def test_export_rejects_an_occlusion_map_of_another_size(tmp_path):
    obj = write_obj(tmp_path)
    occ = str(tmp_path / 'n2m' / 'occlusion_0.png')
    OC.write_occlusion_map(occ, np.full((4, 6), 200, np.uint8))
    with pytest.raises(ValueError, match=r'occlusion_0.png.*6x4.*8x8'):
        GL.export(obj, occlusion_path=occ)


def run_tool(name, args, cwd):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(TOOLS, name)] + args, cwd=cwd, env=env, capture_output=True, text=True)


def test_bake_occlusion_argument_errors(tmp_path):
    write_obj(tmp_path)
    obj = ['--obj', 'n2m/mesh_0.obj']
    for args, msg in ((obj + ['--rays', '0'], '--rays 0'), (obj + ['--rays', '65537'], '--rays 65537'),
                      (obj + ['--distance', '0'], '--distance 0'), (obj + ['--distance', '-0.5'], '--distance -0.5'),
                      (obj + ['--cage-distance', '0.1'], '--cage-distance needs --detail'),
                      (['--obj', 'n2m/none.obj'], 'no such file'), ([], '--obj')):
        r = run_tool('bake_occlusion.py', args, tmp_path)
        assert r.returncode == 2 and msg in r.stderr, (args, r.stderr)
    r = run_tool('export_gltf.py', obj + ['--occlusion', 'n2m/none.png'], tmp_path)
    assert r.returncode == 2 and '--occlusion n2m/none.png' in r.stderr, r.stderr


def test_library_exports_every_symbol_of_the_occlusion_header():
    import __graft_entry__ as g
    lib = ctypes.CDLL(g.build())
    txt = open(os.path.join(ROOT, 'include', 'nero_occlusion.h')).read()
    syms = sorted(set(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(', txt)))
    assert syms == ['nero_occlusion_bytes', 'nero_occlusion_points', 'nero_occlusion_texels']
    for s in syms:
        assert hasattr(lib, s), f'{s} declared in include/nero_occlusion.h but not exported'
    from nero_b200 import ops
    for s in syms:
        assert getattr(ops.lib, s).argtypes is not None and len(getattr(ops.lib, s).argtypes) == len(ops.OCCLUSION_PROTOS[s])


def test_entry_points_refuse_bad_arguments():
    """Checked before any launch, so no device is needed: rays outside [1, 65536], a non-positive or non-finite distance
    and NULL required buffers return 1."""
    from nero_b200 import ops
    lib, one = ops.lib, 1
    buf = ctypes.c_void_p(16)       # never dereferenced: the checks refuse the call first
    for rays, dist in ((0, 0.25), (65537, 0.25), (64, 0.0), (64, -1.0), (64, float('nan')), (64, float('inf'))):
        assert lib.nero_occlusion_points(buf, buf, None, 1, buf, buf, rays, dist, 0, buf, None) == one, (rays, dist)
    assert lib.nero_occlusion_points(None, buf, None, 1, buf, buf, 64, 0.25, 0, buf, None) == one
    assert lib.nero_occlusion_points(buf, buf, None, -1, buf, buf, 64, 0.25, 0, buf, None) == one
    assert lib.nero_occlusion_points(None, None, None, 0, None, None, 64, 0.25, 0, None, None) == 0
    assert lib.nero_occlusion_bytes(buf, 1, buf, 0, 4, 4, buf, None) == one
    assert lib.nero_occlusion_bytes(buf, 17, buf, 64, 4, 4, buf, None) == one
    args = [buf, 4, 4, buf, 1, buf, buf, buf, buf, None, buf, None, 0.02, buf, buf, buf, buf, None, None, None]
    assert lib.nero_occlusion_texels(*args) == one            # a detail BVH without its triangles and normals
    args[10], args[11], args[9], args[12] = buf, buf, buf, 0.0
    assert lib.nero_occlusion_texels(*args) == one            # cage distance 0
