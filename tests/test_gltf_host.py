"""CPU: the GLB container round trip and its structure, the material tables, the oracle's weld, tangent conventions (flat and
mirrored quads), the identity map and the decode accuracy of the tangent-space conversion, and the argument errors of
tools/export_gltf.py."""
import json
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

import nero_oracle_gltf as OG
import nero_oracle_normalmap as ON
from nero_b200 import gltf as GL
from nero_b200 import relight as RL
from nero_b200 import synthetic
from nero_b200 import texmap as TX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools')


def synthetic_arrays(W=37, T=23, seed=0, tangents=True, normal=True):
    rng = np.random.RandomState(seed)
    a = dict(positions=rng.randn(W, 3).astype(np.float32), normals=rng.randn(W, 3).astype(np.float32),
             texcoords=rng.rand(W, 2).astype(np.float32), indices=rng.randint(0, W, (T, 3)).astype(np.uint32),
             tangents=np.concatenate([rng.randn(W, 3), rng.choice([-1.0, 1.0], (W, 1))], 1).astype(np.float32) if tangents else None)
    a['images'] = {'base_color': rng.randint(0, 256, (5, 7, 3)).astype(np.uint8),
                   'metallic_roughness': rng.randint(0, 256, (5, 7, 3)).astype(np.uint8)}
    if normal:
        a['images']['normal'] = rng.randint(0, 256, (9, 4, 3)).astype(np.uint8)
    return a


@pytest.mark.parametrize('with_map', [True, False])
def test_container_round_trips_exactly(with_map):
    a = synthetic_arrays(tangents=with_map, normal=with_map)
    data = GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'], a['images'], a['tangents'], GL.Z_UP_ROTATION)
    r = GL.read_glb(data)
    for k in ('positions', 'normals', 'texcoords', 'indices'):
        assert np.array_equal(r[k], a[k]) and r[k].dtype == a[k].dtype
    assert (r['tangents'] is None) == (not with_map)
    if with_map:
        assert np.array_equal(r['tangents'], a['tangents'])
    assert sorted(r['images']) == sorted(a['images'])
    assert all(np.array_equal(r['images'][k], a['images'][k]) for k in a['images'])
    assert r['rotation'] == GL.Z_UP_ROTATION
    assert data == GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'], a['images'], a['tangents'], GL.Z_UP_ROTATION)
    r0 = GL.read_glb(GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'], a['images'], a['tangents']))
    assert r0['rotation'] is None


def test_container_structure():
    a = synthetic_arrays(W=41, T=30, seed=3)
    data = GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'], a['images'], a['tangents'], GL.Z_UP_ROTATION)
    magic, version, length = struct.unpack('<III', data[:12])
    assert magic == 0x46546C67 and version == 2 and length == len(data)
    jl, jt = struct.unpack('<II', data[12:20])
    assert jt == 0x4E4F534A and jl % 4 == 0
    js = data[20:20 + jl]
    assert js == js.rstrip(b' ') + b' ' * (len(js) - len(js.rstrip(b' ')))
    doc = json.loads(js)
    bl, bt = struct.unpack('<II', data[20 + jl:28 + jl])
    assert bt == 0x004E4942 and bl % 4 == 0 and 28 + jl + bl == len(data)
    blob = data[28 + jl:]
    assert doc['asset']['version'] == '2.0' and doc['buffers'] == [{'byteLength': bl}]
    used = max(v['byteOffset'] + v['byteLength'] for v in doc['bufferViews'])
    assert blob[used:] == b'\0' * (bl - used)
    assert all(v['byteOffset'] % 4 == 0 for v in doc['bufferViews'])
    prim = doc['meshes'][0]['primitives'][0]
    assert sorted(prim['attributes']) == ['NORMAL', 'POSITION', 'TANGENT', 'TEXCOORD_0'] and prim['mode'] == 4
    acc = doc['accessors']
    for name, k in (('POSITION', 'VEC3'), ('NORMAL', 'VEC3'), ('TEXCOORD_0', 'VEC2'), ('TANGENT', 'VEC4')):
        x = acc[prim['attributes'][name]]
        assert x['componentType'] == 5126 and x['type'] == k and x['count'] == 41
    pos = acc[prim['attributes']['POSITION']]
    assert pos['min'] == [float(v) for v in a['positions'].min(0)] and pos['max'] == [float(v) for v in a['positions'].max(0)]
    ind = acc[prim['indices']]
    assert ind['componentType'] == 5125 and ind['type'] == 'SCALAR' and ind['count'] == 90
    assert int(GL.read_glb(data)['indices'].max()) < 41
    for img in doc['images']:
        v = doc['bufferViews'][img['bufferView']]
        assert img['mimeType'] == 'image/png' and blob[v['byteOffset']:v['byteOffset'] + 8] == b'\x89PNG\r\n\x1a\n'
    mat = doc['materials'][0]
    assert mat['pbrMetallicRoughness']['metallicFactor'] == 1 and mat['pbrMetallicRoughness']['roughnessFactor'] == 1
    assert mat['normalTexture'] == {'index': 2} and len(doc['textures']) == 3
    assert doc['samplers'] == [{'magFilter': 9729, 'minFilter': 9987, 'wrapS': 10497, 'wrapT': 10497}]


def test_read_glb_refuses_files_outside_the_subset():
    a = synthetic_arrays()
    data = GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'], a['images'], a['tangents'])
    with pytest.raises(ValueError):
        GL.read_glb(data[:8] + struct.pack('<I', 1) + data[12:])
    with pytest.raises(ValueError):
        GL.read_glb(b'glTF' + struct.pack('<II', 1, 20) + data[12:20])
    jl = struct.unpack('<I', data[12:16])[0]
    doc = json.loads(data[20:20 + jl])
    doc['bufferViews'][0]['byteStride'] = 12
    js = json.dumps(doc).encode()
    js += b' ' * ((4 - len(js) % 4) % 4)
    rest = data[20 + jl:]
    bad = struct.pack('<III', 0x46546C67, 2, 20 + len(js) + len(rest)) + struct.pack('<II', len(js), 0x4E4F534A) + js + rest
    with pytest.raises(ValueError, match='strided'):
        GL.read_glb(bad)
    with pytest.raises(ValueError):
        GL.glb_bytes(a['positions'], a['normals'], a['texcoords'], a['indices'] + 100, a['images'], a['tangents'])


def test_material_tables_follow_the_relighters_decoding():
    lut_m, lut_r = GL.material_tables()
    om, orr = OG.material_tables()
    assert np.array_equal(lut_m, om) and np.array_equal(lut_r, orr)
    k = np.arange(256)
    alpha = RL.srgb_to_linear(k / 255.0)              # UVMaterials' roughness: the BRDF's alpha itself
    assert np.abs(lut_r / 255.0 - np.sqrt(alpha)).max() <= 0.5 / 255 + 1e-12
    assert np.abs(lut_m / 255.0 - alpha).max() <= 0.5 / 255 + 1e-12
    assert lut_m[0] == lut_r[0] == 0 and lut_m[255] == lut_r[255] == 255 and (np.diff(lut_r.astype(int)) >= 0).all()


def test_oracle_weld_counts_distinct_pairs_in_first_corner_order():
    tris = np.array([[0, 1, 2], [2, 1, 3], [3, 1, 3]])     # the last triangle names vertex 3 twice
    ft = np.array([[0, 1, 2], [5, 1, 4], [4, 6, 7]])
    wv, wt, wf = OG.weld(tris, ft, 5)                        # vertex 4 has no triangle
    assert wv.tolist() == [0, 1, 1, 2, 2, 3, 3] and wt.tolist() == [0, 1, 6, 2, 5, 4, 7]
    assert wf.tolist() == [[0, 1, 3], [4, 1, 5], [5, 2, 6]]
    assert np.array_equal(wv[wf], tris) and np.array_equal(wt[wf], ft)


def quad(mirror=False, n=2):
    """A flat n x n grid in z = 0 over [0,1]^2, uv = (x, y) in the OBJ's convention ((1 - x, y) mirrored), wound so that the
    outward normal -cross(e1, e2) is +z."""
    g = np.linspace(0, 1, n + 1, dtype=np.float32)
    x, y = np.meshgrid(g, g)
    v = np.stack([x.ravel(), y.ravel(), np.zeros(x.size, np.float32)], -1)
    i = np.arange(n * n).reshape(n, n) // n * (n + 1) + np.arange(n * n).reshape(n, n) % n
    a, b, c, d = i.ravel(), i.ravel() + 1, i.ravel() + n + 2, i.ravel() + n + 1
    t = np.concatenate([np.stack([a, c, b], -1), np.stack([a, d, c], -1)]).astype(np.int32)
    vt = v[:, :2].copy()
    if mirror:
        vt[:, 0] = 1 - vt[:, 0]
    return v, t, vt, t.copy()


def oracle_export(v, t, vt, ft, omap):
    """weld, frames (cast to float32 as the file stores them) and the conversion on the oracle."""
    wv, wt, wf = OG.weld(t, ft, v.shape[0])
    wn, wtan = OG.frames(v, t, vt, ft, ON.vertex_normals(v, t), wv, wt, wf)
    wn, wtan = wn.astype(np.float32), wtan.astype(np.float32)
    img, fr = OG.tangent_space(vt, ft, wf, wn, wtan, omap)
    return dict(wv=wv, wt=wt, wf=wf, wn=wn, wtan=wtan, img=img, fr=fr)


def tilted(direction, h=16, w=16):
    return np.broadcast_to(ON.encode(direction / np.linalg.norm(direction)), (h, w, 3)).copy()


@pytest.mark.parametrize('mirror', [False, True])
def test_quad_conventions(mirror):
    v, t, vt, ft = quad(mirror)
    for d, channel in (((0.5, 0.0, 1.0), 0), ((0.0, 0.5, 1.0), 1)):
        o = oracle_export(v, t, vt, ft, tilted(np.array(d)))
        assert np.allclose(o['wn'], [0, 0, 1])
        assert np.allclose(o['wtan'][:, :3], [-1 if mirror else 1, 0, 0], atol=1e-6)
        assert (o['wtan'][:, 3] == (-1 if mirror else 1)).all()
        px = o['img'].reshape(-1, 5)[o['fr']['texel'], :3].astype(int)
        assert px.shape[0] > 100
        # +x tilt: R > 128 (R = the tangent's +u); mirrored, u runs along -x so R < 128.  +y tilt: G > 128 either way
        if channel == 0:
            assert ((px[:, 0] < 128) if mirror else (px[:, 0] > 128)).all()
        else:
            assert (px[:, 1] > 128).all()
        fr64 = OG.texel_frames(OG.atlas(vt), ft, o['wf'], o['wn'], o['wtan'], 16, 16, np.float64)
        got = OG.viewer_decode(o['img'], fr64)
        assert OG.angle_deg(got, np.broadcast_to(np.array(d, float), got.shape)).max() < 0.5


def sphere_export(size=64):
    v, f = synthetic.icosphere(3, 0.5)
    t = np.ascontiguousarray(f[:, [0, 2, 1]]).astype(np.int32)
    v = v.astype(np.float32)
    vt_atlas, ft = TX.uv_atlas(v, t, size, size, 2)
    vt = np.stack([vt_atlas[:, 0], np.float32(1) - vt_atlas[:, 1]], -1)     # as the OBJ stores it
    return v, t, vt, ft


def test_identity_map_converts_to_the_flat_normal():
    v, t, vt, ft = sphere_export()
    wv, wt, wf = OG.weld(t, ft, v.shape[0])
    wn, wtan = (a.astype(np.float32) for a in OG.frames(v, t, vt, ft, ON.vertex_normals(v, t), wv, wt, wf))
    fr = OG.texel_frames(OG.atlas(vt), ft, wf, wn, wtan, 64, 64)
    omap = np.zeros((64 * 64, 3), np.uint8)
    omap[fr['texel']] = ON.encode(fr['N'])                 # the interpolated vertex normal: a self-bake's map
    img, _ = OG.tangent_space(vt, ft, wf, wn, wtan, omap.reshape(64, 64, 3))
    px = img.reshape(-1, 5)[fr['texel'], :3].astype(int)
    assert px.shape[0] > 1000
    assert np.abs(px - [128, 128, 255]).max() <= 1


def test_decode_recovers_the_object_space_map():
    """The bounds come from 8-bit quantisation of both maps: within 1 degree at >= 99.9 % of covered texels, median <= 0.4."""
    v, t, vt, ft = sphere_export(128)
    wv, wt, wf = OG.weld(t, ft, v.shape[0])
    wn, wtan = (a.astype(np.float32) for a in OG.frames(v, t, vt, ft, ON.vertex_normals(v, t), wv, wt, wf))
    fr = OG.texel_frames(OG.atlas(vt), ft, wf, wn, wtan, 128, 128)
    rng = np.random.RandomState(5)
    d = fr['N'].astype(np.float64) + 0.6 * rng.randn(fr['texel'].size, 3)
    omap = np.zeros((128 * 128, 3), np.uint8)
    omap[fr['texel']] = ON.encode(d / np.linalg.norm(d, axis=1, keepdims=True))
    img, _ = OG.tangent_space(vt, ft, wf, wn, wtan, omap.reshape(128, 128, 3))
    got = OG.viewer_decode(img, OG.texel_frames(OG.atlas(vt), ft, wf, wn, wtan, 128, 128, np.float64))
    err = OG.angle_deg(got, ON.decode(omap[fr['texel']]).astype(np.float64))
    print(f'decode: {err.size} texels, median {np.median(err):.3f} deg, 99.9th percentile {np.percentile(err, 99.9):.3f}, max {err.max():.3f}')
    assert (err <= 1.0).mean() >= 0.999 and np.median(err) <= 0.4


def test_tool_refuses_bad_arguments(tmp_path):
    v, t, vt, ft = quad()
    maps = (np.full((8, 8, 3), 100, np.uint8), np.full((8, 8, 3), 20, np.uint8), np.full((8, 8, 3), 150, np.uint8))
    TX.write_textured_obj(str(tmp_path), v, t, np.stack([vt[:, 0], 1 - vt[:, 1]], -1), ft, maps)
    import cv2
    cv2.imwrite(str(tmp_path / 'grey.png'), np.full((8, 8), 128, np.uint8))
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, os.path.join(TOOLS, 'export_gltf.py'), *a], cwd=tmp_path, env=env,
                                    capture_output=True, text=True)
    r = run('--obj', 'missing.obj')
    assert r.returncode != 0 and 'no such file' in r.stderr
    r = run('--obj', 'mesh_0.obj', '--normal-map', 'missing.png')
    assert r.returncode != 0 and 'no such file' in r.stderr
    r = run('--obj', 'mesh_0.obj', '--normal-map', 'grey.png')
    assert r.returncode != 0 and '8-bit RGB' in r.stderr
    os.remove(tmp_path / 'feat2_0.png')
    r = run('--obj', 'mesh_0.obj')
    assert r.returncode != 0 and 'feat2_0.png' in r.stderr
