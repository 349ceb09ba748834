"""CPU: the texture-map oracle against the reference fixtures (tests/golden/texmap_*.npz), the OBJ / MTL writer byte for byte,
the host UV unwrapper through ctypes (coverage, injectivity, gutters, uniform density, determinism) and the bindings of
include/nero_texmap.h.  No GPU."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mat as OM
import nero_oracle_mesh as OMesh
import nero_oracle_texmap as OT
from nero_b200 import texmap as TX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
FIXTURES = ['texmap_scene_32x32', 'texmap_blob_40x64']


def load(name):
    return np.load(os.path.join(GOLD, name + '.npz'))


# ------------------------------------------------------------------------------------------------ oracle vs reference
@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_matches_reference_fixture(name):
    from nero_b200 import params as P
    g = load(name)
    h, w = g['mask'].shape
    owner, count, bary = OT.rasterize(g['vt'], g['ft'], w, h)
    np.testing.assert_array_equal(owner >= 0, g['mask'])
    assert count.max() <= 1
    xyz = OT.interpolate(g['verts'], g['tris'], owner, bary)[g['mask']]
    np.testing.assert_array_equal(xyz, g['xyzs'])
    scfg = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}
    sd = O.perturb_params(P.build_material_state_dict(scfg, seed=int(g['seed'])), seed=int(g['pseed']))
    with torch.no_grad():
        m, r, a = OM.predict_materials(sd, torch.from_numpy(xyz))
    mat = torch.cat([a, m, r], 1).float().numpy()
    before = OT.encode(mat, g['mask'])
    d = before.astype(int) - g['img_before'].astype(int)
    assert np.abs(d).max() <= 1 and (d == 0).mean() >= 0.995
    after, src = OT.inpaint(g['img_before'], g['mask'])
    src = src.reshape(-1)
    ti, ts = g['inpaint_texels'], g['inpaint_src']
    np.testing.assert_array_equal(np.flatnonzero(src >= 0), np.sort(ti))
    d2 = lambda a, b: (a // w - b // w) ** 2 + (a % w - b % w) ** 2
    np.testing.assert_array_equal(d2(ti, src[ti]), d2(ti, ts))
    same = src[ti] == ts
    assert same.mean() > 0.5
    np.testing.assert_array_equal(after.reshape(-1, 5)[ti[same]], g['img_after'].reshape(-1, 5)[ti[same]])
    ds = OT.downsample(g['img_after'])
    np.testing.assert_array_equal(ds[..., :3], g['feat0'][..., ::-1])
    np.testing.assert_array_equal(np.repeat(ds[..., 3:4], 3, -1), g['feat1'])
    np.testing.assert_array_equal(np.repeat(ds[..., 4:5], 3, -1), g['feat2'])


@pytest.mark.parametrize('name', FIXTURES)
def test_obj_and_mtl_text_match_reference(name, tmp_path):
    g = load(name)
    obj, mtl = TX.obj_text(g['verts'], g['tris'], g['vt'], g['ft'])
    assert obj == str(g['obj'])
    assert mtl == str(g['mtl']).replace('feat0_0.jpg', 'feat0_0.png')
    assert (obj, str(g['mtl'])) == OT.obj_text(g['verts'], g['tris'], g['vt'], g['ft'])
    imgs = TX.split_images(np.zeros((4, 6, 5), np.uint8))
    TX.write_textured_obj(str(tmp_path), g['verts'], g['tris'], g['vt'], g['ft'], imgs)
    assert (tmp_path / 'mesh_0.obj').read_bytes() == str(g['obj']).encode()
    assert sorted(os.listdir(tmp_path)) == ['feat0_0.png', 'feat1_0.png', 'feat2_0.png', 'mesh_0.mtl', 'mesh_0.obj']


def test_write_png_rgba_output_is_unchanged(tmp_path):
    """write_png_rgba is write_png on RGBA: same bytes as the direct encoding (colour type 6, filter 0, zlib level 6)."""
    import struct
    import zlib
    from nero_b200.relight import write_png, write_png_rgba
    rgba = np.random.RandomState(0).randint(0, 256, (5, 7, 4)).astype(np.uint8)
    write_png_rgba(str(tmp_path / 'a.png'), rgba)
    raw = np.concatenate([np.zeros((5, 1), np.uint8), rgba.reshape(5, 28)], 1).tobytes()
    chunk = lambda t, b: struct.pack('>I', len(b)) + t + b + struct.pack('>I', zlib.crc32(t + b) & 0xffffffff)
    want = (b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', 7, 5, 8, 6, 0, 0, 0)) + chunk(b'IDAT', zlib.compress(raw, 6)) +
            chunk(b'IEND', b''))
    assert (tmp_path / 'a.png').read_bytes() == want
    write_png(str(tmp_path / 'b.png'), rgba[..., :3])
    assert (tmp_path / 'b.png').read_bytes()[24:26] == bytes([8, 2])
    with pytest.raises(ValueError):
        write_png_rgba(str(tmp_path / 'c.png'), rgba[..., :3])


# ------------------------------------------------------------------------------------------------ unwrapper
def mc_mesh(fn, n=64):
    ax = np.linspace(-1.0, 1.0, n)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    v, t = OMesh.marching_cubes(fn(x).astype(np.float32), 0.0)
    return v.astype(np.float32), t.astype(np.int32)


def plane_grid(n=12):
    ij = np.stack(np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing='ij'), -1).reshape(-1, 2)
    v = np.concatenate([ij / n, np.zeros((ij.shape[0], 1))], 1).astype(np.float32)
    a = (np.arange(n)[:, None] * (n + 1) + np.arange(n)[None, :]).reshape(-1)
    return v, np.concatenate([np.stack([a, a + n + 1, a + n + 2], 1), np.stack([a, a + n + 2, a + 1], 1)]).astype(np.int32)


def helicoid(n=24, m=6, turns=3.0):
    """Several turns over the same footprint: a chart that kept growing would overlap itself in projection."""
    s, r = np.meshgrid(np.linspace(0, 1, n * 4 + 1), np.linspace(0.2, 1.0, m + 1), indexing='ij')
    th = 2 * np.pi * turns * s
    v = np.stack([r * np.cos(th), r * np.sin(th), 0.15 * s], -1).reshape(-1, 3).astype(np.float32)
    a = (np.arange(n * 4)[:, None] * (m + 1) + np.arange(m)[None, :]).reshape(-1)
    return v, np.concatenate([np.stack([a, a + m + 1, a + m + 2], 1), np.stack([a, a + m + 2, a + 1], 1)]).astype(np.int32)


def messy_mesh():
    """A grid with zero-area, repeated-index, duplicate and non-manifold (three triangles on one edge) faces."""
    v, t = plane_grid(6)
    extra_v = np.asarray([[0.5, 0.5, 0.7], [2.0, 2.0, 0.0], [2.0, 2.0, 0.0], [2.0, 2.0, 0.0], [3.0, 2.0, 0.0], [4.0, 2.0, 0.0]], np.float32)
    V = v.shape[0]
    extra_t = np.asarray([[0, 1, V], [V + 1, V + 2, V + 3], [V + 1, V + 4, V + 5], [3, 3, 4], t[5], t[7][[0, 2, 1]]], np.int32)
    return np.concatenate([v, extra_v]), np.concatenate([t, extra_t])


def bell(x):
    """a bell: a sphere pinched towards +z with a wavy rim"""
    y = np.concatenate([x[..., :2], x[..., 2:] * (1.4 - 0.5 * x[..., 2:])], -1)
    return np.linalg.norm(y, axis=-1) - 0.6 + 0.08 * np.sin(6 * x[..., 0]) * np.cos(5 * x[..., 1])


MESHES = {
    'scene': lambda: OM.test_scene(2),
    'sphere64': lambda: mc_mesh(lambda x: np.linalg.norm(x, axis=-1) - 0.7),
    'bell64': lambda: mc_mesh(bell),
    'plane': plane_grid,
    'helicoid': helicoid,
    'messy': messy_mesh,
}


def _orient(a, b, c):
    """exact orientation of integer points (Python ints): rows of [..., 2] object arrays"""
    return (b[..., 0] - a[..., 0]) * (c[..., 1] - a[..., 1]) - (b[..., 1] - a[..., 1]) * (c[..., 0] - a[..., 0])


def candidate_pairs(lo, hi, pad=0.0):
    """pairs (i < j) of boxes [lo, hi] (texels) that overlap after growing by pad, found with a uniform grid"""
    cell = max(float(np.max(hi - lo)) + 2 * pad, 1.0)
    buckets = {}
    c0, c1 = np.floor((lo - pad) / cell).astype(int), np.floor((hi + pad) / cell).astype(int)
    for i in range(lo.shape[0]):
        for cx in range(c0[i, 0], c1[i, 0] + 1):
            for cy in range(c0[i, 1], c1[i, 1] + 1):
                buckets.setdefault((cx, cy), []).append(i)
    pairs = set()
    for b in buckets.values():
        for x in range(len(b)):
            for y in range(x + 1, len(b)):
                pairs.add((b[x], b[y]))
    if not pairs:
        return np.zeros((0, 2), int)
    p = np.asarray(sorted(pairs))
    keep = np.all(lo[p[:, 0]] - pad <= hi[p[:, 1]] + pad, 1) & np.all(lo[p[:, 1]] - pad <= hi[p[:, 0]] + pad, 1)
    return p[keep]


def check_atlas(verts, tris, vt, ft, W, H, g):
    T = tris.shape[0]
    assert ft.shape == (T, 3) and ft.min() >= 0 and ft.max() < vt.shape[0]
    assert np.isfinite(vt).all()
    eps = 1e-6
    assert (vt[:, 0] >= g / W - eps).all() and (vt[:, 0] <= 1 - g / W + eps).all()
    assert (vt[:, 1] >= g / H - eps).all() and (vt[:, 1] <= 1 - g / H + eps).all()
    uv = vt[ft].astype(np.float64) * [W, H]                       # [T,3,2] texels
    # exact predicates: float32 uv in [2^-9, 1) are integer multiples of 2^-33
    q = np.round(vt.astype(np.float64) * 2.0 ** 33).astype(np.int64).astype(object)[ft]
    area = _orient(q[:, 0], q[:, 1], q[:, 2])
    pos = np.asarray([a > 0 for a in area])
    neg = np.asarray([a < 0 for a in area])
    q = np.where(neg[:, None, None], q[:, [0, 2, 1]], q)
    lo, hi = uv.min(1), uv.max(1)
    # no two uv triangles have overlapping interiors
    pairs = candidate_pairs(lo, hi)
    pairs = pairs[(pos | neg)[pairs[:, 0]] & (pos | neg)[pairs[:, 1]]]
    if pairs.shape[0]:
        A, B = q[pairs[:, 0]], q[pairs[:, 1]]
        sep = np.zeros(pairs.shape[0], bool)
        for P_, Q_ in ((A, B), (B, A)):
            for e in range(3):
                u, v = P_[:, e], P_[:, (e + 1) % 3]
                s = np.ones(pairs.shape[0], bool)
                for k in range(3):
                    s &= np.asarray([x <= 0 for x in _orient(u, v, Q_[:, k])])
                sep |= s
        assert sep.all(), f'{(~sep).sum()} overlapping uv triangle pairs'
    # charts (triangles joined through shared uv vertices) are at least g texels apart
    parent = np.arange(vt.shape[0])

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x
    for a, b, c in ft:
        for u_ in (b, c):
            ra, rb = find(a), find(u_)
            if ra != rb:
                parent[max(ra, rb)] = min(ra, rb)
    chart = np.asarray([find(f[0]) for f in ft])
    pairs = candidate_pairs(lo, hi, pad=g / 2)
    pairs = pairs[chart[pairs[:, 0]] != chart[pairs[:, 1]]]

    def pt_seg(p, a, b):
        ab = b - a
        t = np.clip(np.sum((p - a) * ab, -1) / np.maximum(np.sum(ab * ab, -1), 1e-300), 0, 1)
        return np.linalg.norm(p - a - t[:, None] * ab, axis=-1)
    if pairs.shape[0]:
        d = np.full(pairs.shape[0], np.inf)
        for P_, Q_ in ((uv[pairs[:, 0]], uv[pairs[:, 1]]), (uv[pairs[:, 1]], uv[pairs[:, 0]])):
            for k in range(3):
                for e in range(3):
                    d = np.minimum(d, pt_seg(P_[:, k], Q_[:, e], Q_[:, (e + 1) % 3]))
        assert d.min() >= g - 1e-3, d.min()
    # one texel density: uv area / world area within [1/2, 1] s^2 on the triangles with an interior
    p = verts[tris].astype(np.float64)
    wa = 0.5 * np.linalg.norm(np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]), axis=-1)
    ua = 0.5 * np.abs((uv[:, 1, 0] - uv[:, 0, 0]) * (uv[:, 2, 1] - uv[:, 0, 1]) - (uv[:, 1, 1] - uv[:, 0, 1]) * (uv[:, 2, 0] - uv[:, 0, 0]))
    ok = wa > 1e-6 * np.median(wa[wa > 0])
    ratio = ua[ok] / wa[ok]
    s2 = np.median(ratio[ratio > 0]) if (ratio > 0).any() else 0.0
    big = ua[ok] > 0.05                                           # texel-scale triangles: fp32 uv resolves their area
    assert (ratio[big] <= 1.0 * ratio[big].max()).all()
    assert ratio[big].min() >= 0.5 * ratio[big].max() * (1 - 1e-3), (ratio[big].min(), ratio[big].max(), s2)


@pytest.mark.parametrize('name', list(MESHES))
def test_unwrapper_properties(name):
    verts, tris = MESHES[name]()
    W, H, g = (512, 384, 4)
    vt, ft = TX.uv_atlas(verts, tris, W, H, g)
    check_atlas(verts, tris, vt, ft, W, H, g)
    vt2, ft2 = TX.uv_atlas(verts, tris, W, H, g)
    assert vt.tobytes() == vt2.tobytes() and ft.tobytes() == ft2.tobytes()


def test_helicoid_is_split_into_injective_charts():
    verts, tris = helicoid()
    vt, ft = TX.uv_atlas(verts, tris, 512, 512, 4)
    assert vt.shape[0] > verts.shape[0]          # the turns overlap in projection, so there is more than one chart


def test_unwrapper_rejects_bad_input():
    verts, tris = plane_grid(2)
    with pytest.raises(RuntimeError):
        TX.uv_atlas(verts, tris + 100, 64, 64, 2)
    with pytest.raises(RuntimeError):
        TX.uv_atlas(verts, tris, 8, 8, 4)
    bad = verts.copy()
    bad[0, 0] = np.nan
    with pytest.raises(RuntimeError):
        TX.uv_atlas(bad, tris, 64, 64, 2)


# ------------------------------------------------------------------------------------------------ bindings
def test_texmap_header_is_bound():
    """Every prototype of include/nero_texmap.h is exported by the library and bound with one argtype per parameter."""
    from nero_b200 import ops
    txt = re.sub(r'/\*.*?\*/', ' ', open(os.path.join(ROOT, 'include', 'nero_texmap.h')).read(), flags=re.S)
    protos = dict(re.findall(r'\bint\s+(nero_[a-z0-9_]+)\s*\(([^)]*)\)', txt))
    assert len(protos) == 7 and set(protos) == set(ops.TEXMAP_PROTOS)
    for name, params in protos.items():
        fn = getattr(ops.lib, name)
        assert fn.argtypes is not None and len(fn.argtypes) == params.count(',') + 1 and fn.restype is ctypes.c_int, name
    with pytest.raises(ctypes.ArgumentError):
        ops.lib.nero_tex_downsample(None, 2.0, 2, None, None)
