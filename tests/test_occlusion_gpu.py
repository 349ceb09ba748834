"""GPU: the ambient-occlusion bake.  Convex meshes are exactly unoccluded (and the inverted mesh exactly occluded), the counts
match two analytic cases and the numpy oracle per texel in both sources, the self-bake points are the texture export's,
bakes are deterministic and keyed by texel, and the glTF export packs the map without changing the file when there is none;
tools/bake_occlusion.py -> tools/export_gltf.py --occlusion end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_mat as OM
import nero_oracle_occlusion as OO
from nero_b200 import gltf as GL
from nero_b200 import occlusion as OC
from nero_b200 import texmap as TX
from test_normalmap_gpu import low_and_detail

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def icospheres():
    lov, lof = OM.icosphere(1, 0.5)
    dev_, def_ = OM.icosphere(3, 0.5)
    return (lov.astype(np.float32), np.ascontiguousarray(lof[:, [0, 2, 1]]).astype(np.int32), dev_.astype(np.float32),
            np.ascontiguousarray(def_[:, [0, 2, 1]]).astype(np.int32))


def test_convex_meshes_are_unoccluded_exactly():
    lov, lof, dev_, def_ = icospheres()
    vt, ft = TX.uv_atlas(lov, lof, 64, 64, 2)
    s = OC.bake_cuda(lov, lof, vt, ft, 64, ssaa=1, rays=128)
    n = s['counts'].shape[0]
    assert n > 300 and bool((s['counts'] == 128).all()) and bool((s['hit'] == 1).all())
    img = s['img'].reshape(-1, 5)
    cov = s['raster']['texel'].long()
    assert bool((img[cov, :3] == 255).all()) and bool((img[:, 3:] == 0).all())
    d = OC.bake_cuda(lov, lof, vt, ft, 64, dev_, def_, ssaa=1, rays=128, cage_distance=0.05)
    assert bool((d['hit'] == 1).all()) and bool((d['counts'] == 128).all())
    assert bool((d['img'].reshape(-1, 5)[cov, :3] == 255).all())


def test_the_inverted_sphere_is_occluded_everywhere():
    """Wound the other way the flat 'outward' normal points into the sphere, so with a distance beyond the diameter every
    ray starts inside a closed mesh and hits it: counts are 0 except on rays the oracle flags as ties."""
    lov, lof, _, _ = icospheres()
    inv = np.ascontiguousarray(lof[:, [0, 2, 1]])
    vt, ft = TX.uv_atlas(lov, inv, 64, 64, 2)
    b = OC.bake_cuda(lov, inv, vt, ft, 64, ssaa=1, rays=64, distance=2.0)
    counts = b['counts'].cpu().numpy()
    oc, ties = OO.counts(b['point'].cpu().numpy(), b['normal'].cpu().numpy(), lov, inv, 64, 2.0, 0, b['key'].cpu().numpy())
    assert counts.size > 300 and (oc <= ties).all() and ties.sum() < 0.01 * counts.size * 64
    assert (counts <= ties).all(), f'{int((counts > ties).sum())} texels see out of the closed mesh'


@pytest.mark.parametrize('ratio', [0.2, 0.5, 0.8])
def test_ceiling_fraction_is_h_over_d_squared(ratio):
    """A point with normal +z under a two-triangle ceiling at height H, distance D > H: a cosine-weighted ray escapes within D
    iff cos(theta) < H / D, which has probability (H/D)^2.  4096 rays per point, 64 keys, within 4 binomial sigma."""
    D, H = 1.0, ratio
    E = 10 * D
    verts = np.asarray([[-E, -E, H], [E, -E, H], [E, E, H], [-E, E, H]], np.float32)
    tris = np.asarray([[0, 1, 2], [0, 2, 3]], np.int32)
    rows, rays = 64, 4096
    c = OC.points(np.zeros((rows, 3), np.float32), np.tile(np.float32([[0, 0, 1]]), (rows, 1)), verts, tris, rays, D, seed=3,
                  keys=np.arange(rows))
    frac, p = c.sum() / (rows * rays), ratio ** 2
    sigma = np.sqrt(p * (1 - p) / (rows * rays))
    print(f'ceiling H/D {ratio}: fraction {frac:.5f}, expected {p:.5f}, sigma {sigma:.2e}')
    assert abs(frac - p) <= 4 * sigma


@pytest.mark.parametrize('r,h', [(0.3, 0.3), (0.2, 0.5), (0.5, 0.2)])
def test_well_floor_fraction(r, h):
    """The floor centre of an open 256-gon well of radius r and depth h, distance beyond the rim: a ray escapes iff
    sin^2(theta) <= r^2 / (r^2 + h^2), the expected fraction."""
    k = 256
    a = 2 * np.pi * np.arange(k) / k
    ring = np.stack([r * np.cos(a), r * np.sin(a)], -1)
    verts = np.concatenate([np.c_[ring, np.zeros(k)], np.c_[ring, np.full(k, h)]]).astype(np.float32)
    i, j = np.arange(k), (np.arange(k) + 1) % k
    tris = np.concatenate([np.stack([i, j, k + j], -1), np.stack([i, k + j, k + i], -1)]).astype(np.int32)
    rows, rays = 64, 4096
    D = 2.0 * np.hypot(r, h)
    c = OC.points(np.zeros((rows, 3), np.float32), np.tile(np.float32([[0, 0, 1]]), (rows, 1)), verts, tris, rays, D, seed=5,
                  keys=np.arange(rows) + 1000)
    frac, p = c.sum() / (rows * rays), r * r / (r * r + h * h)
    sigma = np.sqrt(p * (1 - p) / (rows * rays))
    print(f'well r {r} h {h}: fraction {frac:.5f}, expected {p:.5f}, sigma {sigma:.2e}')
    assert abs(frac - p) <= 4 * sigma


def small_meshes():
    return low_and_detail(40, 32, 600)


def torus_meshes():
    """The marching-cubes torus of test_normalmap_gpu.py at 40^3 and its 32^3 mesh simplified to 800 triangles: its inner
    ring sees the far side across the hole, so a distance of 0.6 occludes part of the hemisphere on about a fifth of the
    texels (the bumpy sphere occludes almost nothing)."""
    from nero_b200.simplify import simplify
    from test_normalmap_gpu import mc_mesh
    dv, dt = mc_mesh(40, 'torus')
    lv, lt, _ = simplify(*mc_mesh(32, 'torus'), 800)
    return lv, lt, dv, dt


@pytest.mark.parametrize('source', ['self', 'detail'])
def test_bake_matches_the_oracle(source):
    lv, lt, dv, dt = torus_meshes()
    vt, ft = TX.uv_atlas(lv, lt, 48, 48, 2)
    det = (dv, dt) if source == 'detail' else (None, None)
    rays, dist = 32, 0.6
    b = OC.bake_cuda(lv, lt, vt, ft, 48, *det, ssaa=1, rays=rays, distance=dist, seed=11)
    o = OO.bake_texels(lv, lt, vt, ft, 48, 48, *det, rays=rays, distance=dist, seed=11)
    g = {k: b[k].cpu().numpy() for k in ('counts', 'hit', 'point', 'normal', 'key', 'surface', 'cage')}
    assert np.array_equal(b['raster']['texel'].cpu().numpy(), o['texel']) and np.array_equal(g['key'], o['key'])
    assert np.array_equal(g['surface'], o['surface']) and np.array_equal(g['cage'], o['cage'])
    if source == 'self':
        assert np.array_equal(g['point'], o['point']) and np.array_equal(g['normal'], o['normal'])
    else:
        ok = ~o['cage_tie']
        assert np.array_equal(g['hit'].astype(bool)[ok], o['hit'][ok]) and o['hit'].mean() > 0.9
        same = ok & o['hit']
        assert np.abs(g['point'] - o['point'])[same].max() <= 1e-6
        assert np.array_equal(g['normal'][same], o['normal'][same])
    ties = o['ties']
    n = ties.size
    print(f'{source}: {n} texels x {rays} rays, {int(ties.sum())} tie rays, mean unoccluded {o["counts"].mean() / rays:.4f}')
    assert np.all(np.abs(g['counts'] - o['counts']) <= ties)
    assert n > 300 and ties.sum() < 0.01 * n * rays and (o['counts'] < rays).mean() > 0.1
    img, ref = b['img'].cpu().numpy().reshape(-1, 5), o['img'].reshape(-1, 5)
    clean = o['texel'][ties == 0]
    assert np.array_equal(img[clean], ref[clean]) and (img[o['owner'].reshape(-1) < 0] == 0).all()


def test_self_bake_points_are_the_texture_exports_points():
    lv, lt, _, _ = small_meshes()
    vt, ft = TX.uv_atlas(lv, lt, 64, 64, 2)
    b = OC.bake_cuda(lv, lt, vt, ft, 64, ssaa=1, rays=8)
    r = TX.raster(vt, ft, lv, lt, 64, 64)
    assert b['point'].shape[0] > 500 and torch.equal(b['point'], r['xyz']) and torch.equal(b['raster']['texel'], r['texel'])


def test_determinism_seeds_and_keys():
    lv, lt, dv, dt = small_meshes()
    vt, ft = TX.uv_atlas(lv, lt, 128, 128, 2)
    a, sa = OC.bake(lv, lt, vt, ft, 64, dv, dt, rays=64)
    b, sb = OC.bake(lv, lt, vt, ft, 64, dv, dt, rays=64)
    assert np.array_equal(a, b) and sa == sb and a.shape == (64, 64, 3)
    assert (a[..., 0] == a[..., 1]).all() and (a[..., 1] == a[..., 2]).all()
    c, _ = OC.bake(lv, lt, vt, ft, 64, dv, dt, rays=64, seed=1)
    assert not np.array_equal(a, c)
    k = OC.bake_cuda(lv, lt, vt, ft, 64, ssaa=2, rays=64)
    pts = OC.points(k['point'], k['normal'], lv, lt, 64, OC.DISTANCE, 0, keys=k['key'])
    assert np.array_equal(pts, k['counts'].cpu().numpy())
    # rows in another order with the same keys count the same rays
    perm = torch.randperm(k['point'].shape[0], generator=torch.Generator().manual_seed(0)).cuda()
    pp = OC.points(k['point'][perm], k['normal'][perm], lv, lt, 64, OC.DISTANCE, 0, keys=k['key'][perm])
    assert np.array_equal(pp, k['counts'][perm].cpu().numpy())


def textured_obj(tmp_path):
    from nero_b200.mesh import write_ply
    lv, lt, dv, dt = small_meshes()
    vt, ft = TX.uv_atlas(lv, lt, 64, 64, 2)
    rng = np.random.RandomState(1)
    maps = (rng.randint(60, 200, (32, 32, 3)).astype(np.uint8), rng.randint(0, 256, (32, 32, 3)).astype(np.uint8),
            rng.randint(0, 256, (32, 32, 3)).astype(np.uint8))
    TX.write_textured_obj(str(tmp_path / 'n2m'), lv, lt, vt, ft, maps)
    write_ply(str(tmp_path / 'detail.ply'), dv, dt)
    return str(tmp_path / 'n2m' / 'mesh_0.obj'), (lv, lt, vt, ft)


def test_gltf_packs_the_map_and_leaves_the_file_alone_without_one(tmp_path):
    obj, (lv, lt, vt, ft) = textured_obj(tmp_path)
    plain = GL.export(obj)
    assert plain == GL.export(obj, occlusion_path=None)
    img, _ = OC.bake(lv, lt, vt, ft, 32, rays=32)
    occ = str(tmp_path / 'n2m' / 'occlusion_0.png')
    OC.write_occlusion_map(occ, img)
    a, b = GL.read_glb(plain), GL.read_glb(GL.export(obj, occlusion_path=occ))
    assert a['occlusion'] is None and 'occlusionTexture' not in a['json']['materials'][0]
    assert b['json']['materials'][0]['occlusionTexture'] == {'index': 1}
    assert np.array_equal(b['occlusion'], img[..., 0]) and np.array_equal(b['images']['metallic_roughness'][..., 0], img[..., 0])
    assert np.array_equal(b['images']['metallic_roughness'][..., 1:], a['images']['metallic_roughness'][..., 1:])
    assert (a['images']['metallic_roughness'][..., 0] == 255).all()
    for k in ('positions', 'normals', 'texcoords', 'indices'):
        assert np.array_equal(a[k], b[k])


def test_tools_end_to_end(tmp_path):
    textured_obj(tmp_path)
    env = dict(os.environ, PYTHONPATH=ROOT)
    tools = os.path.join(ROOT, 'tools')
    out = subprocess.run([sys.executable, os.path.join(tools, 'bake_occlusion.py'), '--obj', 'n2m/mesh_0.obj', '--detail', 'detail.ply',
                          '--rays', '64'], cwd=tmp_path, env=env, capture_output=True, text=True, check=True).stdout
    assert 'misses' in out and 'mean occlusion' in out and 'bvh' in out and (tmp_path / 'n2m' / 'occlusion_0.png').exists()
    occ = OC.read_occlusion_map(str(tmp_path / 'n2m' / 'occlusion_0.png'))
    assert occ.shape == (32, 32) and occ.min() < 255
    subprocess.run([sys.executable, os.path.join(tools, 'export_gltf.py'), '--obj', 'n2m/mesh_0.obj', '--occlusion', 'n2m/occlusion_0.png'],
                   cwd=tmp_path, env=env, capture_output=True, text=True, check=True)
    g = GL.read_glb(str(tmp_path / 'n2m' / 'mesh_0.glb'))
    assert np.array_equal(g['occlusion'], occ) and g['occlusion_strength'] == 1.0
