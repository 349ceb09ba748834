"""GPU: the normal-map bake against the numpy oracle (vertex normals bit for bit, bake points bit for bit with the texture
export's, hits and normals per texel), self-bakes, determinism, the normal-mapped relight kernel against its oracle, the
quality a baked map buys a simplified mesh, and tools/bake_normal_map.py -> tools/relight.py --normal-map end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_mat as OM
import nero_oracle_normalmap as ON
import nero_oracle_texmap as OT
from nero_b200 import normalmap as NM
from nero_b200 import relight as RL
from nero_b200 import texmap as TX
from test_relight_gpu import random_env, scene_camera
from test_relight_tex_gpu import random_uv_materials

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def mc_mesh(n, kind='bumpy'):
    """A marching-cubes mesh of an analytic field on an n^3 grid over [-1, 1]^3 (float32 verts, int32 tris)."""
    from nero_b200.mesh import marching_cubes
    ax = np.linspace(-1.0, 1.0, n)
    x = np.stack(np.meshgrid(ax, ax, ax, indexing='ij'), -1)
    if kind == 'bumpy':
        u = np.linalg.norm(x, axis=-1) - 0.6 + 0.05 * np.sin(9 * x[..., 0]) * np.cos(8 * x[..., 1] + 2 * x[..., 2])
    else:
        u = np.sqrt((np.hypot(x[..., 0], x[..., 1]) - 0.55) ** 2 + x[..., 2] ** 2) - 0.22
    v, t = marching_cubes(u.astype(np.float32), 0.0)
    return (v * (2.0 / (n - 1)) - 1.0).astype(np.float32), t.astype(np.int32)


def low_and_detail(n_detail, n_low, faces):
    from nero_b200.simplify import simplify
    dv, dt = mc_mesh(n_detail)
    lv, lt, _ = simplify(*mc_mesh(n_low), faces)
    return lv, lt, dv, dt


@pytest.mark.parametrize('kind', ['bumpy', 'torus'])
def test_vertex_normals_match_the_oracle_bit_for_bit(kind):
    v, t = mc_mesh(96, kind)
    got = NM.vertex_normals(v, t)
    ref = ON.vertex_normals(v, t)
    assert t.shape[0] > 10000 and np.array_equal(got.view(np.uint32), ref.view(np.uint32))
    assert np.allclose(np.linalg.norm(got, axis=1), 1, atol=1e-6)


def test_bake_points_are_the_texture_exports_points():
    lv, lt, dv, dt = low_and_detail(64, 64, 1500)
    vt, ft = TX.uv_atlas(lv, lt, 128, 128, 2)
    b = NM.bake_cuda(lv, lt, vt, ft, dv, dt, 128, ssaa=1)
    r = TX.raster(vt, ft, lv, lt, 128, 128)
    assert b['point'].shape[0] > 1000
    assert torch.equal(b['point'], r['xyz']) and torch.equal(b['raster']['texel'], r['texel'])


def test_bake_matches_the_oracle():
    lv, lt, dv, dt = low_and_detail(64, 48, 1000)
    vt, ft = TX.uv_atlas(lv, lt, 64, 64, 2)
    b = NM.bake_cuda(lv, lt, vt, ft, dv, dt, 64, ssaa=1)
    o = ON.bake_texels(lv, lt, vt, ft, dv, dt, 64, 64)
    assert np.array_equal(b['raster']['texel'].cpu().numpy(), o['texel'])
    assert np.array_equal(b['point'].cpu().numpy(), o['point']) and np.array_equal(b['cage'].cpu().numpy(), o['cage'])
    tie = o['tie']
    hit = b['hit'].cpu().numpy().astype(bool)
    print(f'bake vs oracle: {tie.size} texels, {int(o["hit"].sum())} hits, {int(tie.sum())} near ties')
    assert tie.mean() < 0.01 and o['hit'].mean() > 0.9
    assert np.array_equal(hit[~tie], o['hit'][~tie])
    nrm = b['normal'].cpu().numpy().astype(np.float64)
    assert np.abs(nrm - o['normal'])[~tie].max() <= 1e-5
    img = b['img'].cpu().numpy().reshape(-1, 5)
    ref = o['img'].reshape(-1, 5)
    keep = np.ones(img.shape[0], bool)
    keep[o['texel'][tie]] = False
    assert np.abs(img[keep].astype(int) - ref[keep]).max() <= 1 and (img[:, 3:] == 0).all()
    assert (img[o['owner'].reshape(-1) < 0] == 0).all()


def test_self_bake_reproduces_the_cage_direction():
    from nero_b200.simplify import simplify
    lv, lt, _ = simplify(*mc_mesh(64), 1500)
    vt, ft = TX.uv_atlas(lv, lt, 128, 128, 2)
    b = NM.bake_cuda(lv, lt, vt, ft, lv, lt, 128, ssaa=1)
    assert bool(b['hit'].all())
    d = (b['normal'] - b['cage']).abs().max().item()
    assert d < 1e-4, d
    img, stats = NM.bake(lv, lt, vt, ft, lv, lt, 64, ssaa=2)
    assert stats['misses'] == 0 and stats['hits'] == stats['covered'] > 0


def test_two_runs_give_identical_bytes():
    lv, lt, dv, dt = low_and_detail(96, 64, 2000)
    vt, ft = TX.uv_atlas(lv, lt, 256, 256, 2)
    a, sa = NM.bake(lv, lt, vt, ft, dv, dt, 128, ssaa=2)
    b, sb = NM.bake(lv, lt, vt, ft, dv, dt, 128, ssaa=2)
    assert np.array_equal(a, b) and sa == sb and a.shape == (128, 128, 3)


def random_normal_map(h, w, seed):
    """Unit vectors within about 50 degrees of +-z, +-x, +-y by texel: maps that agree with some faces and not others."""
    rng = np.random.RandomState(seed)
    n = rng.randn(h, w, 3) * 0.6
    n[np.arange(h)[:, None], np.arange(w)[None, :], rng.randint(0, 3, (h, w))] += rng.choice([-1.0, 1.0], (h, w))
    return (n / np.linalg.norm(n, axis=-1, keepdims=True)).astype(np.float32)


def with_map(uvm, normal):
    return RL.UVMaterials(uvm.vt, uvm.ft, uvm.albedo, uvm.metallic, uvm.roughness, normal=normal)


@pytest.mark.parametrize('geometry', ['schlick', 'ggx_smith'])
def test_nmap_kernel_matches_oracle(geometry):
    verts, tris = OM.test_scene(2)
    uvm = random_uv_materials(verts, tris, 21)
    uvm = with_map(uvm, random_normal_map(*uvm.albedo.shape[:2], 4))
    r = RL.Relighter(verts, tris, uvm, random_env(12), geometry)
    pose, K = scene_camera(32, 32)
    got = r.render(pose, K, 32, 32, 1, 3, seed=5).cpu().numpy().astype(np.float64)
    ref = ON.render(r.verts, r.tris, (r.uv.vt, r.uv.ft, r.tex), r.tables, pose, K, 32, 32, 1, 3, seed=5, ggx_smith=r.ggx_smith)
    np.testing.assert_array_equal(got[..., 3], ref[..., 3])
    assert 0.1 < ref[..., 3].mean() < 0.9
    ok = np.abs(got[..., :3] - ref[..., :3]) <= 1e-4 * np.abs(ref[..., :3]) + 1e-5
    assert ok.mean() >= 0.995, f'{(~ok).sum()} of {ok.size} values differ; max {np.abs(got - ref).max():.3e}'


def test_nmap_alpha_is_the_unmapped_alpha_and_aov_guides_use_the_map():
    verts, tris = OM.test_scene(2)
    uvm = random_uv_materials(verts, tris, 3)
    env = random_env(4)
    plain = RL.Relighter(verts, tris, uvm, env)
    mapped = RL.Relighter(verts, tris, with_map(uvm, random_normal_map(*uvm.albedo.shape[:2], 9)), env)
    pose, K = scene_camera(48, 40)
    a = plain.render(pose, K, 48, 40, 16, 4, seed=9)
    b = mapped.render(pose, K, 48, 40, 16, 4, seed=9)
    c = mapped.render(pose, K, 48, 40, 16, 4, seed=9, spp_per_launch=3)
    assert torch.equal(a[..., 3], b[..., 3]) and torch.equal(b, c) and not torch.equal(a[..., :3], b[..., :3])
    acc, aov = mapped.render_sums(pose, K, 48, 40, 16, 4, seed=9)
    assert torch.equal(acc / 16, b)                                      # the AOV instance keeps accum's bits
    _, aov_plain = plain.render_sums(pose, K, 48, 40, 16, 4, seed=9)
    assert torch.equal(aov[..., 12:], aov_plain[..., 12:]) and not torch.equal(aov[..., 8:11], aov_plain[..., 8:11])


# Quality: a 128^3 marching-cubes bumpy sphere simplified to 2 000 triangles, relit flat and with a map baked from the
# 128^3 mesh, against the 128^3 mesh's own frame (64^2, 256 spp, seed 7, pixels all three frames cover fully).
# Measured on one H100 80GB HBM3 (700 W): MSE flat 2.100e-03, with the map 9.136e-04 over 3 087 pixels, a 2.30x cut.  The
# frames are deterministic, so the margin only has to absorb a change of card or driver: the map must cut the MSE 1.8x.
MIN_GAIN = 1.8


def test_a_baked_map_brings_the_low_mesh_closer_to_the_detail_mesh():
    from nero_b200.simplify import simplify
    dv, dt = mc_mesh(128)
    lv, lt, _ = simplify(dv, dt, 2000)
    vt, ft = TX.uv_atlas(lv, lt, 512, 512, 2)
    img, stats = NM.bake(lv, lt, vt, ft, dv, dt, 256, ssaa=2)
    assert stats['misses'] < 0.01 * stats['covered']
    grey = lambda c: np.full((256, 256) + c, 0.5, np.float32)
    vt_file = np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], -1)       # as the OBJ stores it
    flat = RL.UVMaterials(vt_file, ft, grey((3,)), grey(()) * 0, grey(()) * 0.6)
    mapped = with_map(flat, NM.decode(img))
    V = dv.shape[0]
    vmat = {'albedo': np.full((V, 3), 0.5, np.float32), 'metallic': np.zeros((V, 1), np.float32),
            'roughness': np.full((V, 1), np.sqrt(0.3), np.float32)}
    env = random_env(31, 32, 64)
    pose, K = RL.relight_poses(1, 0.0, 30.0, 1.8)[0], RL.blender_default_K(64, 64)
    frames = [RL.Relighter(v, t, m, env).render(pose, K, 64, 64, 256, 4, seed=7).cpu().numpy().astype(np.float64)
              for v, t, m in ((dv, dt, vmat), (lv, lt, flat), (lv, lt, mapped))]
    full = np.logical_and.reduce([f[..., 3] == 1 for f in frames])
    assert full.sum() > 500
    mse = [float(((f[..., :3] - frames[0][..., :3]) ** 2)[full].mean()) for f in frames[1:]]
    print(f'quality: {int(full.sum())} pixels, MSE flat {mse[0]:.3e}, with the map {mse[1]:.3e}, gain {mse[0] / mse[1]:.2f}x')
    assert mse[1] * MIN_GAIN < mse[0], mse


def test_tools_end_to_end(tmp_path):
    """write_textured_obj -> tools/bake_normal_map.py -> tools/relight.py --obj --normal-map; the same relight call without
    --normal-map writes the frames the unmapped textured path renders."""
    from test_relight_host import read_png, write_hdr
    from nero_b200.mesh import write_ply
    lv, lt, dv, dt = low_and_detail(64, 48, 1200)
    vt, ft = TX.uv_atlas(lv, lt, 128, 128, 2)
    rng = np.random.RandomState(1)
    maps = (rng.randint(60, 200, (64, 64, 3)).astype(np.uint8), np.full((64, 64, 3), 20, np.uint8), np.full((64, 64, 3), 150, np.uint8))
    TX.write_textured_obj(str(tmp_path / 'n2m'), lv, lt, vt, ft, maps)
    write_ply(str(tmp_path / 'detail.ply'), dv, dt)
    write_hdr(tmp_path / 'env.hdr', random_env(7, 32, 64), rle=True)
    env = dict(os.environ, PYTHONPATH=ROOT)
    tools = os.path.join(ROOT, 'tools')
    out = subprocess.run([sys.executable, os.path.join(tools, 'bake_normal_map.py'), '--obj', 'n2m/mesh_0.obj', '--detail', 'detail.ply'],
                         cwd=tmp_path, env=env, capture_output=True, text=True, check=True).stdout
    assert 'misses' in out and (tmp_path / 'n2m' / 'normal_0.png').exists()
    nmap = NM.read_normal_map(str(tmp_path / 'n2m' / 'normal_0.png'))
    assert nmap.shape == (64, 64, 3)
    h, w = 20, 28
    common = ['--hdr', 'env.hdr', '--num', '2', '--width', str(w), '--height', str(h), '--samples', '4', '--cam_dist', '2.0',
              '--bounces', '2', '--obj', 'n2m/mesh_0.obj']
    relight = [sys.executable, os.path.join(tools, 'relight.py')]
    subprocess.check_call(relight + common + ['--name', 'nmap', '--normal-map', 'n2m/normal_0.png'], cwd=tmp_path, env=env)
    subprocess.check_call(relight + common + ['--name', 'plain'], cwd=tmp_path, env=env)
    v, t, vt_f, ft_f, m = RL.load_textured_obj(str(tmp_path / 'n2m' / 'mesh_0.obj'))
    r = RL.Relighter(v, t, RL.UVMaterials(vt_f, ft_f, m['albedo'], m['metallic'], m['roughness']), RL.load_env_map(str(tmp_path / 'env.hdr')))
    poses, K = RL.relight_poses(2, 0.0, 45.0, 2.0), RL.blender_default_K(h, w)
    for k in range(2):
        a, b = read_png(tmp_path / 'data' / 'relight' / 'nmap' / f'{k}.png'), read_png(tmp_path / 'data' / 'relight' / 'plain' / f'{k}.png')
        assert a.shape == (h, w, 4) and np.array_equal(a[..., 3], b[..., 3]) and (a[..., 3] > 0).any()
        assert not np.array_equal(a, b)
        ref = RL.to_rgba8(r.render(poses[k], K, h, w, 4, 2, 0).cpu().numpy())
        assert np.array_equal(b, ref)
