"""Relighting from UV textures on the GPU: nero_relight_render_textured against the numpy oracle (atlas uv and uv outside
[0, 1]), coverage shared with the per-vertex path, determinism, a white furnace with a constant texture, a relight of a
baked texture against the per-vertex export of the same materials, and tools/relight.py --obj end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_mat as OM
import nero_oracle_relight as OR
import nero_oracle_relight_tex as ORT
from nero_b200 import relight as RL
from nero_b200 import texmap as TX
from test_relight_gpu import random_env, random_materials, scene_camera

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def decode(k):
    return RL.srgb_to_linear(np.asarray(k, np.float64) / 255).astype(np.float32)


def random_uv_materials(verts, tris, seed, h=24, w=40):
    """Random texture bytes (roughness decoded >= 0.3, as random_materials keeps it) on an atlas of the mesh."""
    rng = np.random.RandomState(seed)
    vt, ft = TX.uv_atlas(verts, tris, 2 * w, 2 * h, 2)
    return RL.UVMaterials(vt, ft, decode(rng.randint(0, 256, (h, w, 3))), decode(rng.randint(0, 256, (h, w))),
                          decode(rng.randint(150, 256, (h, w))))


def oracle(r, pose, K, h, w, spp, bounces, seed):
    uvm = (r.uv.vt, r.uv.ft, r.tex)
    return ORT.render(r.verts, r.tris, uvm, r.tables, pose, K, h, w, spp, bounces, seed=seed, ggx_smith=r.ggx_smith)


@pytest.mark.parametrize('wrap', [False, True])
@pytest.mark.parametrize('geometry', ['schlick', 'ggx_smith'])
def test_kernel_matches_oracle(geometry, wrap):
    verts, tris = OM.test_scene(2)
    uvm = random_uv_materials(verts, tris, 21)
    if wrap:                                       # uv in [-1.3, 2.2]: every tap wraps somewhere
        uvm = RL.UVMaterials(uvm.vt * np.float32(3.5) - np.float32(1.3), uvm.ft, uvm.albedo, uvm.metallic, uvm.roughness)
        assert uvm.vt.min() < -1 and uvm.vt.max() > 2
    r = RL.Relighter(verts, tris, uvm, random_env(12), geometry)
    pose, K = scene_camera(32, 32)
    got = r.render(pose, K, 32, 32, 1, 3, seed=5).cpu().numpy().astype(np.float64)
    ref = oracle(r, pose, K, 32, 32, 1, 3, 5)
    np.testing.assert_array_equal(got[..., 3], ref[..., 3])
    assert 0.1 < ref[..., 3].mean() < 0.9
    ok = np.abs(got[..., :3] - ref[..., :3]) <= 1e-4 * np.abs(ref[..., :3]) + 1e-5
    assert ok.mean() >= 0.995, f'{(~ok).sum()} of {ok.size} values differ; max {np.abs(got - ref).max():.3e}'


def test_coverage_matches_the_per_vertex_path_and_renders_are_deterministic():
    verts, tris = OM.test_scene(2)
    env = random_env(4)
    rt = RL.Relighter(verts, tris, random_uv_materials(verts, tris, 3), env, 'schlick')
    rv = RL.Relighter(verts, tris, random_materials(verts.shape[0], 3), env, 'schlick')
    pose, K = scene_camera(48, 40)
    a = rt.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=32)
    b = rt.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=32)
    c = rt.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=3)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert not torch.equal(a, rt.render(pose, K, 48, 40, 32, 4, seed=10))
    v = rv.render(pose, K, 48, 40, 32, 4, seed=9)
    assert torch.equal(a[..., 3], v[..., 3]) and 0 < float(a[..., 3].mean()) < 1
    assert not torch.equal(a[..., :3], v[..., :3])


def furnace_expectation(albedo, metallic, alpha, nov):
    """E(NoV) of the oracle BRDF times cos over the hemisphere by quadrature, interpolated at nov -> [n,3]."""
    tab_nov = np.linspace(0.0, 1.0, 101)
    th, ph = np.meshgrid((np.arange(512) + 0.5) / 512 * np.pi / 2, (np.arange(1024) + 0.5) / 1024 * 2 * np.pi, indexing='ij')
    l = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3)
    dw = (np.sin(th) * (np.pi / 2 / 512) * (2 * np.pi / 1024)).reshape(-1)
    M = l.shape[0]
    E = []
    for nv in tab_nov:
        v = np.asarray([np.sqrt(max(1 - nv * nv, 0)), 0.0, max(nv, 1e-4)])
        f = OR.brdf(np.tile([0.0, 0.0, 1.0], (M, 1)), np.tile(v, (M, 1)), l, np.tile(albedo, (M, 1)), np.full(M, metallic),
                    np.full(M, alpha), 0)
        E.append(np.sum(f * (l[:, 2] * dw)[:, None], 0))
    E = np.stack(E)
    return np.stack([np.interp(nov, tab_nov, E[:, k]) for k in range(3)], -1)


@pytest.mark.parametrize('metallic', [0, 255])
def test_white_furnace_with_a_constant_texture(metallic):
    """test_white_furnace's statistics with the materials in a constant texture.  The expected value is computed at
    alpha = r, the decoded roughness byte, and the one at alpha = r^2 is many standard errors away: a kernel that squared
    the texture roughness would fail here."""
    from nero_b200 import ops
    verts, tris = OM.icosphere(4, 0.5)
    tris = np.ascontiguousarray(tris[:, [0, 2, 1]])             # wound like marching-cubes meshes (normal into the solid)
    alb8, r8, Lc = np.asarray([228, 188, 124]), 149, 1.7
    albedo, met, rough = decode(alb8).astype(np.float64), float(decode(metallic)), float(decode(r8))
    assert abs(rough - 0.3) < 0.005 and met == metallic / 255
    vt, ft = TX.uv_atlas(verts, tris, 64, 64, 2)
    uvm = RL.UVMaterials(vt, ft, np.tile(decode(alb8), (8, 8, 1)), np.full((8, 8), decode(metallic)), np.full((8, 8), decode(r8)))
    r = RL.Relighter(verts, tris, uvm, np.full((8, 16, 3), Lc, np.float32), 'schlick')
    h = w = 24
    spp = 256
    pose, K = RL.relight_poses(1, 0.0, 20.0, 1.6)[0], RL.blender_default_K(h, w)
    img = r.render(pose, K, h, w, spp, 4, seed=3).cpu().numpy().astype(np.float64)
    R, t = pose[:, :3], pose[:, 3]
    pix = np.repeat(np.arange(h * w), spp)
    s = np.tile(np.arange(spp), h * w)
    c = np.stack([(pix % w + OR.uniform(3, pix, s, 0, 0) - K[0, 2]) / K[0, 0], (pix // w + OR.uniform(3, pix, s, 0, 1) - K[1, 2]) / K[1, 1],
                  np.ones(pix.size)], -1)
    d = torch.from_numpy(OR.normalize(c @ R)).float().cuda().contiguous()
    o = torch.from_numpy(np.broadcast_to(-R.T @ t, (pix.size, 3)).copy()).float().cuda().contiguous()
    pos, nrm = torch.empty(pix.size, 4, device='cuda'), torch.empty(pix.size, 4, device='cuda')
    ops.K('nero_bvh_trace', r.nodes, r.tri, pix.size, o, 3, d, 3, pos, nrm, 1e30, 1)
    nrm = nrm.cpu().numpy().astype(np.float64)
    hit = nrm[:, 3] > 0
    nov = np.clip(-(nrm[:, :3] * d.cpu().numpy()).sum(-1), 0, 1)
    alpha = np.bincount(pix, weights=hit, minlength=h * w) / spp
    np.testing.assert_array_equal(img[..., 3].reshape(-1), alpha)
    m = alpha > 0
    assert m.sum() > 100

    def residual(a):
        per = np.zeros((h * w, 3))
        np.add.at(per, pix, Lc * furnace_expectation(albedo, met, a, nov) * hit[:, None])
        return img[..., :3].reshape(-1, 3)[m] - per[m] / spp
    res = residual(rough)
    se = res.std(0) / np.sqrt(m.sum())
    assert (np.abs(res.mean(0)) < 3 * se + 1e-4).all(), (res.mean(0), se)
    squared = residual(rough ** 2).mean(0)
    assert (np.abs(squared) > 10 * se).any(), (squared, se)


# ------------------------------------------------------------------------------------------------ through the bake
ROUND_TRIP_SIZE, ROUND_TRIP_SPP = 96, 64
# Measured once on the scene below (one H100 80GB HBM3): mean |rgb difference| over covered pixels 0.0114 and PSNR 38.2 dB
# of the 8-bit frames over the covered pixels; with the texture roughness squared, 0.0944 and 24.0 dB.  The bound leaves a
# margin of about 30 % on the mean and 1.7 dB on the PSNR, and the squared roughness misses it by 6x and 12 dB.
MAX_MEAN_ABS, MIN_PSNR = 0.015, 36.5


def round_trip_renders(tmp_path, square_roughness=False):
    from test_texmap_gpu import material_renderer
    verts, tris = OM.test_scene(3)
    net, _ = material_renderer(verts, tris)
    vt, ft = TX.uv_atlas(verts, tris, 512, 512, 4)
    alb, met, rough = TX.bake_textures(net, verts, tris, vt, ft, (256, 256), 2)
    vt_file = np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], -1)           # as the OBJ stores it
    rough_lin = decode(rough[..., 0])
    uvm = RL.UVMaterials(vt_file, ft, decode(alb), decode(met[..., 0]), rough_lin ** 2 if square_roughness else rough_lin)
    RL.save_materials(str(tmp_path / 'mat'), net.predict_materials())
    env = random_env(31, 32, 64)
    rt = RL.Relighter(verts, tris, uvm, env)
    rv = RL.Relighter(verts, tris, RL.load_materials(str(tmp_path / 'mat')), env)
    n = ROUND_TRIP_SIZE
    pose, K = scene_camera(n, n)
    return (rt.render(pose, K, n, n, ROUND_TRIP_SPP, 4, seed=17).cpu().numpy(),
            rv.render(pose, K, n, n, ROUND_TRIP_SPP, 4, seed=17).cpu().numpy())


def difference(a, b):
    """(mean |rgb difference| of the linear renders, PSNR of their 8-bit frames) over the pixels covered by both."""
    from nero_b200 import metrics
    cov = (a[..., 3] > 0) & (b[..., 3] > 0)
    mad = float(np.abs(a[..., :3] - b[..., :3])[cov].mean())
    qa, qb = (torch.from_numpy(RL.to_rgba8(x)[..., :3][cov][None]).cuda() for x in (a, b))
    return mad, metrics.psnr(qb, qa)


def test_baked_textures_relight_like_the_vertex_materials(tmp_path):
    """The stage-II materials relit from their 256^2 texture bake and from their per-vertex export: same coverage, and
    colours that differ only by the bake's 8-bit quantisation and by texel versus barycentric interpolation.

    The per-vertex path interpolates three exact values linearly over a triangle; the texture holds the material field
    sampled at texel centres, truncated to 8 bits after the sRGB transfer (< 1/255 in sRGB, about 0.4 % of a mid-grey linear
    value), and filters it bilinearly, which follows the field inside a triangle more closely than the barycentric
    interpolation does.  Slightly different materials also choose different BRDF lobes and directions from the same random
    numbers, so at 64 spp part of the difference is Monte-Carlo noise that does not cancel.  All of it is small compared
    with the change that a squared roughness makes, which the last assertion shows."""
    tex, vert = round_trip_renders(tmp_path)
    np.testing.assert_array_equal(tex[..., 3], vert[..., 3])
    cov = tex[..., 3] > 0
    assert 0.1 < cov.mean() < 0.9
    mad, psnr = difference(tex, vert)
    print(f'round trip: mean |rgb difference| {mad:.5f}, PSNR {psnr:.2f} dB over {int(cov.sum())} covered pixels')
    assert mad <= MAX_MEAN_ABS and psnr >= MIN_PSNR, (mad, psnr)
    sq, _ = round_trip_renders(tmp_path, square_roughness=True)
    mad_sq, psnr_sq = difference(sq, vert)
    print(f'round trip with squared roughness: mean |rgb difference| {mad_sq:.5f}, PSNR {psnr_sq:.2f} dB')
    assert mad_sq > MAX_MEAN_ABS and psnr_sq < MIN_PSNR, (mad_sq, psnr_sq)


# ------------------------------------------------------------------------------------------------ the tools
def test_tools_end_to_end(tmp_path):
    """A tiny checkpoint through tools/extract_materials_texture_map.py and tools/relight.py --obj: the frames are written,
    their coverage is that of the --mesh / --material frames of the same checkpoint, and existing frames are skipped."""
    import yaml
    from test_relight_host import read_png, write_hdr
    from test_texmap_gpu import SHADER_CFG, material_renderer
    from nero_b200.mesh import write_ply
    verts, tris = OM.test_scene(2)
    _, sd = material_renderer(verts, tris)
    os.makedirs(tmp_path / 'data' / 'model' / 'tex', exist_ok=True)
    for name in ('model.pth', 'model_best.pth'):
        torch.save({'step': 77, 'network_state_dict': sd}, tmp_path / 'data' / 'model' / 'tex' / name)
    write_ply(str(tmp_path / 'mesh.ply'), verts, tris)
    cfg = {'name': 'tex', 'network': 'material', 'mesh': str(tmp_path / 'mesh.ply'), 'shader_cfg': dict(SHADER_CFG)}
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    tools = os.path.join(ROOT, 'tools')
    subprocess.check_call([sys.executable, os.path.join(tools, 'extract_materials_texture_map.py'), '--cfg', 'cfg.yaml', '--size', '64',
                           '--out', 'n2m'], cwd=tmp_path, env=env)
    subprocess.check_call([sys.executable, os.path.join(tools, 'extract_materials.py'), '--cfg', 'cfg.yaml'], cwd=tmp_path, env=env)
    write_hdr(tmp_path / 'env.hdr', random_env(7, 32, 64), rle=True)
    h, w = 20, 28
    common = ['--hdr', 'env.hdr', '--num', '3', '--width', str(w), '--height', str(h), '--samples', '4', '--cam_dist', '2.0',
              '--bounces', '2', '--trans']
    relight = [sys.executable, os.path.join(tools, 'relight.py')]
    subprocess.check_call(relight + ['--obj', 'n2m/mesh_0.obj', '--name', 'tex'] + common, cwd=tmp_path, env=env)
    subprocess.check_call(relight + ['--mesh', 'mesh.ply', '--material', 'data/materials/tex-77', '--name', 'vert'] + common,
                          cwd=tmp_path, env=env)
    out = tmp_path / 'data' / 'relight'
    for k in range(3):
        a, b = read_png(out / 'tex' / f'{k}.png'), read_png(out / 'vert' / f'{k}.png')
        assert a.shape == (h, w, 4)
        np.testing.assert_array_equal(a[..., 3], b[..., 3])
        assert (a[..., 3] > 0).any() and not (a[..., 3] > 0).all()
        assert (a[..., :3][a[..., 3] > 0] > 0).any()
    before = os.path.getmtime(out / 'tex' / '0.png')
    subprocess.check_call(relight + ['--obj', 'n2m/mesh_0.obj', '--name', 'tex'] + common, cwd=tmp_path, env=env)
    assert os.path.getmtime(out / 'tex' / '0.png') == before      # existing frames are skipped
