"""Relighting on the GPU: nero_relight_render against the numpy oracle, determinism, a white-furnace test and the two tools
end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_mat as OM
import nero_oracle_relight as OR
from nero_b200 import relight as RL

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_materials(V, seed):
    """Linear per-vertex materials; roughness >= 0.3 keeps fp32 GGX peaks within the comparison tolerance."""
    rng = np.random.RandomState(seed)
    return {'metallic': rng.rand(V, 1).astype(np.float32), 'roughness': (0.3 + 0.7 * rng.rand(V, 1)).astype(np.float32),
            'albedo': rng.rand(V, 3).astype(np.float32)}


def random_env(seed, H=16, W=32):
    return np.exp(np.random.RandomState(seed).randn(H, W, 3)).astype(np.float32)


def scene_camera(h, w):
    return RL.relight_poses(3, 20.0, 30.0, 2.0)[1], RL.blender_default_K(h, w)


@pytest.mark.parametrize('geometry', ['schlick', 'ggx_smith'])
def test_kernel_matches_oracle(geometry):
    verts, tris = OM.test_scene(2)
    mats = random_materials(verts.shape[0], 11)
    env = random_env(12)
    r = RL.Relighter(verts, tris, mats, env, geometry)
    pose, K = scene_camera(32, 32)
    got = r.render(pose, K, 32, 32, 1, 3, seed=5).cpu().numpy().astype(np.float64)
    ref = OR.render(verts, tris, r.vmat, r.tables, pose, K, 32, 32, 1, 3, seed=5, ggx_smith=r.ggx_smith)
    np.testing.assert_array_equal(got[..., 3], ref[..., 3])
    assert 0.1 < ref[..., 3].mean() < 0.9
    ok = np.abs(got[..., :3] - ref[..., :3]) <= 1e-4 * np.abs(ref[..., :3]) + 1e-5
    assert ok.mean() >= 0.995, f'{(~ok).sum()} of {ok.size} values differ; max {np.abs(got - ref).max():.3e}'


def test_render_is_deterministic_and_chunking_invariant():
    verts, tris = OM.test_scene(2)
    r = RL.Relighter(verts, tris, random_materials(verts.shape[0], 3), random_env(4), 'schlick')
    pose, K = scene_camera(48, 40)
    a = r.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=32)
    b = r.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=32)
    c = r.render(pose, K, 48, 40, 32, 4, seed=9, spp_per_launch=4)
    assert torch.equal(a, b) and torch.equal(a, c)
    assert not torch.equal(a, r.render(pose, K, 48, 40, 32, 4, seed=10))


@pytest.mark.parametrize('metallic', [0.0, 1.0])
def test_white_furnace(metallic):
    """A convex icosphere under a constant map L: no interreflection, so a hit sample's expected value is
    L (albedo (1-m) + E_spec(NoV)), the hemispherical integral of the BRDF times cos, computed here by quadrature."""
    from nero_b200 import ops
    verts, tris = OM.icosphere(4, 0.5)
    tris = np.ascontiguousarray(tris[:, [0, 2, 1]])             # wound like marching-cubes meshes (normal into the solid)
    V = verts.shape[0]
    albedo, rough, Lc = np.asarray([0.8, 0.5, 0.2]), 0.5, 1.7
    mats = {'metallic': np.full((V, 1), metallic, np.float32), 'roughness': np.full((V, 1), rough, np.float32),
            'albedo': np.tile(albedo.astype(np.float32), (V, 1))}
    r = RL.Relighter(verts, tris, mats, np.full((8, 16, 3), Lc, np.float32), 'schlick')
    h = w = 24
    spp = 256
    pose, K = RL.relight_poses(1, 0.0, 20.0, 1.6)[0], RL.blender_default_K(h, w)
    img = r.render(pose, K, h, w, spp, 4, seed=3).cpu().numpy().astype(np.float64)
    # NoV of every camera sample: the kernel's jitter (same hash) and the product tracer's outward normal
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
    # E(NoV): quadrature of the oracle BRDF times cos over the hemisphere, tabulated in NoV
    tab_nov = np.linspace(0.0, 1.0, 101)
    th, ph = np.meshgrid((np.arange(512) + 0.5) / 512 * np.pi / 2, (np.arange(1024) + 0.5) / 1024 * 2 * np.pi, indexing='ij')
    l = np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], -1).reshape(-1, 3)
    dw = (np.sin(th) * (np.pi / 2 / 512) * (2 * np.pi / 1024)).reshape(-1)
    E = []
    for nv in tab_nov:
        v = np.asarray([np.sqrt(max(1 - nv * nv, 0)), 0.0, max(nv, 1e-4)])
        M = l.shape[0]
        f = OR.brdf(np.tile([0.0, 0.0, 1.0], (M, 1)), np.tile(v, (M, 1)), l, np.tile(albedo, (M, 1)), np.full(M, metallic),
                    np.full(M, rough ** 2), 0)
        E.append(np.sum(f * (l[:, 2] * dw)[:, None], 0))
    E = np.stack(E)
    per = np.zeros((h * w, 3))
    expect = Lc * np.stack([np.interp(nov, tab_nov, E[:, k]) for k in range(3)], -1) * hit[:, None]
    np.add.at(per, pix, expect)
    per /= spp
    alpha = np.bincount(pix, weights=hit, minlength=h * w) / spp
    np.testing.assert_array_equal(img[..., 3].reshape(-1), alpha)
    m = alpha > 0
    res = img[..., :3].reshape(-1, 3)[m] - per[m]
    se = res.std(0) / np.sqrt(m.sum())
    assert (np.abs(res.mean(0)) < 3 * se + 1e-4).all(), (res.mean(0), se)
    assert m.sum() > 100


def test_tools_end_to_end(tmp_path):
    """tools/extract_materials.py on a saved random material checkpoint, then tools/relight.py on that mesh, those materials and
    a written .hdr."""
    import yaml
    from helpers import build_material_params
    from test_relight_host import read_png, write_hdr
    from nero_b200.material import NeROMaterialRenderer
    from nero_b200.mesh import write_ply
    verts, tris = OM.test_scene(2)
    scfg = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}
    sd = build_material_params(scfg)
    os.makedirs(tmp_path / 'data' / 'model' / 'relit', exist_ok=True)
    torch.save({'step': 1234, 'network_state_dict': sd}, tmp_path / 'data' / 'model' / 'relit' / 'model.pth')
    write_ply(str(tmp_path / 'mesh.ply'), verts, tris)
    cfg = {'name': 'relit', 'network': 'material', 'mesh': str(tmp_path / 'mesh.ply'), 'shader_cfg': scfg}
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.check_call([sys.executable, os.path.join(ROOT, 'tools', 'extract_materials.py'), '--cfg', 'cfg.yaml'], cwd=tmp_path, env=env)
    net = NeROMaterialRenderer(cfg, is_train=False)
    net.load_state_dict(sd)
    want = net.cuda().predict_materials()
    mdir = tmp_path / 'data' / 'materials' / 'relit-1234'
    for k in ('metallic', 'roughness', 'albedo'):
        np.testing.assert_array_equal(np.load(mdir / f'{k}.npy'), RL.linear_to_srgb(want[k]))
    write_hdr(tmp_path / 'env.hdr', random_env(7, 32, 64), rle=True)
    h, w, spp = 20, 28, 4
    args = ['--mesh', 'mesh.ply', '--material', str(mdir), '--hdr', 'env.hdr', '--name', 'bell', '--num', '3', '--width', str(w),
            '--height', str(h), '--samples', str(spp), '--cam_dist', '2.0', '--bounces', '2']
    subprocess.check_call([sys.executable, os.path.join(ROOT, 'tools', 'relight.py')] + args, cwd=tmp_path, env=env)
    poses, K = RL.relight_poses(3, 0.0, 45.0, 2.0), RL.blender_default_K(h, w)
    for k in range(3):
        img = read_png(tmp_path / 'data' / 'relight' / 'bell' / f'{k}.png')
        assert img.shape == (h, w, 4)
        R, t = poses[k][:, :3], poses[k][:, 3]
        pix = np.repeat(np.arange(h * w), spp)
        s = np.tile(np.arange(spp), h * w)
        c = np.stack([(pix % w + OR.uniform(0, pix, s, 0, 0) - K[0, 2]) / K[0, 0],
                      (pix // w + OR.uniform(0, pix, s, 0, 1) - K[1, 2]) / K[1, 1], np.ones(pix.size)], -1)
        d = OR.normalize(c @ R)
        hit = OR.trace(verts, tris, np.broadcast_to(-R.T @ t, d.shape).copy(), d)[0] >= 0
        covered = np.bincount(pix, weights=hit, minlength=h * w).reshape(h, w) > 0
        np.testing.assert_array_equal(img[..., 3] > 0, covered)
        assert covered.any() and not covered.all()
    before = os.path.getmtime(tmp_path / 'data' / 'relight' / 'bell' / '0.png')
    subprocess.check_call([sys.executable, os.path.join(ROOT, 'tools', 'relight.py')] + args, cwd=tmp_path, env=env)
    assert os.path.getmtime(tmp_path / 'data' / 'relight' / 'bell' / '0.png') == before     # existing frames are skipped
