"""Environment-light export on the GPU: nero_env_rows against the oracle, the whole map against the oracle and the reference
fixtures, an analytic known-answer test, determinism across runs and batch splits, the renderer hooks (no side effects on
parameters or gradients), a relight of the exported map and the refusal of CPU tensors."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_envmap as OE
import nero_oracle_mat as OM
from nero_b200 import envmap as EM

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, 'envmap_*.npz')))


def stage2_net(sphere=False, rel=0.3, mesh=None):
    from nero_b200 import params as P
    from nero_b200.material import NeROMaterialRenderer
    scfg = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16,
            'outer_light_version': 'sphere_direction' if sphere else 'direction'}
    sd = O.perturb_params(P.build_material_state_dict(scfg, seed=6033), seed=11, rel=rel)
    net = NeROMaterialRenderer({'shader_cfg': scfg}, is_train=False, mesh=mesh or OM.test_scene(2))
    net.load_state_dict(sd)
    return net.cuda(), sd


def stage1_net(sphere=False, rel=0.3):
    from nero_b200 import params as P
    from nero_b200.renderer import NeROShapeRenderer
    cfg = {'shader_config': {'sphere_direction': sphere}, 'n_samples': 16, 'n_importance': 16}
    sd = O.perturb_params(P.build_shape_state_dict(cfg, seed=6033), seed=11, rel=rel)
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(sd)
    return net.cuda(), sd


@pytest.mark.parametrize('sphere,center,kappa', [(None, (0, 0, 0), 0.0), (None, (0, 0, 0), 0.3), ('stage2', (0.3, -0.2, 0.25), 0.0),
                                                 ('stage1', (0.7, -0.6, 0.5), 0.25), ('stage1', (0.1, 0.2, -0.1), 1.0)])
@pytest.mark.parametrize('trans', [False, True])
def test_rows_match_oracle(sphere, center, kappa, trans):
    W, H, s = 24, 12, 3
    frame = EM.trans_frame(trans)
    n_all = W * H * s * s
    row0, n = 37, n_all - 37 - 50               # a range that starts and ends inside texels and warps
    A, dirs = EM.env_rows(row0, n, W, H, s, kappa_inv=kappa, sphere=sphere, center=center, frame=frame)
    want_d = OE.directions(W, H, s, frame)[row0:row0 + n]
    np.testing.assert_array_equal(dirs.cpu().numpy(), want_d)
    want = OE.rows(torch.from_numpy(want_d), kappa, sphere, center).numpy()
    A = A.cpu().numpy()
    k = want.shape[1]
    # within 1e-6 where the encoding is well conditioned; where the z-polynomial cancels (l = 16 near the poles) the two fp32
    # evaluations (the kernel's ascending FMA chain, torch's matmul) may each be off by the dot product's rounding bound
    pts = [want_d] if sphere is None else [want_d, OE.sphere_points(torch.from_numpy(want_d), sphere, center).numpy()]
    kap = [kappa, 0.0 if sphere == 'stage2' else kappa]
    S = np.concatenate([ide_magnitude(p, kv) for p, kv in zip(pts, kap)], 1)
    assert (np.abs(A[:, :k] - want) <= 1e-6 + 1e-5 * np.abs(want) + 2 * 17 * 2.0 ** -24 * S).all()
    assert (np.abs(A[:, :72] - want[:, :72]) <= 1e-6).mean() > 0.99    # same input directions, bit for bit
    assert A.shape[1] == (192 if sphere else 128) and (A[:, k:] == 0).all()


def ide_magnitude(d, kappa_inv):
    """[n,72]: |x + iy|^m * sum_k |z^k mat[k]| * exp(-sigma kappa_inv), the sum of the magnitudes of the terms of each IDE
    value (the scale of its fp32 rounding error)."""
    ml, mat = O.ide_tables(5)
    d = np.asarray(d, np.float64)
    r = np.hypot(d[:, 0], d[:, 1])[:, None] ** ml[0].astype(np.float64)[None]
    zk = np.abs(d[:, 2:3]) ** np.arange(mat.shape[0])[None]
    att = np.exp(-0.5 * ml[1] * (ml[1] + 1.0) * kappa_inv)
    m = r * (zk @ np.abs(mat.astype(np.float64))) * att
    return np.concatenate([m, m], 1)


def run_fixture(g, max_rows=EM.MAX_ROWS):
    sph = bool(g['sphere'])
    if int(g['stage']) == 2:
        net, _ = stage2_net(sph, float(g['rel']))
        mod = net.shader_network.outer_light
        sphere = 'stage2' if sph else None
    else:
        net, _ = stage1_net(sph, float(g['rel']))
        mod = net.color_network.outer_light
        sphere = 'stage1' if sph else None
    env = EM.outer_light_map(mod, width=int(g['width']), height=int(g['height']), ssaa=int(g['ssaa']), kappa_inv=float(g['kappa_inv']),
                             sphere=sphere, center=tuple(g['center'].tolist()), exp_max=float(g['exp_max']), max_rows=max_rows)
    return env.cpu().numpy()


@pytest.mark.parametrize('name', FIXTURES)
def test_map_matches_reference_fixture_and_oracle(name):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    env = run_fixture(g)
    tol = lambda ref: 1e-4 * np.abs(ref) + 1e-6
    assert (np.abs(env - g['env']) <= tol(g['env'])).all(), np.abs(env - g['env']).max()
    sd, prefix, sphere = OE.fixture_params(g)
    ref = OE.envmap(sd, prefix, int(g['width']), int(g['height']), int(g['ssaa']), float(g['kappa_inv']), sphere, g['center'],
                    None, float(g['exp_max']))
    assert (np.abs(env - ref) <= tol(ref)).all(), np.abs(env - ref).max()


def test_known_answer_constant_light():
    """outer_light.6.weight_g = 0 and bias log 2: the last layer's weight is zero, every sub-sample is exp(log 2) and every
    texel exactly 2.0f."""
    net, _ = stage2_net()
    ol = net.shader_network.outer_light
    with torch.no_grad():
        getattr(ol, '6').weight_g.zero_()
        getattr(ol, '6').bias.fill_(float(np.log(2.0)))
    for W, H, s in ((16, 8, 2), (33, 17, 3), (8, 4, 1)):
        env = net.export_lighting(width=W, height=H, ssaa=s).cpu().numpy()
        assert env.shape == (H, W, 3) and (env == np.float32(2.0)).all()


def test_map_is_bit_identical_across_runs_and_batch_splits():
    net, _ = stage2_net(sphere=True)
    mod = net.shader_network.outer_light
    kw = dict(width=40, height=21, ssaa=3, sphere='stage2', center=(0.1, 0.2, -0.3), exp_max=5.0)
    base = EM.outer_light_map(mod, **kw).cpu().numpy()
    np.testing.assert_array_equal(EM.outer_light_map(mod, **kw).cpu().numpy(), base)
    for max_rows in (9, 117, 126, 135, 9 * 29, 1000, 40 * 21 * 9 + 5):
        np.testing.assert_array_equal(EM.outer_light_map(mod, max_rows=max_rows, **kw).cpu().numpy(), base)


def params_and_grads(net):
    return [(p.detach().clone(), None if p.grad is None else p.grad.detach().clone()) for p in net.parameters()]


def assert_unchanged(before, net):
    for (p0, g0), p in zip(before, net.parameters()):
        assert torch.equal(p0, p.detach())
        assert (g0 is None and p.grad is None) or torch.equal(g0, p.grad)


def test_export_lighting_has_no_side_effects():
    net, _ = stage2_net()
    batch = OM.synthetic_surface_batch(*OM.test_scene(2), 8, seed=6033)
    rands = OM.draw_rands(8)
    out = net.shade_batch({k: v.cuda() for k, v in batch.items()}, 5000, {k: v.cuda() for k, v in rands.items()})
    sum(torch.mean(v) for k, v in out.items() if k.startswith('loss')).backward()
    before = params_and_grads(net)
    env = net.export_lighting(width=16, height=8, ssaa=2, trans=True)
    assert env.shape == (8, 16, 3) and env.is_cuda and torch.isfinite(env).all()
    assert_unchanged(before, net)
    snet, _ = stage1_net(sphere=True)
    before = params_and_grads(snet)
    maps = snet.export_lighting(width=16, height=8, ssaa=2, kappa_inv=(0.0, 1.0))
    assert sorted(maps) == [0.0, 1.0] and all(m.shape == (8, 16, 3) for m in maps.values())
    assert not torch.equal(maps[0.0], maps[1.0])
    assert_unchanged(before, snet)


def test_trans_map_is_the_map_of_rotated_directions():
    net, sd = stage2_net()
    env = net.export_lighting(width=16, height=8, ssaa=2, trans=True).cpu().numpy()
    ref = OE.envmap(sd, 'shader_network.outer_light', 16, 8, 2, frame=EM.trans_frame(True), exp_max=5.0)
    assert (np.abs(env - ref) <= 1e-4 * np.abs(ref) + 1e-6).all()


def test_relighter_renders_the_exported_map(tmp_path):
    from nero_b200.relight import Relighter, blender_default_K, load_env_map, relight_poses
    verts, tris = OM.test_scene(2)
    net, _ = stage2_net(mesh=(verts, tris))
    p = str(tmp_path / 'outer_light.hdr')
    EM.write_hdr(p, net.export_lighting(width=32, height=16, ssaa=2))
    env = load_env_map(p)
    rng = np.random.RandomState(3)
    V = verts.shape[0]
    mats = {'metallic': rng.rand(V, 1), 'roughness': 0.3 + 0.7 * rng.rand(V, 1), 'albedo': rng.rand(V, 3)}
    img = Relighter(verts, tris, mats, env).render(relight_poses(3, 0.0, 30.0, 2.0)[1], blender_default_K(16, 16), 16, 16, 2)
    img = img.cpu().numpy()
    assert np.isfinite(img).all() and (img[..., 3] > 0).any() and img[..., :3].max() > 0


def test_cpu_tensors_raise():
    from nero_b200 import params as P
    m = P.MCShadingParams({'human_lights': False})
    with pytest.raises(RuntimeError):
        EM.outer_light_map(m.outer_light, width=8, height=4, ssaa=1, exp_max=5.0)
    with pytest.raises(RuntimeError):
        EM.env_rows(0, 4, 8, 4, 1, device='cpu')
    with pytest.raises(ValueError):
        net, _ = stage2_net(sphere=True)
        net.export_lighting(width=8, height=4, ssaa=1, center=(0.9, 0.5, 0.0))


def test_tool_end_to_end(tmp_path):
    """extract_materials + extract_lighting on a stage-II checkpoint, then relight.py --hdr on the exported map; a stage-I
    checkpoint writes one map per kappa; a config without an outer light is refused."""
    import yaml
    from nero_b200.mesh import write_ply
    from nero_b200.relight import load_env_map
    verts, tris = OM.test_scene(2)
    _, sd = stage2_net(mesh=(verts, tris))
    os.makedirs(tmp_path / 'data' / 'model' / 'lit', exist_ok=True)
    torch.save({'step': 77, 'network_state_dict': sd}, tmp_path / 'data' / 'model' / 'lit' / 'model.pth')
    write_ply(str(tmp_path / 'mesh.ply'), verts, tris)
    scfg = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}
    cfg = {'name': 'lit', 'network': 'material', 'mesh': str(tmp_path / 'mesh.ply'), 'shader_cfg': scfg}
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    run = lambda *a: subprocess.run([sys.executable, *a], cwd=tmp_path, env=env, capture_output=True, text=True)
    tools = os.path.join(ROOT, 'tools')
    p = run(os.path.join(tools, 'extract_lighting.py'), '--cfg', 'cfg.yaml', '--width', '64', '--height', '32', '--ssaa', '2',
            '--trans', '--exr')
    assert p.returncode == 0, p.stderr[-3000:]
    assert 'clamp' in p.stdout
    out = tmp_path / 'data' / 'lights' / 'lit-77'
    hdr, exr = load_env_map(str(out / 'outer_light.hdr')), load_env_map(str(out / 'outer_light.exr'))
    assert hdr.shape == (32, 64, 3) and (out / 'outer_light.png').exists()
    assert (np.abs(hdr - exr) <= exr.max(-1, keepdims=True) * 2.0 ** -8).all()
    p = run(os.path.join(tools, 'extract_materials.py'), '--cfg', 'cfg.yaml')
    assert p.returncode == 0, p.stderr[-3000:]
    p = run(os.path.join(tools, 'relight.py'), '--mesh', 'mesh.ply', '--material', 'data/materials/lit-77', '--hdr',
            str(out / 'outer_light.hdr'), '--name', 'self', '--trans', '--num', '1', '--width', '16', '--height', '16', '--samples', '2')
    assert p.returncode == 0, p.stderr[-3000:]
    _, ssd = stage1_net()
    os.makedirs(tmp_path / 'data' / 'model' / 'shp', exist_ok=True)
    torch.save({'step': 5, 'network_state_dict': ssd}, tmp_path / 'data' / 'model' / 'shp' / 'model.pth')
    (tmp_path / 'shape.yaml').write_text(yaml.safe_dump({'name': 'shp', 'network': 'shape'}))
    p = run(os.path.join(tools, 'extract_lighting.py'), '--cfg', 'shape.yaml', '--width', '16', '--height', '8', '--kappa', '0', '1')
    assert p.returncode == 0, p.stderr[-3000:]
    assert sorted(os.listdir(tmp_path / 'data' / 'lights' / 'shp-5')) == ['outer_light_k0.hdr', 'outer_light_k0.png', 'outer_light_k1.hdr',
                                                                         'outer_light_k1.png']
    (tmp_path / 'bad.yaml').write_text(yaml.safe_dump({'name': 'x', 'network': 'nerf'}))
    p = run(os.path.join(tools, 'extract_lighting.py'), '--cfg', 'bad.yaml')
    assert p.returncode != 0 and 'shape or a material network' in p.stderr
