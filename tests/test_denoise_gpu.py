"""Relit-frame denoising on the GPU: the AOV instances of the path tracer (colour bits, feature sums against the fp64 oracle,
chunking), the filter against the fp64 oracle on the same buffers, determinism, the noise reduction against a 1024-spp
frame and tools/relight.py --denoise end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_denoise as OD
import nero_oracle_mat as OM
from nero_b200 import denoise as DN
from nero_b200 import relight as RL
from test_relight_gpu import random_env, random_materials, scene_camera

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def relighter(kind, seed=11):
    verts, tris = OM.test_scene(2)
    if kind == 'vertex':
        mats = random_materials(verts.shape[0], seed)
    else:
        from nero_b200.texmap import uv_atlas
        vt, ft = uv_atlas(verts, tris, 64, 32, 2)
        rng = np.random.RandomState(seed)
        dec = lambda k: RL.srgb_to_linear(k / 255.0)
        mats = RL.UVMaterials(vt, ft, dec(rng.randint(0, 256, (16, 32, 3))), dec(rng.randint(0, 256, (16, 32))),
                              dec(rng.randint(150, 256, (16, 32))))
    return RL.Relighter(verts, tris, mats, random_env(12), 'schlick'), verts, tris


@pytest.mark.parametrize('kind', ['vertex', 'textured'])
def test_aov_sums_match_oracle_and_keep_the_colour_bits(kind):
    r, verts, tris = relighter(kind)
    h = w = 24
    spp, bounces = 3, 3
    pose, K = scene_camera(h, w)
    accum, aov = r.render_sums(pose, K, h, w, spp, bounces, seed=5)
    assert torch.equal(r.render(pose, K, h, w, spp, bounces, seed=5), accum / spp)
    materials = r.vmat if kind == 'vertex' else (r.uv.vt, r.uv.ft, r.tex)
    ra, rv = OD.features(verts, tris, materials, r.tables, pose, K, h, w, spp, bounces, seed=5, textured=kind == 'textured')
    ga, gv = accum.cpu().numpy().astype(np.float64), aov.cpu().numpy().astype(np.float64)
    np.testing.assert_array_equal(ga[..., 3], ra[..., 3])
    assert 0.1 < (ra[..., 3] > 0).mean() < 0.9
    for sl in (slice(4, 7), slice(8, 11), slice(12, 15), slice(15, 16)):          # guides: albedo, normal, point, depth
        scale = np.linalg.norm(rv[..., sl], axis=-1, keepdims=True)
        assert (np.abs(gv[..., sl] - rv[..., sl]) <= 1e-5 * scale + 1e-7).all(), (sl, np.abs(gv[..., sl] - rv[..., sl]).max())
    assert (gv[..., [7, 11]] == 0).all()
    for sl in (slice(0, 3), slice(3, 4)):                                          # demodulated radiance, luminance squares
        ok = np.abs(gv[..., sl] - rv[..., sl]) <= 1e-4 * np.abs(rv[..., sl]) + 1e-5
        assert ok.mean() >= 0.995, f'{(~ok).sum()} of {ok.size} values differ; max {np.abs(gv[..., sl] - rv[..., sl]).max():.3e}'


def test_aov_sums_are_chunking_invariant():
    r, _, _ = relighter('vertex', 3)
    pose, K = scene_camera(40, 48)
    a = r.render_sums(pose, K, 40, 48, 32, 4, seed=9, spp_per_launch=4)
    b = r.render_sums(pose, K, 40, 48, 32, 4, seed=9, spp_per_launch=32)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_filter_matches_oracle_and_is_deterministic():
    r, _, _ = relighter('vertex')
    h, w, spp = 40, 36, 16
    pose, K = scene_camera(h, w)
    accum, aov = r.render_sums(pose, K, h, w, spp, 4, seed=5)
    out = DN.denoise(accum, aov, spp, float(K[0, 0]))
    assert torch.equal(out, DN.denoise(accum, aov, spp, float(K[0, 0])))
    got = out.cpu().numpy().astype(np.float64)
    ref = OD.denoise(accum.cpu().numpy().astype(np.float64), aov.cpu().numpy().astype(np.float64), spp, float(K[0, 0]))
    np.testing.assert_array_equal(got[..., 3], accum[..., 3].cpu().numpy() / spp)
    ok = np.abs(got - ref) <= 1e-4 * np.abs(ref) + 1e-6
    assert ok.mean() >= 0.999, f'{(~ok).sum()} of {ok.size} values differ; max {np.abs(got - ref).max():.3e}'
    # render(denoise=True) is this sequence with the defaults
    assert torch.equal(r.render(pose, K, h, w, spp, 4, seed=5, denoise=True), out)


def test_denoised_frame_is_closer_to_the_converged_frame():
    """40^2 at 16 spp: the denoised frame's MSE against a 1024-spp frame (another seed) is at most 1/3 of the noisy frame's,
    over fully covered pixels."""
    r, _, _ = relighter('vertex')
    h = w = 40
    pose, K = scene_camera(h, w)
    noisy = r.render(pose, K, h, w, 16, 4, seed=5)
    den = r.render(pose, K, h, w, 16, 4, seed=5, denoise=True)
    ref = r.render(pose, K, h, w, 1024, 4, seed=6, spp_per_launch=64)
    full = (ref[..., 3] == 1) & (noisy[..., 3] == 1)
    assert int(full.sum()) > 400
    mse = lambda a: float(((a[..., :3] - ref[..., :3])[full] ** 2).mean())
    assert torch.equal(den[..., 3], noisy[..., 3])
    assert mse(den) * 3 <= mse(noisy), (mse(den), mse(noisy))


def test_tool_denoise_end_to_end(tmp_path):
    from test_relight_host import read_png, write_hdr
    from nero_b200.mesh import write_ply
    verts, tris = OM.test_scene(2)
    write_ply(str(tmp_path / 'mesh.ply'), verts, tris)
    RL.save_materials(str(tmp_path / 'mat'), random_materials(verts.shape[0], 4))
    write_hdr(tmp_path / 'env.hdr', random_env(7, 32, 64), rle=True)
    env = dict(os.environ, PYTHONPATH=ROOT)
    common = ['--mesh', 'mesh.ply', '--material', 'mat', '--hdr', 'env.hdr', '--num', '2', '--width', '28', '--height', '20',
              '--samples', '8', '--cam_dist', '2.0']
    for name, extra in (('plain', []), ('den', ['--denoise'])):
        subprocess.check_call([sys.executable, os.path.join(ROOT, 'tools', 'relight.py'), '--name', name] + common + extra,
                              cwd=tmp_path, env=env)
    for k in range(2):
        a = read_png(tmp_path / 'data' / 'relight' / 'plain' / f'{k}.png')
        b = read_png(tmp_path / 'data' / 'relight' / 'den' / f'{k}.png')
        assert a.shape == b.shape == (20, 28, 4)
        np.testing.assert_array_equal(a[..., 3], b[..., 3])
        assert (a[..., 3] > 0).any() and not np.array_equal(a, b)
