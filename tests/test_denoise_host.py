"""CPU checks of the relit-frame denoiser: invariants of the fp64 oracle filter (constants, alpha, uncovered pixels, the
luminance, normal and position stops), its noise reduction on a synthetic image, the bindings and constants of
include/nero_denoise.h, the entry points' refusals and the --denoise flag of tools/relight.py.  No GPU."""
import os
import re
import sys

import numpy as np
import pytest

import nero_oracle_denoise as OD
import nero_oracle_relight as OR
from nero_b200 import denoise as DN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FOCAL = 50.0


def sums(D, g, n, x, z, hits, spp):
    """Feature sums of `hits` [h,w] identical samples per pixel with demodulated radiance D [h,w,3], albedo g, normal n,
    point x [h,w,3] and depth z [h,w] -> (accum, aov) as the path tracer writes them."""
    h, w = hits.shape
    k = hits[..., None].astype(np.float64)
    L = D * (g + OD.DEMOD_EPS)
    accum = np.concatenate([L * k, k], -1)
    aov = np.zeros((h, w, OD.AOV))
    aov[..., 0:3], aov[..., 3] = D * k, OR.luminance(D) ** 2 * hits
    aov[..., 4:7], aov[..., 8:11], aov[..., 12:15], aov[..., 15] = g * k, n * k, x * k, z * hits
    return accum, aov


def plane(h, w, spp=4, seed=0):
    """A camera-facing plane at depth 2: unit normals, points one footprint apart, random albedo and colour, all covered."""
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    x = np.stack([xx, yy, np.zeros_like(xx)], -1) * (2.0 / FOCAL)
    n = np.broadcast_to([0.0, 0.0, 1.0], (h, w, 3))
    return dict(D=rng.rand(h, w, 3), g=rng.rand(h, w, 3), n=n, x=x, z=np.full((h, w), 2.0), hits=np.full((h, w), spp), spp=spp)


def test_constant_colour_and_guides_are_unchanged():
    s = plane(24, 20)
    s['D'][:] = [0.3, 0.7, 0.2]
    s['g'][:] = [0.5, 0.25, 0.8]
    accum, aov = sums(s['D'], s['g'], s['n'], s['x'], s['z'], s['hits'], s['spp'])
    out = OD.denoise(accum, aov, s['spp'], FOCAL)
    assert np.abs(out - accum / s['spp']).max() <= 1e-12


def test_alpha_passes_through_and_uncovered_pixels_change_nothing():
    rng = np.random.RandomState(1)
    s = plane(24, 20, spp=8)
    s['hits'] = rng.randint(0, 9, (24, 20))
    s['hits'][:, :3] = 0
    accum, aov = sums(s['D'], s['g'], s['n'], s['x'], s['z'], s['hits'], 8)
    aov += rng.rand(*aov.shape) * (s['hits'][..., None] > 0)           # per-sample noise in every feature sum
    out = OD.denoise(accum, aov, 8, FOCAL)
    np.testing.assert_array_equal(out[..., 3], s['hits'] / 8)
    assert (out[s['hits'] == 0] == 0).all()
    a2, v2 = accum.copy(), aov.copy()
    zero = s['hits'] == 0
    a2[zero, :3] = rng.rand(int(zero.sum()), 3) * 100
    v2[zero] = rng.randn(int(zero.sum()), OD.AOV) * 100
    np.testing.assert_array_equal(OD.denoise(a2, v2, 8, FOCAL), out)


def test_luminance_stop_at_zero_variance():
    """Two constant halves of different luminance and no variance: no weight crosses the step."""
    s = plane(16, 24)
    s['g'][:] = 0.5
    s['D'][:, :12] = 0.2
    s['D'][:, 12:] = 1.5
    accum, aov = sums(s['D'], s['g'], s['n'], s['x'], s['z'], s['hits'], s['spp'])
    col, feat = OD.prep(accum, aov, s['spp'], FOCAL)
    assert np.abs(col[..., 3]).max() <= 1e-15
    out = OD.denoise(accum, aov, s['spp'], FOCAL)
    assert np.abs(out - accum / s['spp']).max() <= 1e-12


@pytest.mark.parametrize('step', ['normal', 'position'])
def test_geometry_steps_are_not_blurred_across(step):
    """Halves with different colours and one sample each (no luminance stop): a normal or depth step keeps them apart,
    and without it they mix."""
    s = plane(16, 24, spp=1)
    s['g'][:] = 0.5
    s['D'][:, :12] = 0.2
    s['D'][:, 12:] = 1.5
    if step == 'normal':
        s['n'] = s['n'].copy()
        s['n'][:, 12:] = [1.0, 0.0, 0.0]
    else:
        s['x'] = s['x'].copy()
        s['x'][:, 12:, 2] += 8.0          # 200 footprints; the stop at step 16 is 1.4 * 16 = 22.4 footprints wide
    accum, aov = sums(s['D'], s['g'], s['n'], s['x'], s['z'], s['hits'], 1)
    assert (OD.prep(accum, aov, 1, FOCAL)[0][..., 3] == OD.VAR_NONE).all()
    out = OD.denoise(accum, aov, 1, FOCAL)
    assert np.abs(out - accum).max() <= 1e-12
    flat = plane(16, 24, spp=1)
    accum2, aov2 = sums(s['D'], s['g'], flat['n'], flat['x'], flat['z'], s['hits'], 1)
    assert np.abs(OD.denoise(accum2, aov2, 1, FOCAL) - accum2).max() > 0.1


def test_filter_reduces_gaussian_noise():
    """A smooth image with Gaussian per-sample noise: the filter cuts the MSE against the truth by at least 4x."""
    h, w, spp, sigma = 48, 48, 4, 0.15
    rng = np.random.RandomState(5)
    yy, xx = np.mgrid[0:h, 0:w] / 48.0
    truth = np.stack([0.5 + 0.3 * np.sin(3 * xx), 0.4 + 0.2 * np.cos(2 * yy), 0.3 + 0.2 * xx * yy], -1)
    s = plane(h, w, spp)
    g = np.full((h, w, 3), 0.6)
    samples = truth[None] + sigma * rng.randn(spp, h, w, 3)
    accum, aov = sums(samples.mean(0), g, s['n'], s['x'], s['z'], s['hits'], spp)
    aov[..., 3] = (OR.luminance(samples) ** 2).sum(0)                   # the per-sample luminance squares
    noisy = accum[..., :3] / spp
    ref = truth * (g + OD.DEMOD_EPS)
    out = OD.denoise(accum, aov, spp, FOCAL)
    mse_noisy, mse_out = ((noisy - ref) ** 2).mean(), ((out[..., :3] - ref) ** 2).mean()
    assert mse_out * 4 <= mse_noisy, (mse_noisy, mse_out)


# ------------------------------------------------------------------------------------------------ bindings and the tool
def header():
    return open(os.path.join(ROOT, 'include', 'nero_denoise.h')).read()


def test_header_binding_and_constants():
    from nero_b200 import ops
    txt = re.sub(r'/\*.*?\*/', ' ', header(), flags=re.S)
    names = set(re.findall(r'\bint\s+(nero_\w+)\s*\(', txt))
    assert names == set(ops.DENOISE_PROTOS) == {'nero_relight_render_aov', 'nero_relight_render_textured_aov', 'nero_denoise_prep',
                                                'nero_denoise_iterate', 'nero_denoise_finish'}
    for name, argtypes in ops.DENOISE_PROTOS.items():
        assert getattr(ops.lib, name).argtypes == argtypes
    assert [len(ops.DENOISE_PROTOS[n]) for n in sorted(names)] == [6, 11, 9, 3, 9]
    defs = dict(re.findall(r'#define NERO_DENOISE_(\w+) ([0-9.e+-]+)f?', header()))
    assert int(defs['AOV']) == DN.AOV == OD.AOV and int(defs['MAX_LEVEL']) + 1 == DN.MAX_ITERATIONS
    assert float(defs['DEMOD_EPS']) == DN.DEMOD_EPS == OD.DEMOD_EPS and float(defs['VAR_NONE']) == DN.VAR_NONE == OD.VAR_NONE
    assert (int(defs['ITERATIONS']), float(defs['SIGMA_L']), float(defs['SIGMA_N']), float(defs['SIGMA_X']), float(defs['EPS'])) == \
        (DN.ITERATIONS, DN.SIGMA_L, DN.SIGMA_N, DN.SIGMA_X, DN.EPS)
    # the relighting record is unchanged
    assert ops.ctypes.sizeof(ops.RelightParams) == ops.lib.nero_abi_sizeof(ops.ABI_RECORDS.index('nero_relight_params'))


def test_entry_point_refusals():
    """Every refusal returns 1 before anything reaches the GPU."""
    from nero_b200 import ops
    fake, s = 0x1000, None
    prep = (fake, fake, 4, 8, 8, 50.0, fake, fake, s)
    for i, bad in ((0, None), (1, None), (2, 0), (3, 0), (4, 0), (5, 0.0), (5, -1.0), (6, None), (7, None)):
        args = list(prep)
        args[i] = bad
        assert ops.lib.nero_denoise_prep(*args) == 1, i
    it = (fake, 0x2000, 8, 8, 0, 4.0, 64.0, 1.4, 1e-3, 0x3000, s)
    for i, bad in ((0, None), (1, None), (2, 0), (3, 0), (4, -1), (4, 8), (5, 0.0), (6, 0.0), (7, -1.0), (8, 0.0), (9, None),
                   (9, fake)):
        args = list(it)
        args[i] = bad
        assert ops.lib.nero_denoise_iterate(*args) == 1, i
    for i, bad in ((0, None), (1, None), (2, 0), (3, 0), (4, None)):
        args = [fake, fake, 8, 8, fake, s]
        args[i] = bad
        assert ops.lib.nero_denoise_finish(*args) == 1, i
    q = ops.RelightParams().set(nodes=fake, tris=fake, tri_ids=fake, faces=fake, vmat=fake, env=fake, env_p=fake, cdf_rows=fake,
                                cdf_cols=fake, accum=fake)
    q.env_w, q.env_h, q.width, q.height, q.spp0, q.spp, q.max_bounces = 4, 2, 8, 8, 0, 0, 1
    assert ops.lib.nero_relight_render_aov(ops.ctypes.byref(q), fake, s) == 0          # spp = 0 launches nothing
    assert ops.lib.nero_relight_render_aov(ops.ctypes.byref(q), None, s) == 1
    q.vmat = None
    assert ops.lib.nero_relight_render_aov(ops.ctypes.byref(q), fake, s) == 1
    assert ops.lib.nero_relight_render_textured_aov(ops.ctypes.byref(q), fake, fake, 3, fake, 4, 2, fake, s) == 0
    assert ops.lib.nero_relight_render_textured_aov(ops.ctypes.byref(q), fake, fake, 3, fake, 4, 2, None, s) == 1


def test_denoise_argument_checks():
    import torch
    a, v = torch.zeros(4, 4, 4), torch.zeros(4, 4, 16)
    with pytest.raises(ValueError, match='expected'):
        DN.denoise(a, torch.zeros(4, 4, 12), 4, 50.0)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        DN.denoise(a, v, 4, 50.0)


def test_tool_denoise_flag():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import relight
    common = ['--mesh', 'm.ply', '--material', 'mat', '--hdr', 'e.hdr', '--name', 'n']
    assert relight.parse(common).denoise is False
    assert relight.parse(common + ['--denoise', '--samples', '64']).denoise is True
