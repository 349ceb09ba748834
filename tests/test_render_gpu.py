"""GPU parity of the CUDA hot path (through the NeROShapeRenderer API -> C ABI) against the golden vectors of the
unmodified reference and against the oracle on the same seeded inputs.

Tolerances (north_star: RGB and SDF within 1e-4 relative):
  * ray_rgb, sdf: |err| <= 1e-4*|ref| + 2e-5   (the atol covers values near zero; the fp32 reference itself moves by
    ~1e-5 when its BLAS blocking changes -- see DESIGN.md "error budget")
  * per-sample gradient_error / alpha: 2e-3 relative (ill-conditioned near sigma'(beta a) ~ 25)
  * parameter gradients: norm-wise 2e-3, element-wise 2e-2 of the tensor's max (ReLU-boundary flips)
  * sampled z: the inverse CDF is discontinuous in its inputs; we require 99% of samples within 1e-4 and check the
    sorted/bounded invariants exactly.
"""
import numpy as np
import pytest
import torch

import nero_oracle as O
from helpers import load_golden, build_params, t, rays_from_golden, FIXTURE_CFGS, FIXTURE_STEPS, VAL_FIXTURES

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def make_net(name):
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden(name)
    cfg = FIXTURE_CFGS[name]
    sd = build_params(cfg, int(g['seed']), int(g['pseed']))
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(sd)
    return net.cuda(), g, cfg, sd


def allclose(got, want, rtol, atol, name):
    got = got.detach().float().cpu().numpy().reshape(-1)
    want = np.asarray(want, dtype=np.float32).reshape(-1)
    assert got.shape == want.shape, f'{name}: shape {got.shape} vs {want.shape}'
    viol = np.abs(got - want) - (atol + rtol * np.abs(want))
    assert viol.max() <= 0, f'{name}: max violation {viol.max():.3e}, max abs err {np.abs(got - want).max():.3e}'


@pytest.mark.parametrize('name', list(FIXTURE_CFGS))
def test_sampling_matches_reference(name):
    net, g, cfg, sd = make_net(name)
    r = {k: v.to(DEV) for k, v in rays_from_golden(g).items()}
    c = O.merged_cfg(cfg)
    n_in = c['n_samples'] + c['n_importance']
    for gold, args in [(g['z_vals'], (0,)), (g['z_vals_perturbed'], (1.0, t(g['rand_inner']).to(DEV), t(g['rand_bg']).to(DEV)))]:
        z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], *args).cpu().numpy()
        d = np.abs(z - gold)
        assert (d[:, n_in:] < 1e-5 * np.abs(gold[:, n_in:]) + 1e-6).all(), 'background samples'
        # inverse-CDF sampling amplifies the ~1e-5 SDF differences of the split-bf16 MLP where a bin holds ~1e-5 of the
        # mass (the fp32 reference itself moves by up to 6e-4 when its BLAS blocking changes): quantile criteria
        frac4, frac3 = np.mean(d[:, :n_in] < 1e-4), np.mean(d[:, :n_in] < 1e-3)
        # a sample whose u lands on a CDF step can move by up to one bin of the level it was drawn in (<= (far-near)/n_samples)
        assert frac4 > 0.90 and frac3 > 0.995 and d[:, :n_in].max() < 2e-2, (frac4, frac3, d[:, :n_in].max())
        assert (np.diff(z[:, :n_in], axis=1) >= 0).all(), 'inner samples must be sorted'
        assert (z[:, 0] >= gold[:, 0] - 1e-5).all() and (z[:, n_in - 1] <= gold[:, n_in - 1] + 1e-5).all()


@pytest.mark.parametrize('name', list(FIXTURE_CFGS))
def test_render_core_matches_reference(name):
    net, g, cfg, sd = make_net(name)
    r = {k: v.to(DEV) for k, v in rays_from_golden(g).items()}
    c = O.merged_cfg(cfg)
    z = t(g['z_vals']).to(DEV)
    names = [str(n) for n in g['param_names']]
    for step in FIXTURE_STEPS[name]:
        net.zero_grad()
        out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], O.get_anneal_val(c, step), step)
        pre = f's{step}_'
        allclose(out['ray_rgb'], g[pre + 'ray_rgb'], 1e-4, 2e-5, 'ray_rgb')
        allclose(out['gradient_error'], g[pre + 'gradient_error'], 2e-3, 2e-5, 'gradient_error')
        allclose(out['std'], g[pre + 'std'], 1e-6, 0, 'std')
        allclose(out['loss_occ'], g[pre + 'loss_occ'], 1e-3, 1e-6, 'loss_occ')
        if step < 1000:
            allclose(out['sdf_pts'], g[pre + 'sdf_pts'], 1e-5, 1e-6, 'sdf_pts')
            allclose(out['sdf_vals'], g[pre + 'sdf_vals'], 1e-4, 2e-5, 'sdf_vals')
        loss = O.training_loss(out, r['rgb'], c, step)      # the YAML loss set incl. init_sdf_reg for step < 1000
        assert abs(float(loss) - float(g[pre + 'loss'])) <= 1e-4 * abs(float(g[pre + 'loss']))
        loss.backward()
        torch.cuda.synchronize()
        P = dict(net.named_parameters())
        gn = np.array([float(P[n].grad.double().norm()) for n in names])
        ref = g[pre + 'grad_norms']
        bad = np.abs(gn - ref) > 2e-3 * ref + 1e-7
        assert not bad.any(), [(names[i], gn[i], ref[i]) for i in np.nonzero(bad)[0][:5]]
        for k in g:
            if k.startswith(pre + 'grad::'):
                want = g[k]
                got = P[k.split('::')[1]].grad.cpu().numpy()
                assert np.abs(got - want).max() <= 2e-2 * np.abs(want).max() + 1e-9, k


def test_render_end_to_end_matches_oracle():
    """sample_ray + render_core through NeROShapeRenderer.render vs the oracle with identical random draws."""
    net, g, cfg, sd = make_net('shape_bell_full_r16')
    rays = rays_from_golden(g)
    r = {k: v.to(DEV) for k, v in rays.items()}
    c = O.merged_cfg(cfg)
    ri, rb = t(g['rand_inner']), t(g['rand_bg'])
    step = 30000
    z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 1.0, ri.to(DEV), rb.to(DEV))
    out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], O.get_anneal_val(c, step), step)
    lut = sd['color_network.FG_LUT'][0]
    with torch.no_grad():
        ref = O.render(sd, cfg, lut, rays['rays_o'], rays['rays_d'], rays['near'], rays['far'], rays['human_poses'],
                       O.get_anneal_val(c, step), step, rand_inner=ri, rand_bg=rb)
    allclose(out['ray_rgb'], ref['ray_rgb'].numpy(), 1e-4, 5e-5, 'ray_rgb end-to-end')


def test_sdf_values_match_reference_1e4():
    """SDF values of the wgmma MLP stack vs the fp32 reference network on random points (north_star: 1e-4)."""
    net, g, cfg, sd = make_net('shape_bell_r32')
    gen = torch.Generator().manual_seed(5)
    x = torch.rand(4096, 3, generator=gen) * 1.6 - 0.8
    with torch.no_grad():
        want = O.sdf_forward(sd, x)
    e = net.engine
    e.prepare_weights()
    e._alloc(32, 128)
    w = e.w
    from nero_b200.ops import K, Mat
    pe = O.embed(x, 6).to(DEV)
    w['SX0'][:4096, :39] = pe
    w['SC'][:4096, 217:256] = pe * 0.7071067811865476
    e.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, 4096)
    allclose(w['SSDF'][:4096, 0], want[:, 0].numpy(), 1e-4, 2e-5, 'sdf')


@pytest.mark.parametrize('name', list(VAL_FIXTURES))
def test_validation_render_matches_reference(name):
    """render_core(is_train=False): depth / normal / shading intermediates / occ_prob_gt (network/renderer.py:465-482)."""
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden(name)
    cfg = VAL_FIXTURES[name]
    sd = build_params(cfg, int(g['seed']), int(g['pseed']))
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(sd)
    net = net.cuda()
    r = {k: v.to(DEV) for k, v in O.synthetic_rays(int(g['R']), seed=int(g['seed'])).items()}
    c = O.merged_cfg(cfg)
    step = int(g['step'])
    with torch.no_grad():
        out = net.render_core(r['rays_o'], r['rays_d'], t(g['z_vals']).to(DEV), r['human_poses'], O.get_anneal_val(c, step), step,
                              is_train=False)
    keys = [k[4:] for k in g if k.startswith('val_')]
    assert set(keys) == set(out.keys()), set(keys) ^ set(out.keys())
    tol = {'gradient_error': (2e-3, 2e-5), 'loss_occ': (1e-3, 1e-6), 'occ_prob_gt': (2e-3, 2e-4), 'normal': (2e-4, 1e-4)}
    for k in keys:
        rt, at = tol.get(k, (2e-4, 3e-5))
        allclose(out[k], g['val_' + k], rt, at, k)


def test_sdf_grid_query_matches_oracle():
    """network.sdf_network.sdf(x) as extract_mesh.py:27 / field.py:1090-1117 use it (value-only, arbitrary points)."""
    net, g, cfg, sd = make_net('shape_bell_r32')
    gen = torch.Generator().manual_seed(5)
    x = torch.rand(150001, 3, generator=gen) * 2 - 1          # > one workspace chunk, ragged tail
    got = net.sdf_network.sdf(x.to(DEV))
    assert got.shape == (150001, 1)
    with torch.no_grad():
        want = O.sdf_forward(sd, x[:20000])[..., :1]
    allclose(got[:20000], want.numpy(), 1e-4, 2e-5, 'sdf grid query')
    # chunk boundary / tail: same values when queried alone
    again = net.sdf_network.sdf(x[131000:].to(DEV))
    assert torch.equal(again, got[131000:])


def test_predict_materials_and_sdf_field_match_reference():
    """NeROShapeRenderer.predict_materials (network/renderer.py:629-647) and the extract_fields grid behind val_geometry /
    extract_mesh.py (field.py:1090-1104) against the unmodified reference."""
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden('shape_materials_field')
    cfg = {'n_samples': 32, 'n_importance': 32}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(cfg, int(g['seed']), int(g['pseed'])))
    net = net.cuda()
    pm = net.predict_materials(g['xyz'], batch_size=128)          # several chunks, ragged tail
    assert pm['albedo'].shape == (300, 3) and pm['metallic'].shape == (300, 1)
    for k in ('metallic', 'roughness', 'albedo'):
        allclose(torch.from_numpy(pm[k]), g[k], 1e-4, 1e-5, k)
    u = net.extract_fields(resolution=24)
    allclose(torch.from_numpy(u), g['field24'], 1e-4, 2e-5, 'sdf field')
    net.cfg['val_geometry'] = True
    try:
        import mcubes  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError):       # the marching-cubes step is the host repo's third-party dependency
            net.extract_geometry(resolution=16)


@pytest.fixture
def per_layer(monkeypatch):
    """The engine's per-layer MLP path: every pass expanded into one nero_linear launch per layer (USE_CHAIN = False)."""
    from nero_b200 import engine
    monkeypatch.setattr(engine, 'USE_CHAIN', False)


@pytest.mark.parametrize('name', list(FIXTURE_CFGS))
def test_render_core_per_layer_matches_reference(name, per_layer):
    test_render_core_matches_reference(name)


def test_sdf_values_per_layer_match_reference_1e4(per_layer):
    test_sdf_values_match_reference_1e4()


@pytest.mark.parametrize('name', list(VAL_FIXTURES))
def test_validation_render_per_layer_matches_reference(name, per_layer):
    test_validation_render_matches_reference(name)


def test_predict_materials_per_layer_match_reference(per_layer):
    """Fails when the per-layer path skips the SDF feature head that feeds the material predictors."""
    test_predict_materials_and_sdf_field_match_reference()


def test_standalone_encodings_match_reference():
    """nero_pe / nero_ide (the stand-alone entry points of the encodings) against the reference KATs, including directions
    within 1e-4 .. 5e-2 of the poles where the reference's fp32 l=16 band is 2.4e-3 away from exact arithmetic."""
    from nero_b200 import ops
    g = load_golden('kat_encodings')
    x = t(g['x']).to(DEV)
    for L in (4, 6, 8):
        allclose(ops.positional_encoding(x, L), g[f'pe{L}'], 1e-5, 2e-6, f'pe{L}')
    allclose(ops.positional_encoding(t(g['x4']).to(DEV), 10), g['pe10_4'], 1e-5, 4e-5, 'pe10 (4-d)')     # sin(512 x): argument rounding
    allclose(ops.integrated_dir_enc(t(g['ide_dirs']).to(DEV), t(g['ide_kappa']).to(DEV)), g['ide'], 1e-5, 1.2e-5, 'ide')
    gp = load_golden('kat_ide_poles')
    allclose(ops.integrated_dir_enc(t(gp['dirs']).to(DEV), t(gp['kappa']).to(DEV)), gp['ide'], 1e-5, 1.2e-5, 'ide near the poles')
    allclose(ops.integrated_dir_enc(t(gp['dirs']).to(DEV), 0.0), O.ide(t(gp['dirs']), torch.zeros(1, 1)).numpy(), 1e-5, 1.2e-5, 'ide, scalar kappa')
