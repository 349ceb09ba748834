"""GPU parity against the oracle AT THE SIZES BASELINE.json QUOTES (not only on the small golden fixtures):

  configs[1]  bell shape stage, 1024 rays x (64+64)+32 samples, steps 10 000 and 30 000 (occlusion march on)
  configs[2]  bear shape stage (human light), 2048 rays x (64+64)+32 samples
  configs[3]  bell material stage, P = 4096 surface points x (512+256) directions on the 21 760-triangle scene; the
              oracle re-computes a 256-point subset with the same per-point random draws
  + one gradient check (loss and per-parameter gradient norms) at 256 rays, full sampling depth.

With >= 994 row tiles of 128 samples every persistent CTA of the tensor-core kernels loops over several tiles here
(the golden fixtures never reach a second iteration), so mbarrier phase handling across tiles is under oracle comparison.
The oracle (CPU, fp32, `no_grad` forward) takes 10-40 s per case.

Tolerances: north_star's "RGB and SDF within 1e-4 relative": |err| <= 1e-4*|ref| + 2e-5 (the absolute term covers values
near zero, as in test_render_gpu.py); per-sample eikonal terms 2e-3 (ill-conditioned in sigma'); loss_occ 3e-3: its
candidate set is thresholded (|sdf| < 0.01, n.d < 0) and a handful of the ~10^5 samples sit within the 1e-5 SDF error of a
threshold, which moves single members of the 2048-point subset.
"""
import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mat as OM
from helpers import build_params, build_material_params

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _net(cfg):
    from nero_b200.renderer import NeROShapeRenderer
    sd = build_params(cfg)
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(sd)
    return net.cuda(), sd


def _viol(got, want, rtol, atol):
    got = got.detach().float().cpu().numpy().reshape(-1)
    want = np.asarray(want.detach() if torch.is_tensor(want) else want, dtype=np.float32).reshape(-1)
    assert got.shape == want.shape, (got.shape, want.shape)
    return np.abs(got - want) - (atol + rtol * np.abs(want)), np.abs(got - want)


def _close(got, want, rtol, atol, name):
    v, e = _viol(got, want, rtol, atol)
    assert v.max() <= 0, f'{name}: max violation {v.max():.3e}, max abs err {e.max():.3e} ({(v > 0).sum()} of {v.size} elements)'


def _shape_case(cfg, R, steps):
    net, sd = _net(cfg)
    rays = O.synthetic_rays(R, seed=6033)
    r = {k: v.to(DEV) for k, v in rays.items()}
    c = O.merged_cfg(cfg)
    lut = sd['color_network.FG_LUT'][0]
    z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
    S = z.shape[1]
    assert S == 160
    zc = z.cpu()
    # the occlusion loss keeps 2048 of its candidates: the first 2048 in sample order on both sides (renderer.py:535-541
    # draws a random permutation; `perm` replaces that draw)
    perm = torch.arange(R * S)
    for step in steps:
        car = O.get_anneal_val(c, step)
        with torch.no_grad():
            out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, step, perm=perm.to(DEV))
            ref = O.render_core(sd, c, lut, rays['rays_o'], rays['rays_d'], zc, rays['human_poses'], car, step, perm=perm)
        n_in = net.engine.state['N_in']
        assert (n_in + 127) // 128 > 4 * 132, 'every persistent CTA must loop over several row tiles in this test'
        assert ref['gradient_error'].shape[0] == n_in, 'inner / outer classification differs from the oracle'
        _close(out['ray_rgb'], ref['ray_rgb'], 1e-4, 2e-5, f'ray_rgb (R={R}, step {step})')
        v, e = _viol(out['gradient_error'], ref['gradient_error'], 2e-3, 2e-5)
        assert (v > 0).mean() <= 1e-5 and e.max() < 1e-2, f'gradient_error: {(v > 0).sum()} violations, max abs err {e.max():.2e}'
        _close(out['std'], ref['std'], 1e-6, 0, 'std')
        lo, lr_ = float(torch.as_tensor(out['loss_occ']).sum()), float(torch.as_tensor(ref['loss_occ']).sum())
        if step >= c['occ_loss_step']:
            assert net.engine.state['P'] == 2048 and lr_ > 0
        assert abs(lo - lr_) <= 3e-3 * abs(lr_) + 1e-7, ('loss_occ', lo, lr_)


def test_bell_1024_rays_render_core_matches_oracle():
    """BASELINE.json configs[1]: 1024 rays x (64+64)+32, sampled by the CUDA path, rendered by both."""
    _shape_case({}, 1024, [10000, 30000])


def test_bear_2048_rays_render_core_matches_oracle():
    """BASELINE.json configs[2]: human light (predict_human_light, field.py:536-552), 2048 rays x (64+64)+32."""
    _shape_case({'shader_config': {'human_light': True}}, 2048, [30000])


def test_gradients_256_rays_full_depth_match_oracle():
    """Loss and per-parameter gradient norms of one training step at 256 rays x (64+64)+32 (31 k inner samples, 250 row
    tiles) against autograd through the oracle."""
    cfg = {}
    net, sd = _net(cfg)
    R, step = 256, 30000
    rays = O.synthetic_rays(R, seed=6033)
    r = {k: v.to(DEV) for k, v in rays.items()}
    c = O.merged_cfg(cfg)
    car = O.get_anneal_val(c, step)
    z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
    perm = torch.arange(R * 160)
    net.zero_grad()
    out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, step, perm=perm.to(DEV))
    loss = O.training_loss(out, r['rgb'], c, step)
    loss.backward()
    torch.cuda.synchronize()
    p = {k: v.clone().requires_grad_(torch.is_floating_point(v) and not k.endswith('FG_LUT')) for k, v in sd.items()}
    ref = O.render_core(p, c, sd['color_network.FG_LUT'][0], rays['rays_o'], rays['rays_d'], z.cpu(), rays['human_poses'], car, step, perm=perm)
    lref = O.training_loss(ref, rays['rgb'], c, step)
    lref.backward()
    assert abs(float(loss) - float(lref)) <= 1e-4 * abs(float(lref)), (float(loss), float(lref))
    _close(out['ray_rgb'], ref['ray_rgb'], 1e-4, 2e-5, 'ray_rgb')
    bad = []
    for name, q in net.named_parameters():
        want = p[name].grad
        gn, wn = float(q.grad.double().norm()), float(want.double().norm())
        if abs(gn - wn) > 2e-3 * wn + 1e-7:
            bad.append((name, gn, wn))
        # direction as well as length: relative L2 distance of the whole tensor
        d = float((q.grad.cpu().double() - want.double()).norm())
        if d > 5e-3 * wn + 1e-7:
            bad.append((name + ' [distance]', d, wn))
    assert not bad, bad[:8]


def test_material_4096_points_match_oracle_on_a_subset():
    """BASELINE.json configs[3]: P = 4096 surface points x (512 diffuse + 256 specular) directions, 21 760-triangle scene.
    The CUDA path shades all 4096 points; the oracle re-computes every 16th point (256 points, 196 608 secondary rays) with the
    same per-point random draws.  Visibility comes from the CUDA BVH on both sides (the exhaustive tracer is compared with it
    separately below and in test_material_gpu.py): what is compared here is sampling, encodings, light / material MLPs and the
    Monte-Carlo estimator at full size.  A secondary ray that grazes the mesh may flip between hit and miss when its
    direction differs in the last bit; that moves a point by ~L/768, hence the quantile criterion."""
    from nero_b200.material import NeROMaterialRenderer
    scfg = {'diffuse_sample_num': 512, 'specular_sample_num': 256, 'outer_light_version': 'direction', 'light_exp_max': 5.0,
            'inner_light_exp_max': 5.0, 'human_lights': False}
    cfg = {'shader_cfg': scfg}
    verts, tris = OM.test_scene(5)
    assert tris.shape[0] >= 20000
    net = NeROMaterialRenderer(cfg, is_train=False, mesh=(verts, tris))
    sd = build_material_params(scfg)
    net.load_state_dict(sd)
    net = net.cuda()
    P, step = 4096, 5000
    rays = O.synthetic_rays(4 * P, seed=6033)
    inters, normals, depth, hit = net.trace(rays['rays_o'].to(DEV), rays['rays_d'].to(DEV))
    idx = torch.nonzero(hit[:, 0])[:P, 0]
    assert idx.shape[0] == P
    ic = idx.cpu()
    batch = {'pts': inters[idx].contiguous(), 'rays_d': rays['rays_d'].to(DEV)[idx].contiguous(), 'normals': normals[idx].contiguous(),
             'rgb': rays['rgb'].to(DEV)[idx].contiguous(), 'human_poses': rays['human_poses'].to(DEV)[idx].contiguous()}
    rands = OM.draw_rands(P)
    with torch.no_grad():
        out = net.shade_batch(batch, step, {k: v.to(DEV) for k, v in rands.items()})
    st = net.engine.state
    assert st['n_hit'] + st['n_miss'] == P * 768 and st['n_hit'] > 0
    sub = torch.arange(0, P, 16)
    sb = {k: v[sub.to(DEV)].cpu() for k, v in batch.items()}
    sr = {k: v[sub] for k, v in rands.items()}
    tabs = (OM.direction_samples(512), OM.direction_samples(256))
    trace_fn = lambda o, d: tuple(x.cpu() for x in net.trace(o.to(DEV).contiguous(), d.to(DEV).contiguous()))
    with torch.no_grad():
        ref = OM.material_train_outputs(sd, cfg, tabs, trace_fn, sb, step, sr)
    for k in ('metallic', 'roughness', 'albedo'):
        _close(out[k][sub.to(DEV)], ref[k], 1e-4, 1e-5, k)
    for k in ('rgb_pr', 'diffuse_light', 'specular_light', 'diffuse_color', 'specular_color'):
        got, want = out[k][sub.to(DEV)].cpu().numpy(), ref[k].numpy()
        err = np.abs(got - want).max(-1)
        ok = err <= 2e-4 * np.abs(want).max(-1) + 3e-5
        assert ok.mean() >= 0.98 and err.max() < 2e-2 * max(1.0, float(np.abs(want).max())), (k, ok.mean(), err.max())
    _close(out['loss_mat_reg'][sub.to(DEV)], ref['loss_mat_reg'], 2e-3, 2e-8, 'loss_mat_reg')
    # the BVH against the exhaustive tracer on this mesh: the secondary rays of 8 of the points
    o8 = sb['pts'][:8, None, :].expand(8, 64, 3).reshape(-1, 3)
    g = torch.Generator().manual_seed(9)
    d8 = torch.nn.functional.normalize(sb['normals'][:8, None, :] + torch.randn(8, 64, 3, generator=g), dim=-1).reshape(-1, 3)
    o8 = o8 + d8 * 1e-5
    want = OM.renderer_trace(verts, tris, o8, d8)
    got = trace_fn(o8, d8)
    agree = (want[3][:, 0] == got[3][:, 0]).float().mean()
    assert agree >= 0.99, agree
    both = want[3][:, 0] & got[3][:, 0]
    assert float((got[2][both] - want[2][both]).abs().median()) < 1e-5
