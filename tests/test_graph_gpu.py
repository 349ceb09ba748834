"""cfg['cuda_graph']: train_step replayed from two captured CUDA graphs (nero_b200/graph.py) must produce what the eager
kernel sequence produces on the same rays -- same ray_rgb, same losses, same parameter gradients -- without reading any
count back to the host.  Tolerances: rgb 1e-6 (same kernels, same inputs); gradients norm-wise 1e-4."""
import sys
import os

import numpy as np
import pytest
import torch

from helpers import load_golden, build_params, rays_from_golden, FIXTURE_CFGS

sys.path.insert(0, os.path.join(os.path.dirname(__file__), '..'))
pytestmark = pytest.mark.gpu


def make(name, extra):
    import bench
    from nero_b200.renderer import NeROShapeRenderer
    g = load_golden(name)
    cfg = {**FIXTURE_CFGS[name], **extra}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(FIXTURE_CFGS[name], int(g['seed']), int(g['pseed'])))
    net = net.cuda()
    rays = rays_from_golden(g)
    R = rays['rays_o'].shape[0]
    net.cfg['train_ray_num'] = R
    bench.synthetic_dataset(net, rays, n_batches=6)
    return net, R


def one_step(net, step):
    net.zero_grad(set_to_none=True)
    out = net.train_step(step)
    loss = out['loss_rgb'].mean() + 0.1 * out['gradient_error'].mean() + out['loss_occ'].mean()
    loss.backward()
    torch.cuda.synchronize()
    grads = {n: p.grad.detach().clone() for n, p in net.named_parameters()}
    return {k: v.detach().clone() for k, v in out.items()}, float(loss), grads


@pytest.mark.parametrize('name,step', [('shape_bell_r32', 10000), ('shape_bell_r32', 30000), ('shape_bear_r24', 30000),
                                       ('shape_sphere_r16', 30000)])
def test_graphed_train_step_matches_eager(name, step):
    net, R = make(name, {'perturb': 0.0})
    net.cfg['cuda_graph'] = False
    ref_out, ref_loss, ref_g = one_step(net, step)
    net.cfg['cuda_graph'] = True
    for rep in range(3):                      # call 0 captures, calls 1-2 replay
        net.train_batch_i = 0
        out, loss, g = one_step(net, step)
        assert torch.allclose(out['ray_rgb'], ref_out['ray_rgb'], rtol=0, atol=1e-6), rep
        assert out['gradient_error'].numel() == 1
        assert abs(float(out['gradient_error']) - float(ref_out['gradient_error'].mean())) <= 1e-5 * abs(float(ref_out['gradient_error'].mean()))
        assert abs(float(out['loss_occ']) - float(ref_out['loss_occ'])) <= 1e-4 * abs(float(ref_out['loss_occ'])) + 1e-7
        assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss)
        for n in ref_g:
            d = (g[n] - ref_g[n]).norm().item()
            assert d <= 1e-4 * ref_g[n].norm().item() + 1e-9, (rep, n, d, ref_g[n].norm().item())


def test_graphed_steps_follow_the_ray_table_and_anneal():
    """Replays must see each step's rays and cos_anneal_ratio (device-side inputs), not the captured ones."""
    net, R = make('shape_bell_r32', {'perturb': 0.0, 'anneal_end': 50000})
    # second batch of the table = the rays in reverse order
    for k, v in net.train_batch.items():
        v[R:2 * R] = v[:R].flip(0)
    net.cfg['cuda_graph'] = True
    net.train_batch_i = 0
    a, _, _ = one_step(net, 30000)
    b, _, _ = one_step(net, 30000)           # reads rows R..2R
    assert torch.allclose(b['ray_rgb'], a['ray_rgb'].flip(0), atol=1e-6)
    net.cfg['cuda_graph'] = False
    net.train_batch_i = 0
    e1, _, g1 = one_step(net, 40000)         # other anneal value, same graph key
    net.cfg['cuda_graph'] = True
    net.train_batch_i = 0
    c, _, g2 = one_step(net, 40000)
    assert torch.allclose(c['ray_rgb'], e1['ray_rgb'], atol=1e-6)
    n = 'sdf_network.lin0.weight_v' if 'sdf_network.lin0.weight_v' in g1 else next(iter(g1))
    assert (g2[n] - g1[n]).norm() <= 1e-4 * g1[n].norm()


def test_occlusion_subset_is_drawn_on_the_device():
    """More candidates than occ_loss_max_pn: the graphed path selects exactly max_pn distinct candidates, uniformly
    (keys + top-k) -- checked through the engine's selection buffers."""
    net, R = make('shape_bell_r32', {'perturb': 0.0, 'occ_loss_max_pn': 64, 'occ_sdf_thresh': 10.0})
    net.cfg['cuda_graph'] = True
    seen = []
    for rep in range(3):
        net.train_batch_i = 0
        out, _, _ = one_step(net, 30000)
        e = net.engine
        g = next(iter(net._graphs.values()))
        cnt = int(e.w['OCC_COUNT'].item())
        assert cnt > 64 and int(g.P_dev.item()) == 64
        sel = e.occ_sel[:64].cpu().numpy()
        cand = np.sort(e.w['SEL'][:cnt].cpu().numpy())
        assert len(set(sel.tolist())) == 64 and np.isin(sel, cand).all()
        assert np.isfinite(float(out['loss_occ']))
        seen.append(tuple(sorted(sel.tolist())))
    assert len(set(seen)) > 1, 'the subset must be re-drawn every step'
