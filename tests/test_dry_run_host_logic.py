"""CPU: walk the host-side sequencing of both renderers with tests/dry_run_harness.py installed (every kernel launch
becomes a symbol lookup plus argument / shape assertions; tensors stay on the CPU).  Catches broken call sequences, buffer-shape mistakes and API
regressions of the Python layer without a GPU; numerical results are meaningless in this mode and are not checked."""
import os
import subprocess
import sys
import textwrap

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SCRIPT = textwrap.dedent('''
    import sys
    sys.path.insert(0, %r); sys.path.insert(0, %r + '/oracle'); sys.path.insert(0, %r + '/tests')
    import numpy as np, torch
    import nero_oracle as O, nero_oracle_mat as OM
    from nero_b200 import ops
    import dry_run_harness
    fake = dry_run_harness.install()
    from nero_b200.renderer import NeROShapeRenderer, name2renderer
    from nero_b200.material import NeROMaterialRenderer
    assert set(name2renderer) == {'shape', 'material'}

    # ---- stage I: training step at three schedule points, validation render, novel view, grid query
    for cfg in ({'n_samples': 32, 'n_importance': 32}, {'shader_config': {'human_light': True}}):
        net = NeROShapeRenderer(cfg, training=False)
        S = net.cfg['n_samples'] + net.cfg['n_importance'] + net.cfg['n_bg_samples']
        r = O.synthetic_rays(24, seed=1)
        for step in (500, 10000, 30000):
            net.zero_grad()
            out = net.render(r['rays_o'], r['rays_d'], r['near'], r['far'], r['human_poses'], -1, net.get_anneal_val(step), True, step)
            assert out['ray_rgb'].shape == (24, 3) and ('sdf_pts' in out) == (step < 1000)
            loss = torch.mean(net.compute_rgb_loss(out['ray_rgb'], r['rgb'])) + torch.mean(out['gradient_error']) + torch.mean(out['loss_occ'])
            if step < 1000:
                loss = loss + out['sdf_vals'].sum() * 0
            loss.backward()
            assert all(p.grad is not None for p in net.parameters())
        with torch.no_grad():
            val = net.render(r['rays_o'], r['rays_d'], r['near'], r['far'], r['human_poses'], 0, 0, False, 30000)
        for k in ('depth', 'normal', 'occ_prob_gt', 'specular_color', 'diffuse_albedo', 'indirect_light'):
            assert val[k].shape[0] == 24, k
        assert ('human_light' in val) == bool(cfg.get('shader_config', {}).get('human_light', False))
    pose = np.concatenate([np.eye(3), np.array([[0], [0], [3.0]])], 1)
    K = np.array([[40., 0, 16], [0, 40., 16], [0, 0, 1]])
    assert net.nvs(pose, K, 8, 12).shape == (8, 12, 3)
    assert net.sdf_network.sdf(torch.zeros(5, 7, 3)).shape == (5, 7, 1)

    # ---- the per-layer path (USE_CHAIN = False) runs the GEMM layers of the fused chains, in the same order
    import nero_b200.engine as E
    net = NeROShapeRenderer({'n_samples': 32, 'n_importance': 32}, training=False)

    def train(step):
        net.zero_grad()
        out = net.render(r['rays_o'], r['rays_d'], r['near'], r['far'], r['human_poses'], -1, net.get_anneal_val(step), True, step)
        loss = torch.mean(net.compute_rgb_loss(out['ray_rgb'], r['rgb'])) + torch.mean(out['gradient_error']) + torch.mean(out['loss_occ'])
        (loss + out['sdf_vals'].sum() * 0 if step < 1000 else loss).backward()

    def validation():
        with torch.no_grad():
            net.render(r['rays_o'], r['rays_d'], r['near'], r['far'], r['human_poses'], 0, 0, False, 30000)
    walks = {'step 500': lambda: train(500), 'step 30000': lambda: train(30000), 'validation render': validation,
             'materials_query': lambda: net.predict_materials(torch.rand(40, 3), batch_size=16),
             'sdf_query': lambda: net.sdf_network.sdf(torch.rand(5, 7, 3))}
    show = lambda g: (g[0].nrows, g[0].K, 'transposed' if g[1] else 'forward', g[2])
    differ = []
    for name, walk in walks.items():
        seqs = []
        for fused in (True, False):
            E.USE_CHAIN = fused
            dry_run_harness.GEMMS.clear()
            walk()
            seqs.append(list(dry_run_harness.GEMMS))     # (PreparedLayer, transposed, ncol_out); layers compare by identity
        if seqs[0] != seqs[1]:
            i = next((i for i, (a, b) in enumerate(zip(*seqs)) if a != b), min(map(len, seqs)))
            differ.append(f'{name}: {len(seqs[0])} fused / {len(seqs[1])} per-layer GEMM layers, first difference at #{i}: '
                          f'{[show(s[i]) if i < len(s) else None for s in seqs]}')
    E.USE_CHAIN = True
    assert not differ, differ

    # ---- stage II: train step (all shader variants), ray-batch construction through the tracer, image chunk loop
    verts, tris = OM.test_scene(1)
    for scfg in ({'human_lights': False}, {'human_lights': True, 'outer_light_version': 'sphere_direction', 'geometry_type': 'ggx_smith'}):
        scfg = dict(scfg, diffuse_sample_num=8, specular_sample_num=8)
        m = NeROMaterialRenderer({'shader_cfg': scfg}, is_train=False, mesh=(verts, tris))
        b = OM.synthetic_surface_batch(verts, tris, 6, seed=2)
        for step in (100, 5000):
            m.zero_grad()
            out = m.shade_batch(b, step)
            for k in ('rgb_pr', 'loss_rgb', 'loss_mat_reg', 'loss_diffuse_light', 'albedo', 'roughness', 'metallic', 'diffuse_light',
                      'specular_light', 'diffuse_color', 'specular_color', 'approximate_light', 'human_lights'):
                assert k in out, k
            sum(torch.mean(v) for k, v in out.items() if k.startswith('loss')).backward()
            assert all(p.grad is not None for p in m.parameters())
        info = {'imgs': torch.rand(2, 3, 6, 5), 'Ks': torch.tensor([[8., 0, 2.5], [0, 8., 3], [0, 0, 1]]).repeat(2, 1, 1),
                'poses': O.synthetic_rays(2, seed=3)['poses']}
        tb = m._construct_ray_batch(info)
        assert set(tb) == {'rays_o', 'rays_d', 'inters', 'normals', 'depth', 'human_poses', 'rgb'} and tb['human_poses'].shape[1:] == (3, 4)
        one = {k: v[:1] for k, v in info.items()}
        eb = m._construct_ray_batch(one, 'cpu', False)
        img = m.render_rays(eb, 6, 5)
        assert img['rgb_pr'].shape == (6, 5, 3) and img['roughness'].shape == (6, 5, 1)
        pm = m.predict_materials(batch_size=40)
        assert pm['albedo'].shape == (verts.shape[0], 3)
    from nero_b200.optim import FlatAdam
    opt = FlatAdam(m, lr=1e-3)
    opt.step(); opt.zero_grad()
    sd = opt.state_dict()
    assert len(sd['state']) == len(list(m.parameters())) and sd['param_groups'][0]['lr'] == 1e-3
    assert fake.calls > 1000

    # ---- stand-alone encodings, mesh extraction, shape evaluation and relighting wrappers
    x = torch.rand(7, 3)
    assert ops.positional_encoding(x, 6).shape == (7, 39) and ops.integrated_dir_enc(x, torch.rand(7, 1)).shape == (7, 72)
    assert ops.integrated_dir_enc(x, 0.5).shape == (7, 72)
    from nero_b200 import mesh as ME, evaluate as EV, relight as RL
    import contextlib
    torch.cuda.device = lambda dev: contextlib.nullcontext()     # marching_cubes_cuda selects the volume's device
    mv, mt = ME.marching_cubes_cuda(torch.rand(4, 5, 6))
    assert mv.shape == (6, 3) and mt.shape == (2, 3)
    dr = EV.DepthRenderer(verts, tris, device='cpu')
    d = dr.render(pose[:3], K, 4, 6)
    pts = EV.depth_to_points_cuda(torch.stack([d, d]), [pose[:3]] * 2, [K] * 2)
    assert pts.shape == (5, 3)
    assert EV.voxel_down_sample_cuda(torch.rand(9, 3)).shape[1] == 3
    assert EV.nearest_dist_cuda(torch.rand(4, 3), torch.rand(3, 3)).shape == (4,)
    mats = {'metallic': np.zeros((verts.shape[0], 1)), 'roughness': np.ones((verts.shape[0], 1)), 'albedo': np.ones((verts.shape[0], 3))}
    rl = RL.Relighter(verts, tris, mats, np.ones((4, 8, 3), np.float32), device='cpu')
    assert rl.render(pose[:3], K, 4, 6, 3, 2, spp_per_launch=2).shape == (4, 6, 4)
    print('DRY RUN OK')
''') % (ROOT, ROOT, ROOT)


def test_host_logic_walks_end_to_end_against_the_header_prototypes():
    env = dict(os.environ)
    r = subprocess.run([sys.executable, '-c', SCRIPT], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and 'DRY RUN OK' in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
