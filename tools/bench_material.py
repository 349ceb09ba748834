"""Stage II (BASELINE.json configs[3] / SURVEY.md 8d config 4: "bell material, 4096 surface samples") on one H100.

    python tools/bench_material.py [--points 4096] [--steps 10] [--warmup 3] [--no-cpu]

A step = NeROMaterialRenderer.shade_batch (512 diffuse + 256 specular directions per surface point -> 3.1 M secondary rays:
sampling, BVH tracing, encodings, light MLPs, estimator) + the YAML loss set ['nerf_render','mat_reg'] + backward + Adam.
Mesh: bumped icosphere, radius 0.5, 20 480 triangles, plus a 1280-triangle satellite (so ~10 % of the rays hit geometry).
Prints ONE JSON line (secondary measurement; the driver's line is bench.py's stage-I metric).
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

CFG = {'shader_cfg': {'diffuse_sample_num': 512, 'specular_sample_num': 256, 'outer_light_version': 'direction', 'light_exp_max': 5.0,
                      'inner_light_exp_max': 5.0, 'human_lights': False}, 'database_name': 'syn/bell'}
A_OUTER, A_INNER, A_MAT = 150272, 163328, 1078272      # MAC per row (SURVEY.md 8d)
STEP = 5000


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--points', type=int, default=4096)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--no-cpu', action='store_true')
    ap.add_argument('--cpu-points', type=int, default=16)
    args = ap.parse_args()
    from nero_b200 import synthetic as O
    from nero_b200 import synthetic as SY
    from nero_b200 import ops, params as PR
    from nero_b200.material import NeROMaterialRenderer
    dev = torch.device('cuda', 0)
    verts, tris = SY.test_scene(5)
    t0 = time.time()
    net = NeROMaterialRenderer(CFG, is_train=False, mesh=(verts, tris))
    sd = O.perturb_params(PR.build_material_state_dict(CFG['shader_cfg'], seed=6033))
    net.load_state_dict(sd)
    net = net.to(dev)
    _ = net.engine
    t_bvh = time.time() - t0
    P = args.points
    # primary hits through the CUDA tracer (the job _construct_ray_batch does at init, renderer.py:756-802)
    rays = O.synthetic_rays(4 * P, seed=6033)
    inters, normals, depth, hit = net.trace(rays['rays_o'].to(dev), rays['rays_d'].to(dev))
    idx = torch.nonzero(hit[:, 0])[:P, 0]
    assert idx.shape[0] == P
    batch = {'pts': inters[idx].contiguous(), 'rays_d': rays['rays_d'].to(dev)[idx].contiguous(), 'normals': normals[idx].contiguous(),
             'rgb': rays['rgb'].to(dev)[idx].contiguous(), 'human_poses': rays['human_poses'].to(dev)[idx].contiguous()}
    from nero_b200.optim import FlatAdam
    _ = net.engine
    opt = FlatAdam(net, lr=5e-4)

    def step():
        opt.zero_grad(set_to_none=True)
        out = net.shade_batch(batch, STEP)
        loss = sum(torch.mean(v) for k, v in out.items() if k.startswith('loss'))
        loss.backward()
        opt.step()
        return loss

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    l0 = ops.launch_count
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / args.steps
    launches = int((ops.launch_count - l0) // args.steps)
    st = net.engine.state
    S = 768
    n_hit, n_miss = st['n_hit'], st['n_miss']
    M = 2 * P
    flops = 2.0 * 3.0 * (n_miss * A_OUTER + n_hit * A_INNER + M * A_MAT)
    # phase breakdown of one extra step
    ev = []

    def mark(name):
        e = torch.cuda.Event(enable_timing=True)
        e.record()
        ev.append((name, e))
    eng = net.engine
    orig = dict(lf=eng.lights_forward, lb=eng.lights_backward, mf=eng.materials_forward, mb=eng.materials_backward)

    def wrap(fn, name):
        def f(*a, **k):
            mark(name + ':begin')
            r = fn(*a, **k)
            mark(name + ':end')
            return r
        return f
    eng.lights_forward, eng.lights_backward = wrap(orig['lf'], 'lights_fwd'), wrap(orig['lb'], 'lights_bwd')
    eng.materials_forward, eng.materials_backward = wrap(orig['mf'], 'materials_fwd'), wrap(orig['mb'], 'materials_bwd')
    step()
    torch.cuda.synchronize()
    phases = {}
    d = dict(ev)
    for n in ('lights_fwd', 'lights_bwd', 'materials_fwd', 'materials_bwd'):
        phases[n + '_ms'] = d[n + ':begin'].elapsed_time(d[n + ':end'])
    # tracing alone
    w = eng.w
    N = P * S
    e0.record()
    for _ in range(5):
        ops.K('nero_bvh_trace', eng.bvh_nodes, eng.bvh_tris, N, w['ORG'], 4, w['DIR'], 4, w['POSD'], w['NRMH'], 10.0, 1)
    e1.record()
    torch.cuda.synchronize()
    trace_ms = e0.elapsed_time(e1) / 5
    line = {'metric': 'stage-II train surface points/sec (768 secondary rays/point)', 'value': P / (ms * 1e-3), 'unit': 'points/s',
            'n_gpus': 1, 'steps': args.steps, 'warmup': args.warmup, 'ms_per_step': ms, 'higher_is_better': True, 'data': 'synthetic',
            'dtype': 'f32 (split-bf16 x3 tensor-core MMAs, fp32 accumulate)',
            'config': {'workload': f'bell_material_{P}pts_x_(512+256)dirs', 'triangles': int(tris.shape[0]), 'secondary_rays': N,
                       'rays_hit': n_hit, 'rays_miss': n_miss, 'bvh_build_s': t_bvh, 'optimizer': 'Adam (nero_adam_flat) inside the timed region'},
            'secondary_rays_per_s': N / (ms * 1e-3), 'gpu_launches': launches,
            'phases': phases, 'trace': {'ms': trace_ms, 'rays_per_s': N / (trace_ms * 1e-3)},
            'step_tensor_tflops': flops / (ms * 1e-3) / 1e12, 'cpu_baseline': None}
    if not args.no_cpu:
        import nero_oracle_mat as OM          # the CPU leg: the oracle port is what is timed here
        Pc = args.cpu_points
        tabs = (OM.direction_samples(512), OM.direction_samples(256))
        bc = {k: v[:Pc].cpu() for k, v in batch.items()}
        rands = OM.draw_rands(Pc)
        trace_fn = lambda o, d_: OM.renderer_trace(verts, tris, o, d_)
        torch.set_num_threads(min(64, os.cpu_count() or 1))

        def one():
            p = {k: v.clone().requires_grad_(torch.is_floating_point(v) and not k.endswith('light_pts')) for k, v in sd.items()}
            out = OM.material_train_outputs(p, CFG, tabs, trace_fn, bc, STEP, rands)
            OM.material_training_loss(out).backward()
        t0 = time.time()
        one()
        dt = time.time() - t0
        line['cpu_baseline'] = {'value': Pc / dt, 'unit': 'points/s', 'cores': torch.get_num_threads(), 'kind': 'port',
                                'sample': f'{Pc} surface points x 768 directions, brute-force tracer over {tris.shape[0]} triangles, one step'}
    print(json.dumps(line))


if __name__ == '__main__':
    main()
