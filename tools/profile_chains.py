"""Developer tool: per-launch CUDA-event times of every fused-chain launch of one training step (bench workload)."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench
from nero_b200 import ops, synthetic as O
dev = torch.device('cuda')
net, sd = bench.build_net({}, dev)
rays = O.synthetic_rays(1024, seed=6033)
r = {k: v.to(dev).contiguous() for k, v in rays.items()}
car = net.get_anneal_val(bench.STEP)
def step():
    net.zero_grad()
    z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
    out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, bench.STEP)
    bench.training_loss(net, out, r['rgb']).backward()
    torch.cuda.synchronize()
for _ in range(2):
    step()
# patch chain() to record layer shapes
recs = []
orig = ops.chain
def chain(A0, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
    desc = f"{tag or '-'}:{len(layers)}L:k{layers[0]['kind']}:n{layers[0]['ncol_out']}"
    return orig(A0, k_valid0, layers, m_ptr, m_cap, tag=desc)
ops.chain = chain          # the engine's passes launch their chains through ops.mlp
ops.PROFILE = []
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); step(); e1.record(); torch.cuda.synchronize()
tot = 0.0
out = []
for tag, a, b, fl, mp, mc in ops.PROFILE:
    ms = a.elapsed_time(b) * 1e3
    tot += ms
    out.append((tag, round(ms, 1)))
print(json.dumps({'lib': os.environ.get('NERO_LIB', 'default'), 'step_ms': e0.elapsed_time(e1), 'chain_total_us': round(tot, 1), 'launches': out}))
