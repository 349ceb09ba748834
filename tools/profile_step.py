"""One training step of the bench workload, for a profiler run."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    sys.path.insert(0, p)
import torch
import bench
from nero_b200 import synthetic as O
dev = torch.device('cuda')
net, sd = bench.build_net({}, dev)
R = int(os.environ.get('RAYS', 1024))
rays = O.synthetic_rays(R, seed=6033)
r = {k: v.to(dev).contiguous() for k, v in rays.items()}
car = net.get_anneal_val(bench.STEP)
nsteps = int(sys.argv[1]) if len(sys.argv) > 1 else 2
for i in range(nsteps):
    net.zero_grad()
    z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
    out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, bench.STEP)
    bench.training_loss(net, out, r['rgb']).backward()
    torch.cuda.synchronize()
print('done', net.engine.state['N_in'])
