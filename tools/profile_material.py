"""A few stage-II training steps of the tools/bench_material.py workload, for a profiler run."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    sys.path.insert(0, p)
import torch
from nero_b200 import synthetic as O
from nero_b200 import synthetic as OM
from nero_b200 import params as PR
from nero_b200.material import NeROMaterialRenderer
sys.path.insert(0, os.path.join(ROOT, 'tools'))
import bench_material as BM
dev = torch.device('cuda')
verts, tris = OM.test_scene(5)
net = NeROMaterialRenderer(BM.CFG, is_train=False, mesh=(verts, tris))
net.load_state_dict(O.perturb_params(PR.build_material_state_dict(BM.CFG['shader_cfg'], seed=6033)))
net = net.to(dev)
P = int(os.environ.get('POINTS', 4096))
rays = O.synthetic_rays(4 * P, seed=6033)
inters, normals, depth, hit = net.trace(rays['rays_o'].to(dev), rays['rays_d'].to(dev))
idx = torch.nonzero(hit[:, 0])[:P, 0]
batch = {'pts': inters[idx].contiguous(), 'rays_d': rays['rays_d'].to(dev)[idx].contiguous(), 'normals': normals[idx].contiguous(),
         'rgb': rays['rgb'].to(dev)[idx].contiguous(), 'human_poses': rays['human_poses'].to(dev)[idx].contiguous()}
for i in range(int(sys.argv[1]) if len(sys.argv) > 1 else 2):
    net.zero_grad()
    out = net.shade_batch(batch, BM.STEP)
    sum(torch.mean(v) for k, v in out.items() if k.startswith('loss')).backward()
    torch.cuda.synchronize()
print('done', net.engine.state['n_hit'], net.engine.state['n_miss'])
