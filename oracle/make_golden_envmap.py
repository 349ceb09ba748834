"""Generate tests/golden/envmap_*.npz by running the UNMODIFIED reference's outer lights on CPU via ref_shim.

Run in the build container only (the reference does not exist on the GPU box):
    python oracle/make_golden_envmap.py
Each fixture is a 16 x 8 map at ssaa 2 (512 sub-sample directions from nero_oracle_envmap.directions) on seeded, perturbed
parameters (nero_b200.params + nero_oracle.perturb_params, regenerated from the seeds and scale stored in the fixture):
  * stage II: MCShadingNetwork.predict_outer_lights (network/field.py:836-854) with 'direction', and with
    'sphere_direction' seen from the origin and from an off-centre point inside the unit sphere;
  * stage I: color_network.outer_light(color_network.sph_enc(d, k)) at k = 0, 0.3, 1 (field.py:556, 564, 581, 588), and the
    sphere_direction input built from the reference's own offset_points_to_sphere / get_sphere_intersection (field.py:559-562), seen from a point outside the 0.999 sphere.
Stored: the directions, the reference's radiance per sub-sample and the map resolved from it (nero_oracle_envmap.resolve).
TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
import warnings

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
warnings.filterwarnings('ignore')

import ref_shim  # noqa: E402
import nero_oracle as O  # noqa: E402
import nero_oracle_envmap as OE  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')
W, H, SSAA = 16, 8, 2
SEED, PSEED, REL = 6033, 11, 0.3   # a larger perturbation than the training fixtures': the light varies over the sphere
INSIDE = (0.3, -0.2, 0.25)         # stage II sees the light from a surface point, inside the unit sphere
OUTSIDE = (0.7, -0.6, 0.5)         # |c| = 1.05 > 0.999: stage I's offset_points_to_sphere pulls it back

# name -> (stage, sphere_direction, kappa_inv, centre)
CASES = {
    'envmap_s2_direction': (2, False, 0.0, (0.0, 0.0, 0.0)),
    'envmap_s2_sphere_origin': (2, True, 0.0, (0.0, 0.0, 0.0)),
    'envmap_s2_sphere_off': (2, True, 0.0, INSIDE),
    'envmap_s1_k000': (1, False, 0.0, (0.0, 0.0, 0.0)),
    'envmap_s1_k030': (1, False, 0.3, (0.0, 0.0, 0.0)),
    'envmap_s1_k100': (1, False, 1.0, (0.0, 0.0, 0.0)),
    'envmap_s1_sphere_k030': (1, True, 0.3, OUTSIDE),
}


def stage2(sphere, centre, d):
    from nero_b200 import params as PR
    scfg = {'human_lights': False, 'outer_light_version': 'sphere_direction' if sphere else 'direction'}
    shader = ref_shim.build_reference_mc_shader(dict(scfg), None, seed=SEED)
    sd_ref = {'shader_network.' + k: v.detach().clone() for k, v in shader.state_dict().items()}
    mine = PR.build_material_state_dict(scfg, seed=SEED)
    assert list(mine.keys()) == list(sd_ref.keys()) and all(torch.equal(mine[k], sd_ref[k]) for k in sd_ref)
    sd = O.perturb_params(sd_ref, seed=PSEED, rel=REL)
    shader.load_state_dict({k[len('shader_network.'):]: v for k, v in sd.items()})
    pts = torch.tensor(centre, dtype=torch.float32).expand(d.shape[0], 3).contiguous()
    with torch.no_grad():
        return shader.predict_outer_lights(pts, d), float(shader.cfg['light_exp_max'])


def stage1(sphere, kappa, centre, d):
    from nero_b200 import params as PR
    cfg = {'shader_config': {'sphere_direction': sphere}}
    net = ref_shim.build_reference_shape_renderer(cfg, seed=SEED)
    sd_ref = {k: v.detach().clone() for k, v in net.state_dict().items()}
    mine = PR.build_shape_state_dict(cfg, seed=SEED)
    assert all(torch.equal(mine[k], sd_ref[k]) for k in sd_ref)
    net.load_state_dict(O.perturb_params(sd_ref, seed=PSEED, rel=REL))
    from network.field import offset_points_to_sphere, get_sphere_intersection
    cn = net.color_network
    rough = torch.full((d.shape[0], 1), kappa)
    with torch.no_grad():
        enc = cn.sph_enc(d, rough)
        if sphere:
            pts = torch.tensor(centre, dtype=torch.float32).expand(d.shape[0], 3).contiguous()
            sp = offset_points_to_sphere(pts)
            sp = torch.nn.functional.normalize(sp + d * get_sphere_intersection(sp, d), dim=-1)
            enc = torch.cat([enc, cn.sph_enc(sp, rough)], -1)
        return cn.outer_light(enc), float(cn.cfg['light_exp_max'])


def main():
    ref_shim.install()
    d = torch.from_numpy(OE.directions(W, H, SSAA))
    for name, (stage, sphere, kappa, centre) in CASES.items():
        rad, exp_max = stage2(sphere, centre, d) if stage == 2 else stage1(sphere, kappa, centre, d)
        rad = rad.float().numpy()
        out = {'dirs': d.numpy(), 'rad': rad, 'env': OE.resolve(rad, W, H, SSAA), 'stage': stage, 'sphere': int(sphere),
               'kappa_inv': np.float32(kappa), 'center': np.asarray(centre, np.float32), 'exp_max': np.float32(exp_max),
               'width': W, 'height': H, 'ssaa': SSAA, 'seed': SEED, 'pseed': PSEED, 'rel': np.float32(REL)}
        np.savez_compressed(os.path.join(GOLD, name + '.npz'), **out)
        print(f'{name}: radiance in [{rad.min():.4f}, {rad.max():.4f}]')


if __name__ == '__main__':
    main()
