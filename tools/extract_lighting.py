"""Checkpoint -> the learned environment light as HDR maps (the outer light of stage I or stage II).

    python tools/extract_lighting.py --cfg configs/material/bell.yaml [--width 1024 --height 512 --ssaa 4] [--trans]
                                     [--center x y z] [--kappa 0 0.1 0.25 0.5 1] [--exr] [--exposure 0]

Loads data/model/<name>/model.pth ({'step', 'network_state_dict', ...}) and evaluates its outer light on an equirectangular
map in the convention of tools/relight.py (nero_b200/envmap.py states it):
  * a material (stage II) config writes data/lights/<name>-<step>/outer_light.hdr, outer_light(IDE(d, 0));
  * a shape (stage I) config writes outer_light_k<k>.hdr for every --kappa k, outer_light(IDE(d, k)): k = 1 is the diffuse
    light, smaller k the pre-filtered specular light at roughness k;
each with a clamped sRGB .png preview (and a float .exr with --exr).  --trans writes the map that matches relight.py --trans.
A sphere_direction light depends on where it is seen from: --center sets that point (the origin by default).  Not in the
map: the capturer's pose-dependent "human light" of real scenes and stage II's inner (indirect) light.  Prints the mean and
largest radiance and the fraction of texels at the exp(light_exp_max) clamp.  Paths are relative to the working directory.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--cfg', type=str, required=True)
    parser.add_argument('--width', type=int, default=1024)
    parser.add_argument('--height', type=int, default=512)
    parser.add_argument('--ssaa', type=int, default=4)
    parser.add_argument('--trans', action='store_true', help='the map relight.py --trans expects')
    parser.add_argument('--center', type=float, nargs=3, default=(0.0, 0.0, 0.0), metavar=('X', 'Y', 'Z'))
    parser.add_argument('--kappa', type=float, nargs='+', default=(0.0, 0.1, 0.25, 0.5, 1.0), help='stage I: kappa_inv values')
    parser.add_argument('--exr', action='store_true', help='also write float OpenEXR files')
    parser.add_argument('--exposure', type=float, default=0.0, help='preview exposure in stops')
    flags = parser.parse_args(argv)
    if flags.width < 1 or flags.height < 1 or not 1 <= flags.ssaa <= 16:
        parser.error('--width and --height must be positive and --ssaa in [1, 16]')
    if any(k < 0 for k in flags.kappa):
        parser.error('--kappa values must be non-negative')
    return flags


def load_cfg(path):
    import yaml
    with open(path) as f:
        cfg = yaml.safe_load(f)
    if not isinstance(cfg, dict) or cfg.get('network') not in ('shape', 'material'):
        net = cfg.get('network') if isinstance(cfg, dict) else None
        raise SystemExit(f"extract_lighting: {path} configures network '{net}'; the outer light comes from a shape or a "
                         'material network')
    return cfg


def main(argv=None):
    flags = parse(argv)
    cfg = load_cfg(flags.cfg)

    import torch
    from nero_b200 import envmap as EM

    if cfg['network'] == 'material':
        from nero_b200.material import NeROMaterialRenderer
        network = NeROMaterialRenderer(cfg, is_train=False)
    else:
        from nero_b200.renderer import NeROShapeRenderer
        network = NeROShapeRenderer(cfg, training=False)
    ckpt = torch.load(f'data/model/{cfg["name"]}/model.pth', map_location='cpu')
    step = ckpt['step']
    network.load_state_dict(ckpt['network_state_dict'])
    network = network.eval().cuda()
    print(f'successfully load {cfg["name"]} step {step}!')

    kw = dict(width=flags.width, height=flags.height, ssaa=flags.ssaa, center=tuple(flags.center), trans=flags.trans)
    if cfg['network'] == 'material':
        maps = {'outer_light': network.export_lighting(**kw)}
        exp_max = network.shader_network.cfg['light_exp_max']
    else:
        maps = {f'outer_light_k{k:g}': m for k, m in network.export_lighting(kappa_inv=flags.kappa, **kw).items()}
        exp_max = network.color_network.cfg['light_exp_max']
    out_dir = os.path.join('data', 'lights', f'{cfg["name"]}-{step}')
    os.makedirs(out_dir, exist_ok=True)
    for name, env in maps.items():
        base = os.path.join(out_dir, name)
        EM.write_hdr(base + '.hdr', env)
        EM.write_preview_png(base + '.png', env, flags.exposure)
        if flags.exr:
            EM.write_exr(base + '.exr', env)
        print(f'{base}.hdr: {flags.width} x {flags.height}, mean {float(env.mean()):.4f}, max {float(env.max()):.4f}, '
              f'{100 * EM.clamp_fraction(env, exp_max):.2f} % of texels at the exp({exp_max:g}) clamp')
    return out_dir


if __name__ == '__main__':
    main()
