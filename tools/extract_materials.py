"""Stage-II checkpoint -> per-vertex materials (the reference's extract_materials.py).

    python tools/extract_materials.py --cfg configs/material/bell.yaml

Loads data/model/<name>/model.pth ({'step', 'network_state_dict', ...}), predicts the materials at the vertices of the
configured mesh on the GPU (NeROMaterialRenderer.predict_materials) and writes data/materials/<name>-<step>/
{metallic,roughness,albedo}.npy, [V,1], [V,1], [V,3] with linear_to_srgb applied as the reference does (see
nero_b200.relight.save_materials for why).  Paths are relative to the working directory.
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--cfg', type=str, required=True)
    flags = parser.parse_args(argv)

    import torch
    import yaml
    from nero_b200.material import NeROMaterialRenderer
    from nero_b200.relight import save_materials

    with open(flags.cfg) as f:
        cfg = yaml.safe_load(f)
    if cfg.get('network') != 'material':
        raise SystemExit(f"extract_materials: {flags.cfg} configures network '{cfg.get('network')}'; materials come from a material network")
    network = NeROMaterialRenderer(cfg, is_train=False)
    ckpt = torch.load(f'data/model/{cfg["name"]}/model.pth', map_location='cpu')
    step = ckpt['step']
    network.load_state_dict(ckpt['network_state_dict'])
    network = network.eval().cuda()
    print(f'successfully load {cfg["name"]} step {step}!')

    material_dir = os.path.join('data', 'materials', f'{cfg["name"]}-{step}')
    save_materials(material_dir, network.predict_materials())
    print(f'{material_dir}: metallic.npy, roughness.npy, albedo.npy (sRGB-encoded, as the reference writes them)')
    return material_dir


if __name__ == '__main__':
    main()
