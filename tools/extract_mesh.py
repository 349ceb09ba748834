"""Stage-I checkpoint -> triangle mesh for stage II, on the GPU (the reference's extract_mesh.py).

    python tools/extract_mesh.py --cfg configs/shape/syn/bell.yaml [--resolution 512]

Loads data/model/<name>/model.pth ({'step', 'network_state_dict', ...}), samples the SDF on a resolution^3 grid over [-1,1]^3
(1.0 outside the unit sphere), runs marching cubes at level 0 and writes data/meshes/<name>-<step>.ply, the path
NeROMaterialRenderer's `mesh` option and predict_materials read.  Paths are relative to the working directory.
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
    parser.add_argument('--resolution', type=int, default=512)
    flags = parser.parse_args(argv)

    import torch
    import yaml
    from nero_b200.mesh import write_ply
    from nero_b200.renderer import NeROShapeRenderer

    with open(flags.cfg) as f:
        cfg = yaml.safe_load(f)
    if cfg.get('network', 'shape') != 'shape':
        raise SystemExit(f"extract_mesh: {flags.cfg} configures network '{cfg['network']}'; meshes come from a shape network")
    network = NeROShapeRenderer(cfg, training=False)
    ckpt = torch.load(f'data/model/{cfg["name"]}/model.pth', map_location='cpu')
    step = ckpt['step']
    network.load_state_dict(ckpt['network_state_dict'])
    network = network.eval().cuda()
    print(f'successfully load {cfg["name"]} step {step}!')

    vertices, triangles = network.extract_mesh(resolution=flags.resolution, threshold=0.0)
    os.makedirs('data/meshes', exist_ok=True)
    path = os.path.join('data', 'meshes', f'{cfg["name"]}-{step}.ply')
    write_ply(path, vertices, triangles)
    print(f'{path}: {vertices.shape[0]} vertices, {triangles.shape[0]} triangles')
    return path


if __name__ == '__main__':
    main()
