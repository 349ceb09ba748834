"""Stage-II checkpoint -> UV texture maps and a textured OBJ (the reference's extract_materials_texture_map.py).

    python tools/extract_materials_texture_map.py --cfg configs/material/bell.yaml [--size 1024] [--ssaa 2] [--out n2m_test]

Loads data/model/<name>/model_best.pth ({'step', 'network_state_dict', ...}), unwraps the configured mesh into a
(ssaa size)^2 atlas with a gutter of 2 output texels, bakes albedo / metallic / roughness on the GPU and writes
<out>/feat0_0.png, feat1_0.png, feat2_0.png (size x size), mesh_0.obj and mesh_0.mtl.  The protocol, and how it differs
from the reference (PNG instead of JPEG, fp32 instead of fp16, this project's unwrapper instead of xatlas), is stated in
nero_b200/texmap.py.  Paths are relative to the working directory.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--cfg', type=str, required=True)
    parser.add_argument('--size', type=int, default=1024)
    parser.add_argument('--ssaa', type=int, default=2, choices=(1, 2))
    parser.add_argument('--out', type=str, default='n2m_test')
    flags = parser.parse_args(argv)

    import torch
    import yaml
    from nero_b200 import texmap as TX
    from nero_b200.material import NeROMaterialRenderer

    with open(flags.cfg) as f:
        cfg = yaml.safe_load(f)
    if cfg.get('network') != 'material':
        raise SystemExit(f"extract_materials_texture_map: {flags.cfg} configures network '{cfg.get('network')}'; "
                         'materials come from a material network')
    network = NeROMaterialRenderer(cfg, is_train=False)
    ckpt = torch.load(f'data/model/{cfg["name"]}/model_best.pth', map_location='cpu')
    network.load_state_dict(ckpt['network_state_dict'])
    network = network.eval().cuda()
    print(f'successfully load {cfg["name"]} step {ckpt["step"]}!')
    verts, tris = network._mesh
    n = flags.size * flags.ssaa
    t0 = time.time()
    vt, ft = TX.uv_atlas(verts, tris, n, n, 2 * flags.ssaa)
    print(f'unwrapped {tris.shape[0]} triangles into {vt.shape[0]} uv vertices in {time.time() - t0:.2f} s')
    images = TX.bake_textures(network, verts, tris, vt, ft, (flags.size, flags.size), flags.ssaa)
    TX.write_textured_obj(flags.out, verts, tris, vt, ft, images)
    print(f'{flags.out}: feat0_0.png, feat1_0.png, feat2_0.png, mesh_0.obj, mesh_0.mtl')
    return flags.out


if __name__ == '__main__':
    main()
