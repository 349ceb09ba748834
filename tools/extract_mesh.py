"""Stage-I checkpoint -> triangle mesh for stage II, on the GPU (the reference's extract_mesh.py).

    python tools/extract_mesh.py --cfg configs/shape/syn/bell.yaml [--resolution 512] [--sparse [--brick 8] [--lipschitz 2.0]]
                                 [--faces N]

Loads data/model/<name>/model.pth ({'step', 'network_state_dict', ...}), samples the SDF on a resolution^3 grid over [-1,1]^3
(1.0 outside the unit sphere), runs marching cubes at level 0 and writes data/meshes/<name>-<step>.ply, the path
NeROMaterialRenderer's `mesh` option and predict_materials read.  Paths are relative to the working directory.

With --sparse the SDF is sampled only in bricks of brick^3 cubes around the surface (NeROShapeRenderer.extract_mesh_sparse):
the same mesh, at a cost that follows the surface, which is what makes --resolution 1024 and 2048 possible on one card.  A
closed piece of surface smaller than a brick where the SDF is steeper than --lipschitz can be missed; raise --lipschitz or
lower --brick then.

With --faces N the mesh is reduced to about N triangles by quadric edge collapse (nero_b200/simplify.py) before it is
written, to the same path: `--sparse --resolution 2048 --faces 888056` gives a stage-II-sized mesh that keeps the detail
of the fine grid where the surface curves.
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
    parser.add_argument('--sparse', action='store_true', help='sample the SDF in a narrow band around the surface only')
    parser.add_argument('--brick', type=int, default=8, choices=(4, 8, 16), help='cubes per brick edge (with --sparse)')
    parser.add_argument('--lipschitz', type=float, default=2.0, help='bound on the SDF slope used for seeding (with --sparse)')
    parser.add_argument('--faces', type=int, default=None, help='simplify the mesh to about this many triangles (>= 4)')
    flags = parser.parse_args(argv)
    if flags.faces is not None and flags.faces < 4:
        raise SystemExit(f'extract_mesh: --faces must be >= 4, got {flags.faces}')

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

    stats = None
    if flags.sparse:
        vertices, triangles, stats = network.extract_mesh_sparse(resolution=flags.resolution, threshold=0.0, brick=flags.brick,
                                                                 lipschitz=flags.lipschitz, return_stats=True)
    else:
        vertices, triangles = network.extract_mesh(resolution=flags.resolution, threshold=0.0)
    simplified = None
    if flags.faces is not None:
        from nero_b200.simplify import simplify, stats_line
        n_in = triangles.shape[0]
        vertices, triangles, simplified = simplify(vertices, triangles, flags.faces)
        print(f'simplified {n_in} -> {triangles.shape[0]} triangles')
    os.makedirs('data/meshes', exist_ok=True)
    path = os.path.join('data', 'meshes', f'{cfg["name"]}-{step}.ply')
    write_ply(path, vertices, triangles)
    print(f'{path}: {vertices.shape[0]} vertices, {triangles.shape[0]} triangles')
    if stats is not None:
        print('sparse: ' + ', '.join(f'{k} {v}' for k, v in stats.items()))
    if simplified is not None:
        print(stats_line(simplified))
    return path


if __name__ == '__main__':
    main()
