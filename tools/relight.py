"""Relight a stage-II result under an HDR environment map on the GPU (the reference's relight.py, without Blender).

    python tools/relight.py --mesh data/meshes/bell_shape-300000.ply --material data/materials/bell_material-100000 \
        --hdr data/hdr/neon_photostudio_4k.exr --name bell [--trans]
    python tools/relight.py --obj n2m_test/mesh_0.obj --hdr data/hdr/neon_photostudio_4k.exr --name bell [--trans]

The materials are per-vertex (--mesh with --material, as tools/extract_materials.py writes them) or UV textures (--obj, the
textured OBJ of tools/extract_materials_texture_map.py with its MTL and feat{0,1,2} images); exactly one form is accepted.

Renders frames k = 0 .. num-1 of the reference's turntable (blender_backend/relight_backend.py) to data/relight/<name>/<k>.png
(RGBA8, transparent background); frames that already exist are skipped.  The scene -- geometry, materials, BRDF, cameras,
environment mapping and output encoding -- is stated in nero_b200/relight.py.  Paths are relative to the working directory.

--denoise filters each frame with the feature-guided a-trous filter of nero_b200/denoise.py before it is written; frames,
names and the PNG format are unchanged, and so is the alpha channel.  The intended use is `--samples 64 --denoise` in place of
the default 1024 samples:

    python tools/relight.py --mesh ... --material ... --hdr ... --name bell --samples 64 --denoise
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    parser = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    parser.add_argument('--mesh', type=str, default=None)
    parser.add_argument('--material', type=str, default=None, help='directory with metallic.npy, roughness.npy, albedo.npy')
    parser.add_argument('--obj', type=str, default=None, help='textured OBJ (with its MTL and feat0/1/2 texture images)')
    parser.add_argument('--hdr', type=str, required=True, help='environment map (.hdr or .exr)')
    parser.add_argument('--name', type=str, required=True)
    parser.add_argument('--trans', action='store_true', default=False, help='rotate the mesh by +90 degrees about x')
    parser.add_argument('--num', type=int, default=360)
    parser.add_argument('--width', type=int, default=800)
    parser.add_argument('--height', type=int, default=800)
    parser.add_argument('--samples', type=int, default=1024)
    parser.add_argument('--cam_dist', type=float, default=3.0)
    parser.add_argument('--azimuth', type=float, default=0.0)
    parser.add_argument('--elevation', type=float, default=45.0)
    parser.add_argument('--bounces', type=int, default=4)
    parser.add_argument('--geometry', choices=('schlick', 'ggx_smith'), default='schlick')
    parser.add_argument('--seed', type=int, default=0)
    parser.add_argument('--denoise', action='store_true', default=False, help='denoise each frame (use with --samples 64)')
    flags = parser.parse_args(argv)
    if flags.obj is not None:
        if flags.mesh is not None or flags.material is not None:
            parser.error('--obj cannot be combined with --mesh / --material')
    elif flags.mesh is None or flags.material is None:
        parser.error('give --mesh with --material, or --obj')
    return flags


def main(argv=None):
    flags = parse(argv)

    import numpy as np
    import torch
    from nero_b200.material import read_ply
    from nero_b200.relight import (MESH_TRANS, Relighter, UVMaterials, blender_default_K, load_env_map, load_materials,
                                   load_textured_obj, relight_poses, to_rgba8, write_png_rgba)

    if flags.obj is not None:
        verts, tris, vt, ft, maps = load_textured_obj(flags.obj)
        materials = UVMaterials(vt, ft, maps['albedo'], maps['metallic'], maps['roughness'])
    else:
        verts, tris = read_ply(flags.mesh)
        materials = load_materials(flags.material)
    if flags.trans:
        verts = (verts.astype(np.float64) @ MESH_TRANS.T).astype(np.float32)
    relighter = Relighter(verts, tris, materials, load_env_map(flags.hdr), flags.geometry)
    K = blender_default_K(flags.height, flags.width)
    poses = relight_poses(flags.num, flags.azimuth, flags.elevation, flags.cam_dist)
    out_dir = os.path.join('data', 'relight', flags.name)
    os.makedirs(out_dir, exist_ok=True)
    for k in range(flags.num):
        path = os.path.join(out_dir, f'{k}.png')
        if os.path.exists(path):
            continue
        img = relighter.render(poses[k], K, flags.height, flags.width, flags.samples, flags.bounces, flags.seed,
                               denoise=flags.denoise)
        torch.cuda.synchronize()
        write_png_rgba(path, to_rgba8(img.cpu().numpy()))
        print(path)
    return out_dir


if __name__ == '__main__':
    main()
