"""Export a textured OBJ (and its baked normal and occlusion maps) as one self-contained glTF 2.0 binary on the GPU
(nero_b200/gltf.py).

    python tools/export_gltf.py --obj n2m/mesh_0.obj [--normal-map n2m/normal_0.png] [--occlusion n2m/occlusion_0.png] \
        [--out n2m/mesh_0.glb] [--trans]

The OBJ is the textured mesh of tools/extract_materials_texture_map.py (the reference's JPEG export is read too); the normal
map is the object-space map of tools/bake_normal_map.py, converted to tangent space against the tangents the file carries.
The occlusion map is the ambient-occlusion map of tools/bake_occlusion.py, of the material maps' size: its byte replaces the
constant 255 in the red channel of the metallic-roughness texture, which the material then also names as its occlusionTexture.
--trans: the object is stored the way tools/relight.py --trans takes it (y-up), so the node is not rotated; otherwise the node
turns the z-up object to glTF's y-up.  The file is written to --out (default mesh_0.glb next to the OBJ).
Prints the vertex counts before and after welding, the covered texels of the normal map, the file size and the times of the
phases.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--obj', type=str, required=True, help='textured OBJ (mesh_0.obj with its MTL and feat0/1/2 images)')
    ap.add_argument('--normal-map', type=str, default=None, help='object-space normal map (normal_0.png of bake_normal_map.py)')
    ap.add_argument('--occlusion', type=str, default=None, help='ambient-occlusion map (occlusion_0.png of bake_occlusion.py)')
    ap.add_argument('--out', type=str, default=None, help='output .glb (default: mesh_0.glb next to the OBJ)')
    ap.add_argument('--trans', action='store_true', help='the object is y-up already (tools/relight.py --trans): no node rotation')
    flags = ap.parse_args(argv)
    if not os.path.isfile(flags.obj):
        ap.error(f'--obj {flags.obj}: no such file')
    if flags.normal_map is not None and not os.path.isfile(flags.normal_map):
        ap.error(f'--normal-map {flags.normal_map}: no such file')
    if flags.occlusion is not None and not os.path.isfile(flags.occlusion):
        ap.error(f'--occlusion {flags.occlusion}: no such file')
    return flags


def main(argv=None):
    flags = parse(argv)
    from nero_b200 import gltf
    t0 = time.perf_counter()
    prof, stats = {}, {}
    try:
        data = gltf.export(flags.obj, flags.normal_map, flags.trans, profile=prof, stats=stats, occlusion_path=flags.occlusion)
    except ValueError as e:
        raise SystemExit(f'export_gltf: {e}')
    out = flags.out or os.path.join(os.path.dirname(os.path.abspath(flags.obj)), gltf.FILE_NAME.format(cas=0))
    t1 = time.perf_counter()
    with open(out, 'wb') as f:
        f.write(data)
    t2 = time.perf_counter()
    cov = f', {stats["covered"]} covered texels of the normal map' if flags.normal_map else ' (no normal map)'
    cov += ', occlusion in the metallic-roughness red channel' if flags.occlusion else ''
    print(f'export_gltf: {stats["triangles"]} triangles, {stats["positions"]} positions -> {stats["welded"]} welded vertices{cov}')
    print('export_gltf: ' + ', '.join(f'{k} {v:.1f} ms' for k, v in prof.items()) +
          f'; total {(t1 - t0) * 1e3:.1f} ms, write {(t2 - t1) * 1e3:.1f} ms -> {out} ({len(data)} bytes)')
    return out, stats


if __name__ == '__main__':
    main()
