"""Bake an object-space normal map of a fine mesh onto the atlas of a textured OBJ on the GPU (nero_b200/normalmap.py).

    python tools/bake_normal_map.py --obj n2m/mesh_0.obj --detail data/meshes/bell-2048.ply [--size N] [--ssaa 2] \\
        [--distance 0.02] [--out n2m/normal_0.png]

The OBJ is the textured mesh of tools/extract_materials_texture_map.py (typically of a mesh simplified with
tools/simplify_mesh.py or extract_mesh.py --faces); --detail is the fine mesh it came from, a PLY read with
material.read_ply.  --size defaults to the OBJ's albedo map size, so every map of the OBJ shares one resolution; the atlas
is rasterised at --ssaa x that.  The map is written to --out (default normal_0.png next to the OBJ); the OBJ and its MTL
are not changed.  Relight with it through tools/relight.py --obj ... --normal-map ....
Prints the covered texels, the rays that found the detail mesh and the misses (texels that keep the low mesh's own
interpolated normal), and the times of the phases.
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
    ap.add_argument('--detail', type=str, required=True, help='fine mesh (PLY)')
    ap.add_argument('--size', type=int, default=None, help='map size (default: the albedo map size)')
    ap.add_argument('--ssaa', type=int, choices=(1, 2), default=2)
    ap.add_argument('--distance', type=float, default=None, help='cage distance in scene units (default 0.02)')
    ap.add_argument('--out', type=str, default=None, help='output PNG (default: normal_0.png next to the OBJ)')
    flags = ap.parse_args(argv)
    if flags.size is not None and flags.size < 1:
        ap.error(f'--size {flags.size}: expected a positive size')
    if flags.distance is not None and not flags.distance > 0:
        ap.error(f'--distance {flags.distance}: expected a positive distance')
    return flags


def main(argv=None):
    flags = parse(argv)
    import numpy as np
    from nero_b200 import normalmap as NM
    from nero_b200.material import read_ply
    from nero_b200.relight import load_textured_obj
    t0 = time.perf_counter()
    verts, tris, vt_file, ft, maps = load_textured_obj(flags.obj)
    dverts, dtris = read_ply(flags.detail)
    size = maps['albedo'].shape[:2] if flags.size is None else (flags.size, flags.size)
    vt = np.stack([vt_file[:, 0], np.float32(1) - vt_file[:, 1]], -1)    # the OBJ stores 1 - v of the atlas
    t1 = time.perf_counter()
    img, stats = NM.bake(verts, tris, vt, ft, dverts, dtris, size, flags.ssaa, NM.DISTANCE if flags.distance is None else flags.distance)
    t2 = time.perf_counter()
    out = flags.out or os.path.join(os.path.dirname(os.path.abspath(flags.obj)), NM.FILE_NAME.format(cas=0))
    NM.write_normal_map(out, img)
    t3 = time.perf_counter()
    n = stats['covered']
    print(f'bake_normal_map: {tris.shape[0]} low / {dtris.shape[0]} detail triangles, {img.shape[1]}x{img.shape[0]} map at ssaa '
          f'{flags.ssaa}: {n} covered texels, {stats["hits"]} hits, {stats["misses"]} misses ({stats["misses"] / n:.4%})')
    print(f'bake_normal_map: read {t1 - t0:.2f} s, bake {t2 - t1:.2f} s (host BVH build included), write {t3 - t2:.2f} s -> {out}')
    return out, stats


if __name__ == '__main__':
    main()
