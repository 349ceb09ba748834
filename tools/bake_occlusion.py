"""Bake an ambient-occlusion map onto the atlas of a textured OBJ on the GPU (nero_b200/occlusion.py).

    python tools/bake_occlusion.py --obj n2m/mesh_0.obj [--detail data/meshes/bell-2048.ply] [--size N] [--ssaa 2] \\
        [--rays 256] [--distance 0.25] [--cage-distance 0.02] [--seed 0] [--out n2m/occlusion_0.png]

The OBJ is the textured mesh of tools/extract_materials_texture_map.py.  Without --detail the rays start from the OBJ's own
surface and the OBJ occludes them; with --detail (the fine mesh the OBJ was simplified from, a PLY read with
material.read_ply) each texel first casts the normal bake's cage ray (--cage-distance, tools/bake_normal_map.py's
--distance) and the rays start from the fine surface it hits, occluded by the fine mesh.  --rays rays per texel count the
unoccluded share of the cosine-weighted hemisphere within --distance scene units.  --size defaults to the OBJ's albedo map
size, so every map of the OBJ shares one resolution; the atlas is rasterised at --ssaa x that.  The map is written to --out
(default occlusion_0.png next to the OBJ) as 8-bit RGB with R = G = B; the OBJ and its MTL are not changed.  Export it with
tools/export_gltf.py --occlusion ....
Prints the covered texels, the cage hits and misses (texels that store 255), the mean unoccluded fraction and the times of
the phases, the host BVH build among them.
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MAX_RAYS = 65536     # nero_b200.occlusion.MAX_RAYS, restated so that argument errors need no library


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--obj', type=str, required=True, help='textured OBJ (mesh_0.obj with its MTL and feat0/1/2 images)')
    ap.add_argument('--detail', type=str, default=None, help='fine mesh (PLY) to take the surface and the occluders from')
    ap.add_argument('--size', type=int, default=None, help='map size (default: the albedo map size)')
    ap.add_argument('--ssaa', type=int, choices=(1, 2), default=2)
    ap.add_argument('--rays', type=int, default=256, help=f'rays per texel, 1 to {MAX_RAYS} (default 256)')
    ap.add_argument('--distance', type=float, default=0.25, help='occlusion distance in scene units (default 0.25)')
    ap.add_argument('--cage-distance', type=float, default=None, help='cage distance of --detail in scene units (default 0.02)')
    ap.add_argument('--seed', type=int, default=0)
    ap.add_argument('--out', type=str, default=None, help='output PNG (default: occlusion_0.png next to the OBJ)')
    flags = ap.parse_args(argv)
    if flags.size is not None and flags.size < 1:
        ap.error(f'--size {flags.size}: expected a positive size')
    if not 1 <= flags.rays <= MAX_RAYS:
        ap.error(f'--rays {flags.rays}: expected 1 to {MAX_RAYS}')
    if not (flags.distance > 0 and flags.distance < float('inf')):
        ap.error(f'--distance {flags.distance}: expected a positive distance')
    if flags.cage_distance is not None and not (flags.cage_distance > 0 and flags.cage_distance < float('inf')):
        ap.error(f'--cage-distance {flags.cage_distance}: expected a positive distance')
    if flags.cage_distance is not None and flags.detail is None:
        ap.error('--cage-distance needs --detail')
    if not 0 <= flags.seed < 2 ** 32:
        ap.error(f'--seed {flags.seed}: expected 0 to 2^32 - 1')
    if not os.path.isfile(flags.obj):
        ap.error(f'--obj {flags.obj}: no such file')
    if flags.detail is not None and not os.path.isfile(flags.detail):
        ap.error(f'--detail {flags.detail}: no such file')
    return flags


def main(argv=None):
    flags = parse(argv)
    import numpy as np
    from nero_b200 import normalmap as NM
    from nero_b200 import occlusion as OC
    from nero_b200.material import read_ply
    from nero_b200.relight import load_textured_obj
    t0 = time.perf_counter()
    verts, tris, vt_file, ft, maps = load_textured_obj(flags.obj)
    dverts, dtris = read_ply(flags.detail) if flags.detail else (None, None)
    size = maps['albedo'].shape[:2] if flags.size is None else (flags.size, flags.size)
    vt = np.stack([vt_file[:, 0], np.float32(1) - vt_file[:, 1]], -1)    # the OBJ stores 1 - v of the atlas
    t1 = time.perf_counter()
    prof = {}
    img, stats = OC.bake(verts, tris, vt, ft, size, dverts, dtris, flags.ssaa, flags.rays, flags.distance, flags.seed,
                         NM.DISTANCE if flags.cage_distance is None else flags.cage_distance, profile=prof)
    t2 = time.perf_counter()
    out = flags.out or os.path.join(os.path.dirname(os.path.abspath(flags.obj)), OC.FILE_NAME.format(cas=0))
    OC.write_occlusion_map(out, img)
    t3 = time.perf_counter()
    n = stats['covered']
    src = f'{dtris.shape[0]} detail triangles' if flags.detail else 'the mesh itself'
    print(f'bake_occlusion: {tris.shape[0]} triangles, occluders {src}, {img.shape[1]}x{img.shape[0]} map at ssaa {flags.ssaa}, '
          f'{flags.rays} rays within {flags.distance}: {n} covered texels, {stats["hits"]} hits, {stats["misses"]} misses '
          f'({stats["misses"] / n:.4%}), mean occlusion {1 - stats["mean"]:.4f} (unoccluded {stats["mean"]:.4f})')
    print('bake_occlusion: ' + ', '.join(f'{k} {v:.1f} ms' for k, v in prof.items()) +
          f'; read {t1 - t0:.2f} s, bake {t2 - t1:.2f} s, write {t3 - t2:.2f} s -> {out}')
    return out, stats


if __name__ == '__main__':
    main()
