"""Normal maps baked from a fine mesh onto the UV atlas of its simplification, on the GPU (k_normalmap.cu,
include/nero_normalmap.h), and read back for relighting (relight.UVMaterials(normal=...)).

Quadric simplification (nero_b200/simplify.py) keeps the shape of a 2048^3 extraction at a size the unwrapper and the
relighter handle, but the flat faces of the simplified mesh shade faceted.  A normal map puts the fine mesh's shading back:
each texel of the low mesh's atlas stores the normal of the fine mesh where a short ray from the texel's surface point
meets it ("selected to active" in DCC tools).

Convention
----------
  * Object-space maps: a texel holds the outward unit normal in the OBJ's own coordinates, the coordinates the relighter
    renders in (tools/relight.py --trans rotates the map with the mesh).  Object space, because the relighter shades flat
    faces and an object-space map leaves no tangent-basis convention for the bake and the renderer to disagree on.
    The bake writes no tangent-space map; nero_b200/gltf.py (tools/export_gltf.py) converts this map to tangent space
    against the tangents it writes into a glTF 2.0 file.
  * Outward normals.  Marching-cubes meshes are wound with cross(e1, e2) pointing into the solid, so outward is
    -cross(e1, e2); simplified meshes keep that winding.
  * Encoding per channel: k = floor((n 0.5 + 0.5) 255 + 0.5) clamped to [0, 255]; decoding is linear, 2k/255 - 1, with no
    sRGB transfer (so relight._read_map, which applies one, is not used for this file).  The file is normal_0.png next to
    the textured OBJ: 8-bit RGB, row 0 the top row, written by relight.write_png.  Uncovered texels outside the seam band are
    0, as in the material maps.
  * The MTL is not changed: other readers take `norm` / `bump` to mean a tangent-space map.  tools/relight.py takes the map
    with --normal-map.

Bake
----
  1. Raster: the low mesh's atlas at (ssaa size)^2 with texmap.raster (texel centres, snapped uv, top-left rule).
  2. Vertex normals of both meshes: per vertex, the sum of -cross(e1, e2) of its triangles in ascending triangle order (the
     CSR of simplify._vertex_triangles) with fp32 _rn adds, normalised; a zero sum gives (0, 0, 0).  No scheduling enters.
  3. One thread per covered texel: the texel's barycentrics b and point p exactly as texmap.raster computes xyz; the cage
     direction c = normalize(sum b_i n_i) from the low mesh's vertex normals; one ray from p + distance c along -c; the
     closest hit with t in (0, 2 distance) on the detail mesh's BVH.  Hit: the detail vertex normals interpolated with the
     hit's barycentrics, normalised.  Miss: c.  The bytes go to channels 0-2 of a [w h, 5] image (3-4 zero), which then
     takes the texture export's seam inpainting and, at ssaa 2, its 2x down-sampling, unchanged.
  distance defaults to 0.02 scene units (objects lie in the unit sphere): a cage that reaches the fine surface across the
  simplification error without jumping to a neighbouring sheet.
"""
import os

import numpy as np

DISTANCE = 0.02          # cage distance in scene units
FILE_NAME = 'normal_{cas}.png'


def encode(n):
    """Unit normals [..., 3] -> uint8 bytes: floor((n 0.5 + 0.5) 255 + 0.5) clamped, each fp32 operation rounded (the
    kernel's arithmetic)."""
    n = np.asarray(n, np.float32)
    k = np.floor((n * np.float32(0.5) + np.float32(0.5)) * np.float32(255) + np.float32(0.5))
    return np.clip(k, 0, 255).astype(np.uint8)


def decode(k):
    """uint8 bytes -> float32 2k/255 - 1 (linear; not renormalised)."""
    return (2.0 * np.asarray(k, np.float64) / 255.0 - 1.0).astype(np.float32)


def vertex_normals_cuda(verts, tris):
    """Area-weighted outward vertex normals (module docstring, step 2) -> CUDA float32 [V,3].  verts [V,3], tris [T,3] as
    numpy arrays or tensors."""
    import torch
    from . import ops
    from .simplify import _vertex_triangles
    dev = torch.device('cuda')
    v = torch.as_tensor(np.ascontiguousarray(verts, np.float32) if isinstance(verts, np.ndarray) else verts).to(dev, torch.float32).contiguous()
    t = torch.as_tensor(np.ascontiguousarray(tris, np.int32) if isinstance(tris, np.ndarray) else tris).to(dev, torch.int32).contiguous()
    if v.ndim != 2 or v.shape[1] != 3 or t.ndim != 2 or t.shape[1] != 3:
        raise ValueError(f'vertex_normals needs verts [V,3] and tris [T,3], got {tuple(v.shape)} and {tuple(t.shape)}')
    V, T = v.shape[0], t.shape[0]
    if T and (int(t.min()) < 0 or int(t.max()) >= V):
        raise ValueError(f'vertex_normals: triangle indices outside [0, {V})')
    ptr, tri = _vertex_triangles(t, V)
    out = torch.empty(V, 3, dtype=torch.float32, device=dev)
    ops.K('nero_normalmap_vertex_normals', v, V, t, T, ptr, tri, out)
    return out


def vertex_normals(verts, tris):
    """vertex_normals_cuda as a numpy float32 [V,3] array."""
    return vertex_normals_cuda(verts, tris).cpu().numpy()


def _size(size, ssaa):
    h0, w0 = (size, size) if np.isscalar(size) else tuple(int(x) for x in size)
    if ssaa not in (1, 2):
        raise ValueError(f'ssaa {ssaa}: expected 1 or 2')
    if h0 < 1 or w0 < 1:
        raise ValueError(f'map size {h0}x{w0}: expected positive')
    return h0, w0


def bake_cuda(verts, tris, vt, ft, detail_verts, detail_tris, size, ssaa=2, distance=DISTANCE, profile=None):
    """The bake before inpainting -> dict of CUDA tensors: raster (texmap.raster's dict at (ssaa h0) x (ssaa w0)), img
    [h,w,5] uint8, hit [n] uint8, point / cage / normal [n,3] float32 per covered texel in row-major order.  vt, ft: the
    atlas with v = 0 at the first texel row (texmap.uv_atlas's layout, not the OBJ's 1 - v).  profile (a dict) gets
    host-clock milliseconds of the phases normals / bvh / raster / bake, each ended by a device synchronise.  The dict also
    holds both meshes' vertex normals and `args`, the arguments of the nero_normalmap_bake launch."""
    import time
    import torch
    from . import ops
    from .texmap import raster
    h0, w0 = _size(size, ssaa)
    if not (np.isfinite(distance) and distance > 0):
        raise ValueError(f'distance {distance}: expected a positive finite number')
    h, w = h0 * ssaa, w0 * ssaa
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    dverts = np.ascontiguousarray(detail_verts, np.float32)
    dtris = np.ascontiguousarray(detail_tris, np.int32)
    if np.asarray(ft).shape != tris.shape:
        raise ValueError(f'ft has shape {np.asarray(ft).shape} for tris of shape {tris.shape}')
    if dtris.ndim != 2 or dtris.shape[1] != 3 or dtris.shape[0] < 1:
        raise ValueError(f'the detail mesh needs tris [T,3] with T >= 1, got {dtris.shape}')
    clock = [time.perf_counter()]

    def lap(phase):
        if profile is not None:
            torch.cuda.synchronize()
            now = time.perf_counter()
            if phase is not None:
                profile[phase] = profile.get(phase, 0.0) + (now - clock[0]) * 1e3
            clock[0] = now
    lap(None)
    dev = torch.device('cuda')
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    low_n = vertex_normals_cuda(verts, tris)
    det_n = vertex_normals_cuda(dverts, dtris)
    lap('normals')
    nodes, btri, ids = ops.bvh_build(dverts, dtris)
    nodes, btri, ids = up(nodes), up(btri), up(ids)
    lap('bvh')
    r = raster(vt, ft, verts, tris, w, h)
    lap('raster')
    n = r['texel'].shape[0]
    img = torch.empty(h, w, 5, dtype=torch.uint8, device=dev)
    hit = torch.empty(n, dtype=torch.uint8, device=dev)
    point, cage, normal = (torch.empty(n, 3, dtype=torch.float32, device=dev) for _ in range(3))
    args = (r['owner'], w, h, r['texel'], n, up(np.asarray(vt, np.float32)), up(np.asarray(ft, np.int32)), up(verts), up(tris), low_n,
            nodes, btri, ids, up(dtris), det_n, float(distance), img, hit, point, cage, normal)
    ops.K('nero_normalmap_bake', *args)
    lap('bake')
    return dict(raster=r, img=img, hit=hit, point=point, cage=cage, normal=normal, low_normals=low_n, detail_normals=det_n,
                args=args)


def bake(verts, tris, vt, ft, detail_verts, detail_tris, size, ssaa=2, distance=DISTANCE):
    """Bake the detail mesh's normals onto the atlas (vt, ft) of the low mesh (verts, tris) -> (img uint8 [h0,w0,3] numpy,
    row 0 at v = 0 of the atlas, stats {covered, hits, misses}).  size = h0 = w0 or (h0, w0); the atlas is rasterised at
    ssaa x that.  vt is texmap.uv_atlas's layout (for an OBJ's vt, pass 1 - v: the OBJ stores the flipped coordinate)."""
    from .texmap import downsample, inpaint
    b = bake_cuda(verts, tris, vt, ft, detail_verts, detail_tris, size, ssaa, distance)
    n = int(b['hit'].shape[0])
    if n == 0:
        raise ValueError('no texel of the atlas is covered by a triangle (an empty mesh or atlas)')
    hits = int(b['hit'].sum())
    img, _ = inpaint(b['img'], b['raster']['owner'])
    if ssaa == 2:
        img = downsample(img)
    return img[..., :3].cpu().numpy(), {'covered': n, 'hits': hits, 'misses': n - hits}


def write_normal_map(path, img):
    """Write uint8 [h,w,3] bytes as the 8-bit RGB PNG (relight.write_png)."""
    from .relight import write_png
    write_png(path, np.asarray(img, np.uint8))


def read_normal_map(path):
    """An 8-bit RGB(A) normal-map image -> float32 [H,W,3] 2k/255 - 1 per channel (linear, not renormalised), row 0 the top
    row of the file.  A missing file, an unreadable one or one that is not 8-bit colour raises ValueError naming it."""
    return decode(read_normal_map_bytes(path))


def read_normal_map_bytes(path):
    """read_normal_map's image as its uint8 RGB bytes [H,W,3], with the same checks."""
    import cv2
    if not os.path.isfile(path):
        raise ValueError(f'{path}: normal map file is missing')
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise ValueError(f'{path}: not an image OpenCV can read')
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] not in (3, 4):
        raise ValueError(f'{path}: a normal map must be an 8-bit RGB image, got {img.dtype} with shape {img.shape}')
    return np.ascontiguousarray(img[..., [2, 1, 0]])
