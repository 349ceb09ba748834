"""Ambient occlusion baked onto the UV atlas on the GPU (k_occlusion.cu, include/nero_occlusion.h), for the glTF export's
occlusion texture (nero_b200/gltf.py, tools/export_gltf.py --occlusion).

tools/relight.py is a path tracer and finds occlusion by itself; a glTF viewer lights the object with image-based lighting
and has no visibility term, so it darkens what the environment cannot reach only through the material's occlusionTexture.
NeRO objects are glossy, so this matters for the specular light as much as for the diffuse light: the Khronos sample viewer
applies the texture to both.

Convention
----------
  * Stored value: cosine-weighted visibility within a distance.  N rays over the cosine-weighted hemisphere of the point's
    flat outward normal n_g (-cross(e1, e2) normalised: meshes are wound with cross(e1, e2) pointing into the solid); a ray
    is unoccluded if it hits no occluder triangle with t in (0, distance).  The value is the unoccluded count c of N.  The
    hemisphere is the flat normal's, not the interpolated one's, so every direction leaves the face's own half-space and a
    convex mesh is exactly unoccluded.
  * Sampler: a Hammersley set rotated per point (Cranley-Patterson) by two rl_uniform numbers of (seed, key), key = the
    texel's row-major index in the (ssaa-size) raster, so the result depends neither on compaction nor on launch shape.
    Rays start kRelightEps (1e-4) along n_g.  include/nero_occlusion.h states every formula.
  * Byte: k = (510 c + N) div (2N), round-half-up of 255 c / N, linear (no sRGB transfer); uncovered texels outside the seam
    band are 0, as in the material maps.  The file is occlusion_0.png next to the OBJ: 8-bit RGB with R = G = B, row 0 the
    top row (relight.write_png), the layout of the other maps.  glTF reads occlusion from the red channel.
  * Sources of the point: self (the low mesh's texel point and the owner triangle's flat normal, occluders the low mesh), or
    a detail mesh (the normal bake's cage ray from the texel, normalmap.py; the point is the hit on the detail mesh, n_g the
    hit triangle's flat normal and the occluders the detail mesh; a cage miss stores 255).

Defaults: distance 0.25 scene units (a quarter of the unit sphere's radius the objects lie in) and 256 rays are choices, not
measurements: the distance sets how large a cavity darkens, and 256 rays give bytes within about 255 / (2 sqrt(256)) = 8 of
the converged value at 50 % visibility.
"""
import os

import numpy as np

from .normalmap import DISTANCE as CAGE_DISTANCE, _size

DISTANCE = 0.25          # occlusion distance in scene units
RAYS = 256
MAX_RAYS = 65536
FILE_NAME = 'occlusion_{cas}.png'


def encode(counts, rays):
    """Unoccluded counts c of N rays -> uint8 bytes (510 c + N) div (2N), in integers."""
    c = np.asarray(counts, np.int64)
    return ((510 * c + rays) // (2 * rays)).astype(np.uint8)


def _check(rays, distance, seed):
    if not isinstance(rays, (int, np.integer)) or not 1 <= rays <= MAX_RAYS:
        raise ValueError(f'rays {rays}: expected an integer in [1, {MAX_RAYS}]')
    if not (np.isfinite(distance) and distance > 0):
        raise ValueError(f'distance {distance}: expected a positive finite number')
    if not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 32:
        raise ValueError(f'seed {seed}: expected an integer in [0, 2^32)')


def _bvh_cuda(verts, tris):
    from . import ops
    return ops.bvh_cuda(verts, tris, 'the occluder mesh')[:2]


def points_cuda(points, normals, occluder_verts, occluder_tris, rays=RAYS, distance=DISTANCE, seed=0, keys=None, bvh=None):
    """The counting kernel on arbitrary rows -> CUDA int32 [n] unoccluded counts of `rays`.  points / normals [n,3] (unit
    normals; a zero normal counts every ray unoccluded), keys [n] uint32 hash keys (default: the row index), as numpy arrays
    or tensors.  bvh: (nodes, tris) CUDA tensors of the occluder mesh to reuse instead of building it."""
    import torch
    from . import ops
    _check(rays, distance, seed)
    dev = torch.device('cuda')
    f32 = lambda a: torch.as_tensor(np.ascontiguousarray(a, np.float32) if isinstance(a, np.ndarray) else a).to(dev, torch.float32).contiguous()
    p, nrm = f32(points), f32(normals)
    if p.ndim != 2 or p.shape[1] != 3 or nrm.shape != p.shape:
        raise ValueError(f'points and normals must both be [n,3], got {tuple(p.shape)} and {tuple(nrm.shape)}')
    n = p.shape[0]
    k = None
    if keys is not None:
        k = torch.as_tensor(np.ascontiguousarray(keys, np.int64) if isinstance(keys, np.ndarray) else keys).to(dev)
        if k.shape != (n,):
            raise ValueError(f'keys must be [{n}], got {tuple(k.shape)}')
        if k.dtype != torch.int32:       # the kernel reads uint32: store the same bits in int32
            k = k.to(torch.int64)
            if bool((k < 0).any()) or bool((k >= 2 ** 32).any()):
                raise ValueError('keys must lie in [0, 2^32)')
            k = torch.where(k >= 2 ** 31, k - 2 ** 32, k).to(torch.int32)
        k = k.contiguous()
    nodes, btri = bvh if bvh is not None else _bvh_cuda(occluder_verts, occluder_tris)
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    ops.K('nero_occlusion_points', p, nrm, k, n, nodes, btri, int(rays), float(distance), int(seed), counts)
    return counts


def points(points, normals, occluder_verts, occluder_tris, rays=RAYS, distance=DISTANCE, seed=0, keys=None):
    """points_cuda as a numpy int32 [n] array."""
    return points_cuda(points, normals, occluder_verts, occluder_tris, rays, distance, seed, keys).cpu().numpy()


def bake_cuda(verts, tris, vt, ft, size, detail_verts=None, detail_tris=None, ssaa=2, rays=RAYS, distance=DISTANCE, seed=0,
              cage_distance=CAGE_DISTANCE, profile=None):
    """The bake before inpainting -> dict of CUDA tensors: raster (texmap.raster's dict at (ssaa h0) x (ssaa w0)), img
    [h,w,5] uint8, and per covered texel in row-major order counts [n] int32, hit [n] uint8 (1 for the self source), point /
    normal [n,3] float32 (where the rays start from, before the kRelightEps offset), key [n] (the row-major texel index),
    surface / cage [n,3] float32 (the texel's point on the low mesh and the cage direction, zero for the self source).  vt,
    ft: the atlas with v = 0 at the first texel row (texmap.uv_atlas's layout, not the OBJ's 1 - v).  Without detail_verts the
    source is the low mesh itself.  profile (a dict) gets host-clock milliseconds of the phases normals (detail only) / bvh /
    raster / texels / count / bytes, each ended by a device synchronise.  `args` and `texel_args` hold the arguments of the
    nero_occlusion_points launch (the counting kernel) and of the nero_occlusion_texels launch."""
    import time
    import torch
    from . import ops
    from .normalmap import vertex_normals_cuda
    from .texmap import raster
    h0, w0 = _size(size, ssaa)
    _check(rays, distance, seed)
    detail = detail_verts is not None or detail_tris is not None
    if detail and (detail_verts is None or detail_tris is None):
        raise ValueError('a detail mesh needs both detail_verts and detail_tris')
    if detail and not (np.isfinite(cage_distance) and cage_distance > 0):
        raise ValueError(f'cage distance {cage_distance}: expected a positive finite number')
    h, w = h0 * ssaa, w0 * ssaa
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    if np.asarray(ft).shape != tris.shape:
        raise ValueError(f'ft has shape {np.asarray(ft).shape} for tris of shape {tris.shape}')
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
    low_n = None
    if detail:
        low_n = vertex_normals_cuda(verts, tris)
        lap('normals')
        nodes, btri = _bvh_cuda(detail_verts, detail_tris)
    else:
        nodes, btri = _bvh_cuda(verts, tris)
    lap('bvh')
    r = raster(vt, ft, verts, tris, w, h)
    lap('raster')
    n = r['texel'].shape[0]
    point, normal, surface, cage = (torch.empty(n, 3, dtype=torch.float32, device=dev) for _ in range(4))
    key = torch.empty(n, dtype=torch.int32, device=dev)
    hit = torch.empty(n, dtype=torch.uint8, device=dev)
    texel_args = (r['owner'], w, h, r['texel'], n, up(np.asarray(vt, np.float32)), up(np.asarray(ft, np.int32)), up(verts), up(tris), low_n,
                  nodes if detail else None, btri if detail else None, float(cage_distance), point, normal, key, hit, surface, cage)
    ops.K('nero_occlusion_texels', *texel_args)
    lap('texels')
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    args = (point, normal, key, n, nodes, btri, int(rays), float(distance), int(seed), counts)
    ops.K('nero_occlusion_points', *args)
    lap('count')
    img = torch.empty(h, w, 5, dtype=torch.uint8, device=dev)
    ops.K('nero_occlusion_bytes', r['texel'], n, counts, int(rays), w, h, img)
    lap('bytes')
    return dict(raster=r, img=img, counts=counts, hit=hit, point=point, normal=normal, key=key, surface=surface, cage=cage,
                low_normals=low_n, args=args, texel_args=texel_args)


def bake(verts, tris, vt, ft, size, detail_verts=None, detail_tris=None, ssaa=2, rays=RAYS, distance=DISTANCE, seed=0,
         cage_distance=CAGE_DISTANCE, profile=None):
    """Bake ambient occlusion onto the atlas (vt, ft) of the mesh (verts, tris) -> (img uint8 [h0,w0,3] numpy with R = G = B,
    row 0 at v = 0 of the atlas, stats {covered, hits, misses, mean}: covered texels of the (ssaa-size) raster, cage hits and
    misses (every texel hits for the self source), mean unoccluded fraction c / N over the covered texels).  size = h0 = w0 or
    (h0, w0); the atlas is rasterised at ssaa x that, inpainted and, at ssaa 2, down-sampled as the normal bake is.  vt is
    texmap.uv_atlas's layout (for an OBJ's vt, pass 1 - v).  profile as bake_cuda's, plus inpaint / downsample."""
    import time
    import torch
    from .texmap import downsample, inpaint
    b = bake_cuda(verts, tris, vt, ft, size, detail_verts, detail_tris, ssaa, rays, distance, seed, cage_distance, profile)
    n = int(b['hit'].shape[0])
    if n == 0:
        raise ValueError('no texel of the atlas is covered by a triangle (an empty mesh or atlas)')
    hits = int(b['hit'].sum())
    mean = float(b['counts'].sum().item()) / (n * rays)
    t0 = time.perf_counter()
    img, _ = inpaint(b['img'], b['raster']['owner'])
    if profile is not None:
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        profile['inpaint'] = profile.get('inpaint', 0.0) + (t1 - t0) * 1e3
        t0 = t1
    if ssaa == 2:
        img = downsample(img)
        if profile is not None:
            torch.cuda.synchronize()
            profile['downsample'] = profile.get('downsample', 0.0) + (time.perf_counter() - t0) * 1e3
    return img[..., :3].cpu().numpy(), {'covered': n, 'hits': hits, 'misses': n - hits, 'mean': mean}


def write_occlusion_map(path, img):
    """Write an occlusion map, uint8 [h,w] or [h,w,3] with R = G = B, as an 8-bit RGB PNG with R = G = B
    (relight.write_png)."""
    from .relight import write_png
    img = np.asarray(img, np.uint8)
    if img.ndim == 3 and img.shape[2] == 3:
        img = img[..., 0]
    if img.ndim != 2:
        raise ValueError(f'an occlusion map is [h,w] or [h,w,3], got {img.shape}')
    write_png(path, np.repeat(img[..., None], 3, axis=2))


def read_occlusion_map(path):
    """An 8-bit RGB(A) occlusion image -> its red channel, uint8 [H,W], row 0 the top row of the file.  A missing file, an
    unreadable one or one that is not 8-bit colour raises ValueError naming it."""
    import cv2
    if not os.path.isfile(path):
        raise ValueError(f'{path}: occlusion map file is missing')
    img = cv2.imread(path, cv2.IMREAD_UNCHANGED)
    if img is None:
        raise ValueError(f'{path}: not an image OpenCV can read')
    if img.dtype != np.uint8 or img.ndim != 3 or img.shape[2] not in (3, 4):
        raise ValueError(f'{path}: an occlusion map must be an 8-bit RGB image, got {img.dtype} with shape {img.shape}')
    return np.ascontiguousarray(img[..., 2])
