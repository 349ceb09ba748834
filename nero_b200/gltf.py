"""glTF 2.0 export of the textured mesh on the GPU (k_gltf.cu, include/nero_gltf.h): one self-contained .glb that web viewers
and game engines load, with the baked materials and, optionally, the normal map in tangent space.

NeRO's BRDF is glTF 2.0's metallic-roughness model: albedo (1-m)/pi + F D G / (4 NoV NoL), F0 = 0.04 (1-m) + m albedo, Schlick
F, a GGX D (math_relight.cuh:rl_brdf), with glTF's roughness = sqrt(alpha).  So the file carries a NeRO result without
changing its meaning.

Input: the directory of tools/extract_materials_texture_map.py (mesh_0.obj, mesh_0.mtl, feat{0,1,2}_0.png, or the
reference's JPEGs) as relight.load_textured_obj reads it, optionally the object-space normal map of
tools/bake_normal_map.py (normal_0.png, nero_b200/normalmap.py's convention) and optionally the ambient-occlusion map of
tools/bake_occlusion.py (occlusion_0.png, nero_b200/occlusion.py's convention).

The file:
  * One scene, one node, one mesh, one triangle primitive.  Attributes POSITION (float32 with min / max), NORMAL, TEXCOORD_0
    and, with a normal map only, TANGENT (VEC4, w = +-1); uint32 indices.
  * Vertices are the distinct (position, uv) pairs of the OBJ's corners (the weld of include/nero_gltf.h).  POSITION is the
    OBJ's vertex, NORMAL its outward area-weighted vertex normal (nero_normalmap_vertex_normals), TEXCOORD_0 = (u, 1 - v) of
    the file's vt (glTF's uv origin is the image's top-left corner, the OBJ's the bottom-left).
  * Winding: the meshes here are wound with cross(e1, e2) pointing into the solid; glTF's front faces are counter-clockwise
    seen from outside, so each face (a, b, c) is written (a, c, b).
  * Orientation: NeRO objects are z-up and glTF is y-up, so the node rotates by -90 degrees about x (quaternion
    [-sqrt(1/2), 0, 0, sqrt(1/2)]); with trans=True (objects that tools/relight.py --trans rotates +90 degrees about x to make
    them z-up) the node has no rotation.  The vertex data is the OBJ's, unrotated.
  * One material: baseColorTexture = feat0's bytes (both sRGB), metallicRoughnessTexture = (255, roughness, metallic) from
    feat1 / feat2 through the tables of include/nero_gltf.h (stored alpha -> sqrt, sRGB -> linear), factors 1; with a normal
    map, normalTexture = the map converted to tangent space against the file's own TANGENT and NORMAL, then seam-inpainted
    with texmap.inpaint.  With an occlusion map, the metallic-roughness texture's red channel is the map's byte instead of
    255 (glTF's "ORM" packing) and occlusionTexture = that same texture (index 1, strength 1 by default); G and B are
    unchanged.  Without one the file is byte for byte what it is without the option.  Images are PNGs (relight.png_bytes) in bufferViews; one sampler: LINEAR, LINEAR_MIPMAP_LINEAR,
    REPEAT.
  * GLB container: JSON chunk padded with spaces, BIN chunk with zeros, every bufferView 4-byte aligned.

Shading in other tools.  The tangent-space map is exact for readers that use the file's TANGENT, as the glTF 2.0
specification asks: the conversion solves the frame the glTF sample viewer interpolates per fragment, so its decode gives back
the object-space map up to 8-bit quantisation.  Tools that recompute MikkTSpace tangents themselves get slightly different
frames; those differences are unmeasured.  Without a normal map the file has no TANGENT and no normal texture, and viewers
shade with the smooth NORMAL, whereas tools/relight.py shades flat faces.
"""
import json
import math
import os
import struct
import time
import zlib

import numpy as np

FILE_NAME = 'mesh_{cas}.glb'
Z_UP_ROTATION = [-math.sqrt(0.5), 0.0, 0.0, math.sqrt(0.5)]   # -90 degrees about x: NeRO's z-up to glTF's y-up
WELD_THREADS = 256            # position vertices per block of nero_gltf_weld_count

# glTF 2.0 enumerations
_FLOAT, _UINT = 5126, 5125
_ARRAY_BUFFER, _ELEMENT_ARRAY_BUFFER = 34962, 34963
_LINEAR, _LINEAR_MIPMAP_LINEAR, _REPEAT = 9729, 9987, 10497
_TRIANGLES = 4
_GLB_MAGIC, _CHUNK_JSON, _CHUNK_BIN = 0x46546C67, 0x4E4F534A, 0x004E4942
_PNG_SIGNATURE = b'\x89PNG\r\n\x1a\n'
_ATTRIBUTES = (('POSITION', 'positions', 3), ('NORMAL', 'normals', 3), ('TEXCOORD_0', 'texcoords', 2), ('TANGENT', 'tangents', 4))
_IMAGES = ('base_color', 'metallic_roughness', 'normal')


def material_tables():
    """(lut_m, lut_r) uint8 [256]: round(255 srgb_to_linear(k/255)) and round(255 sqrt(srgb_to_linear(k/255))) in fp64, the
    relighter's decoding of feat1 (metallic) and feat2 (alpha) re-encoded as glTF's linear metallic and roughness."""
    from .relight import srgb_to_linear
    lin = srgb_to_linear(np.arange(256, dtype=np.float64) / 255.0)
    return np.rint(255.0 * lin).astype(np.uint8), np.rint(255.0 * np.sqrt(lin)).astype(np.uint8)


# ------------------------------------------------------------------------------------------------ kernels
def weld_cuda(tris, ft, V, vt_ptr, vt_tri):
    """The weld of include/nero_gltf.h on CUDA int32 tensors -> (wv [W], wt [W], wf [T,3]) int32 CUDA tensors."""
    import torch
    from . import ops
    dev = tris.device
    T = tris.shape[0]
    nblk = max(1, ops.ceil_div(V, WELD_THREADS))
    blk_cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
    blk_off = torch.empty(nblk, dtype=torch.int64, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    ops.K('nero_gltf_weld_count', tris, ft, T, V, vt_ptr, vt_tri, blk_cnt, blk_off, total, launches=2 if V else 0)
    W = int(total.item())
    wv = torch.empty(W, dtype=torch.int32, device=dev)
    wt = torch.empty(W, dtype=torch.int32, device=dev)
    wf = torch.empty(T, 3, dtype=torch.int32, device=dev)
    ops.K('nero_gltf_weld_emit', tris, ft, T, V, vt_ptr, vt_tri, blk_off, W, wv, wt, wf)
    return wv, wt, wf


def frames_cuda(verts, tris, vt, ft, vt_ptr, vt_tri, normals, wv, wt):
    """Tangent frames of the welded vertices -> (wnormal [W,3], wtangent [W,4]) float32 CUDA tensors.  vt: the file's uv."""
    import torch
    from . import ops
    W = wv.shape[0]
    wn = torch.empty(W, 3, dtype=torch.float32, device=verts.device)
    wtan = torch.empty(W, 4, dtype=torch.float32, device=verts.device)
    ops.K('nero_gltf_tangents', verts, tris, vt, ft, vt_ptr, vt_tri, normals, wv, wt, W, wn, wtan)
    return wn, wtan


def tangent_space_cuda(verts, tris, vt, ft, wf, wnormal, wtangent, omap):
    """The conversion of include/nero_gltf.h before inpainting -> dict raster (texmap.raster at the map's size on the atlas
    (u, 1 - v)), img [h,w,5] uint8 CUDA.  verts, tris, vt (the file's), ft as numpy; omap uint8 [h,w,3] numpy, row 0 the top
    row of the image file."""
    import torch
    from . import ops
    from .texmap import raster
    h, w = omap.shape[:2]
    vt = np.asarray(vt, np.float32)
    atlas = np.ascontiguousarray(np.stack([vt[:, 0], np.float32(1) - vt[:, 1]], -1))
    r = raster(atlas, ft, verts, tris, w, h)
    dev = torch.device('cuda')
    img = torch.empty(h, w, 5, dtype=torch.uint8, device=dev)
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    ops.K('nero_gltf_tangent_space', r['owner'], w, h, r['texel'], r['texel'].shape[0], up(atlas), up(np.asarray(ft, np.int32)), wf,
          wnormal, wtangent, up(np.asarray(omap, np.uint8)), img)
    return dict(raster=r, img=img)


def metal_rough_cuda(metallic, roughness):
    """uint8 [h,w] planes (the red channel of feat1 / feat2) -> the metallic-roughness texture [h,w,3] uint8 CUDA tensor."""
    import torch
    from . import ops
    dev = torch.device('cuda')
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.uint8)).to(dev)
    lut_m, lut_r = material_tables()
    h, w = metallic.shape
    out = torch.empty(h, w, 3, dtype=torch.uint8, device=dev)
    ops.K('nero_gltf_metal_rough', up(metallic), up(roughness), h * w, up(lut_m), up(lut_r), out)
    return out


def export_arrays(verts, tris, vt, ft, albedo, metallic, roughness, omap=None, profile=None, occlusion=None):
    """The GPU stages of the export -> dict of numpy arrays: positions, normals, texcoords, tangents (None without omap),
    indices [T,3] uint32 (glTF's winding), images {base_color, metallic_roughness, normal (without omap: absent)}, and wv, wt,
    wf, covered (texels of the conversion, 0 without omap).  verts, tris, vt (the file's), ft as load_textured_obj returns
    them; albedo [h,w,3], metallic / roughness [h,w] uint8 (the files' bytes); omap uint8 [h',w',3] (an object-space map);
    occlusion uint8 [h,w] (an ambient-occlusion map of the material maps' size, stored in metallic_roughness's red channel).
    profile (a dict) gets host-clock milliseconds of the phases normals / weld / tangents / tangent_space / metal_rough, each
    ended by a device synchronise."""
    import torch
    from .normalmap import vertex_normals_cuda
    from .simplify import _vertex_triangles
    from .texmap import inpaint
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    vt = np.ascontiguousarray(vt, np.float32)
    ft = np.ascontiguousarray(ft, np.int32)
    if tris.ndim != 2 or tris.shape[1] != 3 or tris.shape[0] < 1 or ft.shape != tris.shape:
        raise ValueError(f'export needs tris [T,3] with T >= 1 and ft of the same shape, got {tris.shape} and {ft.shape}')
    V = verts.shape[0]
    if tris.min() < 0 or tris.max() >= V or ft.min() < 0 or ft.max() >= vt.shape[0]:
        raise ValueError('export: triangle or uv indices out of range')
    if occlusion is not None:
        occlusion = np.asarray(occlusion, np.uint8)
        mh, mw = np.asarray(metallic).shape[:2]
        if occlusion.shape != (mh, mw):
            raise ValueError(f'the occlusion map is {occlusion.shape[1]}x{occlusion.shape[0]} but the material maps are {mw}x{mh}'
                             if occlusion.ndim == 2 else f'the occlusion map must be [h,w] uint8, got {occlusion.shape}')
    clock = [time.perf_counter()]

    def lap(phase):
        if profile is not None:
            torch.cuda.synchronize()
            now = time.perf_counter()
            profile[phase] = profile.get(phase, 0.0) + (now - clock[0]) * 1e3
            clock[0] = now
    dev = torch.device('cuda')
    up = lambda a: torch.from_numpy(a).to(dev)
    v_d, t_d, vt_d, ft_d = up(verts), up(tris), up(vt), up(ft)
    vt_ptr, vt_tri = _vertex_triangles(t_d, V)
    normals = vertex_normals_cuda(v_d, t_d)
    lap('normals')
    wv, wt, wf = weld_cuda(t_d, ft_d, V, vt_ptr, vt_tri)
    lap('weld')
    wn, wtan = frames_cuda(v_d, t_d, vt_d, ft_d, vt_ptr, vt_tri, normals, wv, wt)
    lap('tangents')
    images = {'base_color': np.ascontiguousarray(albedo, np.uint8)}
    covered = 0
    if omap is not None:
        c = tangent_space_cuda(verts, tris, vt, ft, wf, wn, wtan, omap)
        covered = int(c['raster']['texel'].shape[0])
        if covered == 0:
            raise ValueError('no texel of the normal map is covered by a triangle (an empty mesh or atlas)')
        images['normal'] = inpaint(c['img'], c['raster']['owner'])[0][..., :3].cpu().numpy()
        lap('tangent_space')
    images['metallic_roughness'] = metal_rough_cuda(metallic, roughness).cpu().numpy()
    if occlusion is not None:
        images['metallic_roughness'][..., 0] = occlusion
    lap('metal_rough')
    wv, wt, wf = wv.cpu().numpy(), wt.cpu().numpy(), wf.cpu().numpy()
    uv = vt[wt]
    return dict(positions=verts[wv], normals=wn.cpu().numpy(), texcoords=np.stack([uv[:, 0], np.float32(1) - uv[:, 1]], -1),
                tangents=None if omap is None else wtan.cpu().numpy(), indices=wf[:, [0, 2, 1]].astype(np.uint32), images=images,
                wv=wv, wt=wt, wf=wf, covered=covered)


# ------------------------------------------------------------------------------------------------ GLB container
def _pad4(n):
    return (4 - n % 4) % 4


def glb_bytes(positions, normals, texcoords, indices, images, tangents=None, rotation=None, occlusion=False):
    """The GLB file of the module docstring -> bytes.  positions / normals [W,3], texcoords [W,2], tangents [W,4] float32 or
    None, indices [T,3] (written as uint32, already in glTF's winding), images {'base_color', 'metallic_roughness' and
    optionally 'normal': uint8 [h,w,3]}, rotation a node quaternion [x,y,z,w] or None (identity).  occlusion: the
    metallic-roughness texture's red channel holds ambient occlusion, so the material also names it as its
    occlusionTexture.  Deterministic: the same arrays give the same bytes."""
    from .relight import png_bytes
    arrays = {'positions': np.ascontiguousarray(positions, np.float32), 'normals': np.ascontiguousarray(normals, np.float32),
              'texcoords': np.ascontiguousarray(texcoords, np.float32)}
    if tangents is not None:
        arrays['tangents'] = np.ascontiguousarray(tangents, np.float32)
    W = arrays['positions'].shape[0]
    idx = np.ascontiguousarray(indices).reshape(-1)
    if idx.size and (idx.min() < 0 or idx.max() >= W):
        raise ValueError(f'indices outside [0, {W})')
    idx = idx.astype(np.uint32)
    for name, key, k in _ATTRIBUTES:
        if key in arrays and arrays[key].shape != (W, k):
            raise ValueError(f'{name} has shape {arrays[key].shape}; expected ({W}, {k})')
    if set(images) - set(_IMAGES) or not {'base_color', 'metallic_roughness'} <= set(images):
        raise ValueError(f'images must hold base_color and metallic_roughness and may hold normal, got {sorted(images)}')
    if 'normal' in images and tangents is None:
        raise ValueError('a normal texture needs tangents')

    blob, views = bytearray(), []

    def add_view(data, target=None):
        blob.extend(b'\0' * _pad4(len(blob)))
        view = {'buffer': 0, 'byteOffset': len(blob), 'byteLength': len(data)}
        if target is not None:
            view['target'] = target
        views.append(view)
        blob.extend(data)
        return len(views) - 1

    accessors, attributes = [], {}
    for name, key, k in _ATTRIBUTES:
        if key not in arrays:
            continue
        a = arrays[key]
        acc = {'bufferView': add_view(a.tobytes(), _ARRAY_BUFFER), 'componentType': _FLOAT, 'count': W, 'type': f'VEC{k}'}
        if name == 'POSITION':
            acc['min'] = [float(x) for x in (a.min(0) if W else np.zeros(3, np.float32))]
            acc['max'] = [float(x) for x in (a.max(0) if W else np.zeros(3, np.float32))]
        attributes[name] = len(accessors)
        accessors.append(acc)
    accessors.append({'bufferView': add_view(idx.tobytes(), _ELEMENT_ARRAY_BUFFER), 'componentType': _UINT, 'count': int(idx.size),
                      'type': 'SCALAR'})
    gl_images, textures = [], []
    for key in _IMAGES:
        if key in images:
            gl_images.append({'bufferView': add_view(png_bytes(images[key])), 'mimeType': 'image/png'})
            textures.append({'sampler': 0, 'source': len(gl_images) - 1})
    pbr = {'baseColorTexture': {'index': 0}, 'metallicRoughnessTexture': {'index': 1}, 'baseColorFactor': [1.0, 1.0, 1.0, 1.0],
           'metallicFactor': 1.0, 'roughnessFactor': 1.0}
    material = {'name': 'defaultMat', 'pbrMetallicRoughness': pbr}
    if 'normal' in images:
        material['normalTexture'] = {'index': 2}
    if occlusion:
        material['occlusionTexture'] = {'index': 1}
    node = {'mesh': 0}
    if rotation is not None:
        node['rotation'] = [float(x) for x in rotation]
    doc = {'asset': {'version': '2.0', 'generator': 'nero_b200 gltf export'}, 'scene': 0, 'scenes': [{'nodes': [0]}], 'nodes': [node],
           'meshes': [{'primitives': [{'attributes': attributes, 'indices': len(accessors) - 1, 'material': 0, 'mode': _TRIANGLES}]}],
           'materials': [material], 'textures': textures, 'images': gl_images,
           'samplers': [{'magFilter': _LINEAR, 'minFilter': _LINEAR_MIPMAP_LINEAR, 'wrapS': _REPEAT, 'wrapT': _REPEAT}],
           'accessors': accessors, 'bufferViews': views, 'buffers': [{'byteLength': len(blob) + _pad4(len(blob))}]}
    js = json.dumps(doc, separators=(',', ':')).encode()
    js += b' ' * _pad4(len(js))
    blob.extend(b'\0' * _pad4(len(blob)))
    total = 12 + 8 + len(js) + 8 + len(blob)
    return (struct.pack('<III', _GLB_MAGIC, 2, total) + struct.pack('<II', len(js), _CHUNK_JSON) + js +
            struct.pack('<II', len(blob), _CHUNK_BIN) + bytes(blob))


def export(obj_path, normal_map_path=None, trans=False, profile=None, stats=None, occlusion_path=None):
    """The .glb of the textured OBJ at obj_path (and the object-space normal map at normal_map_path, and the ambient-occlusion
    map at occlusion_path) -> bytes.  trans: the object is stored as tools/relight.py --trans takes it, so the node is not
    rotated.  profile (a dict) gets host-clock
    milliseconds of the phases read / normals / weld / tangents / tangent_space / metal_rough / container; stats (a dict) gets
    positions, welded, triangles, covered."""
    import cv2
    from .normalmap import read_normal_map_bytes
    from .relight import textured_obj_files
    t0 = time.perf_counter()
    verts, tris, vt, ft, files = textured_obj_files(obj_path)
    imgs = {}
    for k, path in files.items():
        im = cv2.imread(path, cv2.IMREAD_COLOR) if os.path.isfile(path) else None
        if im is None:
            raise ValueError(f'{path}: texture file is missing or not an image OpenCV can read')
        imgs[k] = im[..., ::-1]
    sizes = {k: im.shape[:2] for k, im in imgs.items()}
    if len(set(sizes.values())) != 1:
        raise ValueError(f'{obj_path}: texture maps differ in size: ' + ', '.join(f'{files[k]} {s[1]}x{s[0]}' for k, s in sizes.items()))
    omap = None if normal_map_path is None else read_normal_map_bytes(normal_map_path)
    occ = None
    if occlusion_path is not None:
        from .occlusion import read_occlusion_map
        occ = read_occlusion_map(occlusion_path)
        (mh, mw), (oh, ow) = imgs['metallic'].shape[:2], occ.shape
        if (oh, ow) != (mh, mw):
            raise ValueError(f'{occlusion_path}: the occlusion map is {ow}x{oh} but the material maps are {mw}x{mh}')
    if profile is not None:
        profile['read'] = (time.perf_counter() - t0) * 1e3
    out = export_arrays(verts, tris, vt, ft, imgs['albedo'], imgs['metallic'][..., 0], imgs['roughness'][..., 0], omap, profile, occ)
    t1 = time.perf_counter()
    data = glb_bytes(out['positions'], out['normals'], out['texcoords'], out['indices'], out['images'], out['tangents'],
                     None if trans else Z_UP_ROTATION, occ is not None)
    if profile is not None:
        profile['container'] = (time.perf_counter() - t1) * 1e3
    if stats is not None:
        stats.update(positions=int(verts.shape[0]), welded=int(out['wv'].shape[0]), triangles=int(tris.shape[0]), covered=out['covered'])
    return data


# ------------------------------------------------------------------------------------------------ reading back
def _png_decode(data):
    """This exporter's PNGs (relight.png_bytes: 8-bit RGB or RGBA, not interlaced, filter type 0 on every row) -> uint8
    [h,w,c].  Anything else raises ValueError."""
    if data[:8] != _PNG_SIGNATURE:
        raise ValueError('image is not a PNG')
    pos, idat, hdr = 8, [], None
    while pos + 8 <= len(data):
        n, tag = struct.unpack('>I4s', data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        if len(body) != n or struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])[0] != zlib.crc32(tag + body) & 0xffffffff:
            raise ValueError(f'PNG chunk {tag!r} is truncated or fails its CRC')
        if tag == b'IHDR':
            hdr = struct.unpack('>IIBBBBB', body)
        elif tag == b'IDAT':
            idat.append(body)
        elif tag == b'IEND':
            break
        pos += 12 + n
    if hdr is None or hdr[2] != 8 or hdr[3] not in (2, 6) or hdr[4:] != (0, 0, 0):
        raise ValueError(f'PNG header {hdr}: only 8-bit RGB / RGBA, not interlaced, is read')
    w, h, c = hdr[0], hdr[1], 4 if hdr[3] == 6 else 3
    raw = np.frombuffer(zlib.decompress(b''.join(idat)), np.uint8)
    if raw.size != h * (1 + w * c):
        raise ValueError('PNG image data has the wrong size')
    raw = raw.reshape(h, 1 + w * c)
    if (raw[:, 0] != 0).any():
        raise ValueError('PNG rows use a filter other than type 0')
    return raw[:, 1:].reshape(h, w, c).copy()


def read_glb(path):
    """Read a .glb of this exporter's subset (a path or the bytes) -> dict json (the parsed JSON), positions, normals,
    texcoords, tangents (or None) float32, indices [T,3] uint32, rotation (or None), images {base_color, metallic_roughness[,
    normal]: uint8 [h,w,3]}, occlusion (the red channel [h,w] uint8 of the occlusionTexture's image, or None) and
    occlusion_strength (its strength, 1.0 when not given, or None).  Anything outside the subset raises ValueError: another container version, chunk layout, more
    than one buffer / mesh / primitive, attributes other than this exporter's, component types, strides, sparse accessors,
    unaligned views or images that are not this exporter's PNGs."""
    data = path if isinstance(path, (bytes, bytearray)) else open(path, 'rb').read()
    data = bytes(data)
    if len(data) < 20:
        raise ValueError('not a GLB file: too short')
    magic, version, length = struct.unpack('<III', data[:12])
    if magic != _GLB_MAGIC or version != 2 or length != len(data):
        raise ValueError(f'not a glTF 2.0 GLB file (magic {magic:#x}, version {version}, length {length} of {len(data)} bytes)')
    jl, jt = struct.unpack('<II', data[12:20])
    if jt != _CHUNK_JSON or jl % 4 or 20 + jl + 8 > len(data):
        raise ValueError('the first GLB chunk is not a 4-byte aligned JSON chunk')
    doc = json.loads(data[20:20 + jl].decode())
    bl, bt = struct.unpack('<II', data[20 + jl:28 + jl])
    if bt != _CHUNK_BIN or bl % 4 or 28 + jl + bl != len(data):
        raise ValueError('the second GLB chunk is not a 4-byte aligned BIN chunk ending the file')
    blob = data[28 + jl:]
    if doc.get('asset', {}).get('version') != '2.0' or len(doc.get('buffers', [])) != 1 or 'uri' in doc['buffers'][0]:
        raise ValueError('expected asset version 2.0 and one buffer held in the BIN chunk')
    if doc['buffers'][0]['byteLength'] > len(blob):
        raise ValueError('the buffer is longer than the BIN chunk')
    if len(doc.get('meshes', [])) != 1 or len(doc['meshes'][0]['primitives']) != 1 or len(doc.get('nodes', [])) != 1:
        raise ValueError('expected one node, one mesh and one primitive')
    prim = doc['meshes'][0]['primitives'][0]
    if prim.get('mode', _TRIANGLES) != _TRIANGLES or 'indices' not in prim:
        raise ValueError('expected an indexed triangle primitive')

    def view_bytes(i):
        v = doc['bufferViews'][i]
        off, n = v.get('byteOffset', 0), v['byteLength']
        if v.get('buffer') != 0 or 'byteStride' in v or off % 4 or off + n > len(blob):
            raise ValueError(f'bufferView {i} is strided, unaligned or outside the buffer')
        return blob[off:off + n]

    def accessor(i, ctype, kind):
        a = doc['accessors'][i]
        if a.get('componentType') != ctype or a.get('type') != kind or 'sparse' in a or a.get('byteOffset', 0) or a.get('normalized'):
            raise ValueError(f'accessor {i}: expected {kind} of component type {ctype} without offset or sparse storage')
        k = {'SCALAR': 1, 'VEC2': 2, 'VEC3': 3, 'VEC4': 4}[kind]
        raw = view_bytes(a['bufferView'])
        if len(raw) < 4 * k * a['count']:
            raise ValueError(f'accessor {i}: its bufferView is too short')
        return np.frombuffer(raw[:4 * k * a['count']], np.float32 if ctype == _FLOAT else np.uint32).reshape(a['count'], k).copy()

    attrs = prim['attributes']
    if set(attrs) - {n for n, _, _ in _ATTRIBUTES} or not {'POSITION', 'NORMAL', 'TEXCOORD_0'} <= set(attrs):
        raise ValueError(f'attributes {sorted(attrs)}: expected POSITION, NORMAL, TEXCOORD_0 and optionally TANGENT')
    out = {'json': doc}
    for name, key, k in _ATTRIBUTES:
        out[key] = accessor(attrs[name], _FLOAT, f'VEC{k}') if name in attrs else None
    W = out['positions'].shape[0]
    if any(out[key] is not None and out[key].shape[0] != W for _, key, _ in _ATTRIBUTES):
        raise ValueError('attributes differ in count')
    idx = accessor(prim['indices'], _UINT, 'SCALAR').reshape(-1)
    if idx.size % 3 or (idx.size and idx.max() >= W):
        raise ValueError('indices are not triangles of the vertices')
    out['indices'] = idx.reshape(-1, 3)
    out['rotation'] = doc['nodes'][0].get('rotation')
    mats = doc.get('materials', [])
    if len(mats) != 1 or prim.get('material') != 0:
        raise ValueError('expected one material')
    pbr = mats[0].get('pbrMetallicRoughness', {})
    refs = {'base_color': pbr.get('baseColorTexture'), 'metallic_roughness': pbr.get('metallicRoughnessTexture'),
            'normal': mats[0].get('normalTexture')}
    out['images'] = {}
    for key, ref in refs.items():
        if ref is None:
            continue
        img = doc['images'][doc['textures'][ref['index']]['source']]
        if img.get('mimeType') != 'image/png' or 'bufferView' not in img:
            raise ValueError(f'{key} image is not a PNG held in a bufferView')
        out['images'][key] = _png_decode(view_bytes(img['bufferView']))
    occ = mats[0].get('occlusionTexture')
    out['occlusion'], out['occlusion_strength'] = None, None
    if occ is not None:
        img = doc['images'][doc['textures'][occ['index']]['source']]
        if img.get('mimeType') != 'image/png' or 'bufferView' not in img:
            raise ValueError('occlusion image is not a PNG held in a bufferView')
        out['occlusion'] = _png_decode(view_bytes(img['bufferView']))[..., 0].copy()
        out['occlusion_strength'] = float(occ.get('strength', 1.0))
    return out
