"""UV texture-map export of stage-II materials on the GPU: the reference's extract_materials_texture_map.py, stated once.

Reference being replaced (paths relative to the reference repository):
  extract_materials_texture_map.py:75-82    xatlas unwrap (max_iterations = 0)            -> uv_atlas (host, uv_atlas.cu)
  extract_materials_texture_map.py:89-106   nvdiffrast rasterize / interpolate of uv*2-1   -> raster (k_texmap.cu)
  extract_materials_texture_map.py:108-129  predict_materials_n2m on the covered texels   -> the stage-II material chain
  extract_materials_texture_map.py:130-133  linear_to_srgb, x 255, astype(uint8)          -> encode
  extract_materials_texture_map.py:136-149  dilation / erosion / kd-tree inpainting       -> inpaint
  extract_materials_texture_map.py:152-160  RGB -> BGR, cv2.resize(INTER_LINEAR) 2x        -> downsample
  extract_materials_texture_map.py:162-197  feat{0,1,2}_0.jpg, mesh_0.obj, mesh_0.mtl     -> write_textured_obj
  network/field.py:925-932                  [albedo(3), metallic, roughness]

The protocol:
  * The atlas is (ssaa h0) x (ssaa w0) texels.  Texel (x, y) samples uv = ((x + 1/2) / w, (y + 1/2) / h); row 0 is v = 0 and
    is the first image row written.  A texel belongs to at most one triangle (snapped uv, exact edge functions, top-left
    rule); xyz is the mesh position interpolated with the triangle's barycentrics.
  * Materials: albedo, metallic and roughness rescaled to [0.04^2, 1] and NOT square-rooted (unlike the per-vertex export),
    computed in fp32.  The reference runs under torch.cuda.amp.autocast, i.e. in fp16 on its GPU.
  * Encoding: linear_to_srgb of all five channels in fp64, x 255, truncated; uncovered texels are 0.
  * Inpainting: every uncovered texel with a covered texel within Manhattan distance 32 copies the 5 bytes of the nearest
    search texel (covered, within Manhattan distance 3 of an uncovered texel or of the border): smallest squared distance,
    ties to the smallest row-major index (the reference's kd-tree breaks ties arbitrarily).
  * Down-sampling by ssaa = 2: (a + b + c + d + 2) >> 2 per channel; ssaa = 1 skips it.
  * Files: feat0_0.png (albedo RGB), feat1_0.png (metallic), feat2_0.png (roughness), both grey replicated to RGB.  They
    are 8-bit PNGs, not the reference's JPEGs: the output is lossless and needs no image library; so mesh_0.mtl's map_Kd
    names feat0_0.png.  Otherwise mesh_0.obj / mesh_0.mtl are byte for byte what the reference writes for the same arrays.
  * The unwrapper is this project's own (charts, packing and the uv coordinates differ from xatlas's; DESIGN.md section 2).
"""
import ctypes
import os

import numpy as np

MAT_CHANNELS = 5          # albedo rgb, metallic, roughness
BATCH = 1 << 18           # material rows per chain launch: ~29.8 KB of workspace per row, ~7.8 GB


def uv_atlas(verts, tris, width, height, gutter):
    """Unwrap a mesh into a width x height texel atlas with `gutter` texels between charts and from the border.
    -> (vt [N_uv,2] float32 in [0,1], ft [T,3] int32), xatlas's format: ft indexes vt, the mesh keeps its vertices."""
    from . import ops
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    T = tris.shape[0]
    vt = np.zeros((3 * T, 2), np.float32)
    ft = np.zeros((T, 3), np.int32)
    n_uv, n_charts = ctypes.c_int(0), ctypes.c_int(0)
    ops.call('nero_uv_atlas_host', verts, verts.shape[0], tris, T, width, height, gutter, vt, ft, ctypes.byref(n_uv),
             ctypes.byref(n_charts))
    return vt[:n_uv.value].copy(), ft


def raster(vt, ft, verts, tris, width, height):
    """-> dict of CUDA tensors: owner [h,w] int32 (-1 uncovered), cover [h,w] int32 (covering triangles), texel [n] int32
    (covered texels in row-major order) and xyz [n,3] float32 (interpolated positions)."""
    import torch
    from . import ops
    dev = torch.device('cuda')
    up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).to(dev)
    vt_d, ft_d, v_d, f_d = up(vt, np.float32), up(ft, np.int32), up(verts, np.float32), up(tris, np.int32)
    N = width * height
    owner = torch.empty(N, dtype=torch.int32, device=dev)
    cover = torch.empty(N, dtype=torch.int32, device=dev)
    ops.K('nero_tex_raster', vt_d, ft_d, ft_d.shape[0], width, height, owner, cover)
    nblk = ops.ceil_div(N, 1024)
    blk_cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
    blk_off = torch.empty(nblk, dtype=torch.int64, device=dev)
    total = torch.empty(1, dtype=torch.int64, device=dev)
    ops.K('nero_tex_compact_count', owner, width, height, blk_cnt, blk_off, total, launches=2)
    n = int(total.item())
    texel = torch.empty(n, dtype=torch.int32, device=dev)
    xyz = torch.empty(n, 3, dtype=torch.float32, device=dev)
    ops.K('nero_tex_compact_emit', owner, width, height, vt_d, ft_d, v_d, f_d, blk_off, n, texel, xyz)
    return {'owner': owner.view(height, width), 'cover': cover.view(height, width), 'texel': texel, 'xyz': xyz}


def query_materials(renderer, xyz, batch=BATCH):
    """[n,5] float32 CUDA tensor (albedo rgb, metallic, roughness in [0.04^2, 1]) of NeROMaterialRenderer at the points."""
    import torch
    out = torch.empty(xyz.shape[0], MAT_CHANNELS, dtype=torch.float32, device=xyz.device)
    for i in range(0, xyz.shape[0], batch):
        m, r, a = renderer.query_materials(xyz[i:i + batch])
        out[i:i + batch, :3], out[i:i + batch, 3:4], out[i:i + batch, 4:5] = a, m, r
    return out


def encode(mat, texel, width, height):
    """-> [h,w,5] uint8 CUDA tensor: the sRGB-encoded, truncated materials at their texels, 0 elsewhere."""
    import torch
    from . import ops
    img = torch.empty(height, width, MAT_CHANNELS, dtype=torch.uint8, device=mat.device)
    ops.K('nero_tex_encode', mat.contiguous(), texel, texel.shape[0], width, height, img)
    return img


def inpaint(img, owner):
    """-> (img with the seam band filled [h,w,5] uint8, src [h,w] int32: the texel each filled texel copies, -1 elsewhere)."""
    import torch
    from . import ops
    h, w = owner.shape
    dev = img.device
    search = torch.empty(h, w, dtype=torch.uint8, device=dev)
    tiles = torch.empty(ops.ceil_div(h, 16) * ops.ceil_div(w, 16), dtype=torch.int32, device=dev)
    out = torch.empty_like(img)
    src = torch.empty(h, w, dtype=torch.int32, device=dev)
    ops.K('nero_tex_inpaint', img, owner, w, h, search, tiles, out, src, launches=2)
    return out, src


def downsample(img):
    """2x down-sample of [h,w,5] uint8 (h, w even)."""
    import torch
    from . import ops
    h, w = img.shape[:2]
    out = torch.empty(h // 2, w // 2, img.shape[2], dtype=torch.uint8, device=img.device)
    ops.K('nero_tex_downsample', img, w, h, out)
    return out


def split_images(img):
    """[h,w,5] uint8 -> (albedo [h,w,3], metallic [h,w,3], roughness [h,w,3]) numpy, RGB order, grey replicated."""
    img = img.cpu().numpy() if hasattr(img, 'cpu') else np.asarray(img)
    rep = lambda c: np.ascontiguousarray(np.repeat(img[..., c:c + 1], 3, -1))
    return np.ascontiguousarray(img[..., :3]), rep(3), rep(4)


def bake_textures(renderer, verts, tris, vt, ft, size=(1024, 1024), ssaa=2):
    """The material textures of a stage-II NeROMaterialRenderer on the atlas (vt, ft) of the mesh (verts, tris).
    size = (h0, w0) of the output; the atlas is rasterised at ssaa x that.  -> (albedo, metallic, roughness), each
    [h0,w0,3] uint8 numpy."""
    h0, w0 = size
    if ssaa not in (1, 2):
        raise ValueError(f'ssaa {ssaa}: expected 1 or 2')
    h, w = h0 * ssaa, w0 * ssaa
    r = raster(vt, ft, verts, tris, w, h)
    if r['texel'].shape[0] == 0:
        raise ValueError(f'no texel of the {w}x{h} atlas is covered by a triangle (an empty mesh or atlas)')
    mat = query_materials(renderer, r['xyz'])
    img, _ = inpaint(encode(mat, r['texel'], w, h), r['owner'])
    if ssaa == 2:
        img = downsample(img)
    return split_images(img)


def _fmt(a):
    """Each value as the reference's f-string writes a numpy scalar: a float32 as repr(float(x)), an integer as str."""
    a = np.asarray(a)
    return a.astype(np.float64).astype(str) if a.dtype.kind == 'f' else a.astype(str)


def _lines(prefix, cols, sep):
    out = np.strings.add(prefix, cols[0])
    for c, s in zip(cols[1:], sep):
        out = np.strings.add(np.strings.add(out, s), c)
    return np.strings.add(out, ' \n')


def obj_text(verts, tris, vt, ft, cas=0):
    """(obj, mtl) text of extract_materials_texture_map.py:170-197 for the same arrays, with map_Kd naming the PNG."""
    v = np.asarray(verts, np.float32)
    vt = np.asarray(vt, np.float32)
    f = np.asarray(tris).astype(np.int64) + 1
    t = np.asarray(ft).astype(np.int64) + 1
    parts = [f'mtllib mesh_{cas}.mtl \n']
    if v.shape[0]:
        parts += _lines('v ', [_fmt(v[:, k]) for k in range(3)], [' ', ' ']).tolist()
    if vt.shape[0]:
        parts += _lines('vt ', [_fmt(vt[:, 0]), _fmt(np.float32(1) - vt[:, 1])], [' ']).tolist()
    parts.append('usemtl defaultMat \n')
    if f.shape[0]:
        parts += _lines('f ', [_fmt(f[:, 0]), _fmt(t[:, 0]), _fmt(f[:, 1]), _fmt(t[:, 1]), _fmt(f[:, 2]), _fmt(t[:, 2])],
                        ['/', ' ', '/', ' ', '/']).tolist()
    mtl = f'newmtl defaultMat \nKa 1 1 1 \nKd 1 1 1 \nKs 0 0 0 \nTr 1 \nillum 1 \nNs 0 \nmap_Kd feat0_{cas}.png \n'
    return ''.join(parts), mtl


def write_textured_obj(out_dir, verts, tris, vt, ft, images, cas=0):
    """Write mesh_0.obj, mesh_0.mtl and feat{0,1,2}_0.png (images = bake_textures' (albedo, metallic, roughness))."""
    from .relight import write_png
    os.makedirs(out_dir, exist_ok=True)
    for k, im in enumerate(images):
        write_png(os.path.join(out_dir, f'feat{k}_{cas}.png'), im)
    obj, mtl = obj_text(verts, tris, vt, ft, cas)
    with open(os.path.join(out_dir, f'mesh_{cas}.obj'), 'w') as fp:
        fp.write(obj)
    with open(os.path.join(out_dir, f'mesh_{cas}.mtl'), 'w') as fp:
        fp.write(mtl)
