"""Relighting of stage-II results on the GPU: the scene the reference renders with Blender Cycles, stated once.

Reference being replaced (paths relative to the reference repository):
  relight.py:15-24                                   runs Blender on blender_backend/relight_backend.py
  blender_backend/relight_backend.py:20-85           scene set-up: mesh, vertex-colour materials, environment light, cameras
  blender_backend/blender_utils.py:48-68, 101-116    set_camera_by_pose, generate_relghting_poses
  extract_materials.py:23-33                         per-vertex material export (`save_materials` here)

The scene, in scene coordinates (= Blender world coordinates, z up):
  * Geometry: the PLY mesh; with --trans rotated by +90 degrees about x (relight_backend.py:46-48), x_scene = MESH_TRANS @ x_mesh.
    Flat shading with the face normal.  Marching-cubes meshes here are wound with cross(v1-v0, v2-v0) pointing into the
    solid, so the outward normal is the negated cross product; it is flipped towards the incoming ray where it faces away
    (two-sided surfaces).
  * Materials: the exported per-vertex values decoded with srgb_to_linear (undoing the export gamma, as Blender's
    vertex-colour path does), interpolated barycentrically at the hit point.  The BRDF's roughness argument is
    alpha = (decoded roughness)^2, the value NeRO's shading functions take (network/field.py:794, 893).
  * Textured materials (the textured OBJ of tools/extract_materials_texture_map.py, read by load_textured_obj): the texels
    decoded with srgb_to_linear(k / 255).  At a hit with barycentrics (u, v), w0 = 1 - u - v:
      uv = w0 uv0 + u uv1 + v uv2 in fp32, as the per-vertex rows are interpolated;
      s = uv.x W - 1/2, t = (1 - uv.y) H - 1/2 for a W x H texture whose row 0 is the top row of the image file (the
      OBJ / Blender convention, v = 0 at the bottom row; texmap.obj_text stores 1 - v_atlas, so this is the baked texel);
      x0 = floor(s), fx = s - x0, likewise y0, fy; the four taps wrap (repeat, positive modulo);
      bilinear in lerp form a + f (b - a) per channel, along x first, so a constant texture gives its value exactly.
    albedo and metallic are the filtered values and alpha = the filtered roughness, NOT squared: the texture export stores
    the rescaled roughness NeRO's shading takes (predict_materials_n2m, network/field.py:925-932), the per-vertex export its
    square root.  There is no mip-mapping: the per-pixel jitter averages the texture over the pixel footprint as samples
    accumulate, and a texture minified to several texels per pixel aliases at low sample counts.
  * BRDF: NeRO's stage-II model (the terms the materials were fitted under), not Blender's Principled BSDF:
    albedo (1-m)/pi + F D G / (4 NoV NoL), F0 = 0.04 (1-m) + m albedo, Schlick F, NeRO's D (with its +1e-4) and
    G = 'schlick' or 'ggx_smith' (nero_b200/csrc/math_relight.cuh, math_mc.cuh).
  * Cameras: frame k of generate_relghting_poses(num, azimuth, elevation, cam_dist) moved into Blender space as
    set_camera_by_pose does: the camera sits at dist (cos az cos el, sin az cos el, sin el), looks at the origin with up +z,
    az sweeps azimuth +- 90 degrees.  Poses are world -> camera [R | t] with OpenCV axes (x right, y down, z forward).
    Intrinsics of Blender's default camera (50 mm lens, 36 mm sensor, sensor fit auto): f = 50/36 max(W, H) pixels, principal
    point at the image centre.  The pixel sample is jittered uniformly inside the pixel (a box filter; Cycles' default is a
    1.5 px Blackman-Harris filter).
  * Environment: an equirectangular map with Cycles' default mapping as we read it, u = 0.5 - atan2(d_y, d_x) / 2pi,
    v = 0.5 + atan2(d_z, hypot(d_x, d_y)) / pi, v = 0 at the bottom row; piecewise constant per texel, the function the
    importance sampler integrates.
  * Output: transparent film (relight_backend.py:21).  A pixel is linear RGB, premultiplied, plus alpha = the fraction of
    camera samples that hit the mesh.  PNGs are RGBA8 with straight alpha and the plain sRGB transfer with clamping (Blender
    2.8-3.x's default Filmic view transform is not reproduced).
Parity with Blender is unpinned (DESIGN.md section 2).
"""
import os
import struct
import zlib

import numpy as np

MESH_TRANS = np.asarray([[1, 0, 0], [0, 0, -1], [0, 1, 0]], np.float64)   # --trans: +90 degrees about x


# ------------------------------------------------------------------------------------------------ colour transfer
def linear_to_srgb(linear):
    """utils/raw_utils.py:11-15 (numpy branch), the export gamma of extract_materials.py."""
    eps = np.finfo(np.float32).eps
    srgb0 = 323 / 25 * linear
    srgb1 = (211 * np.maximum(eps, linear) ** (5 / 12) - 11) / 200
    return np.where(linear <= 0.0031308, srgb0, srgb1)


def srgb_to_linear(srgb):
    """utils/raw_utils.py:26-31 (numpy branch)."""
    eps = np.finfo(np.float32).eps
    linear0 = 25 / 323 * srgb
    linear1 = np.maximum(((200 * srgb + 11) / 211), eps) ** (12 / 5)
    return np.where(srgb <= 0.04045, linear0, linear1)


# ------------------------------------------------------------------------------------------------ materials
MATERIAL_NAMES = ('metallic', 'roughness', 'albedo')


def save_materials(material_dir, materials):
    """Write NeROMaterialRenderer.predict_materials() output as the reference does (extract_materials.py:31-33):
    {metallic,roughness,albedo}.npy = linear_to_srgb of the [V,1], [V,1], [V,3] arrays.

    The gamma is applied on purpose.  The reference's Blender script stores the materials as vertex colours, and Blender
    applies an inverse gamma to vertex colours, so without it the rendered values would be wrong
    (https://blender.stackexchange.com/questions/87576/vertex-colors-loose-color-data/87583#87583).  `load_materials`
    undoes it the same way."""
    os.makedirs(material_dir, exist_ok=True)
    for k in MATERIAL_NAMES:
        np.save(os.path.join(material_dir, f'{k}.npy'), linear_to_srgb(materials[k]))


def load_materials(material_dir):
    """The exported arrays decoded with srgb_to_linear: {'metallic': [V,1], 'roughness': [V,1], 'albedo': [V,3]} float32."""
    return {k: srgb_to_linear(np.load(os.path.join(material_dir, f'{k}.npy'))).astype(np.float32) for k in MATERIAL_NAMES}


def vertex_material_table(materials):
    """[V,8] float32 rows (albedo rgb, metallic, roughness, 0, 0, 0), the layout nero_relight_render reads."""
    a = np.asarray(materials['albedo'], np.float32).reshape(-1, 3)
    m = np.asarray(materials['metallic'], np.float32).reshape(-1)
    r = np.asarray(materials['roughness'], np.float32).reshape(-1)
    if not (a.shape[0] == m.shape[0] == r.shape[0]):
        raise ValueError(f'material arrays disagree on the vertex count: {a.shape[0]}, {m.shape[0]}, {r.shape[0]}')
    t = np.zeros((a.shape[0], 8), np.float32)
    t[:, :3], t[:, 3], t[:, 4] = a, m, r
    return t


class UVMaterials:
    """Materials as UV textures: vt [N,2] float uv, ft [T,3] int indices into vt (one row per triangle of the mesh), and
    linear (decoded) maps with row 0 at the top of the image: albedo [H,W,3], metallic [H,W] or [H,W,1], roughness [H,W] or
    [H,W,1] (the rescaled roughness, the BRDF's alpha itself)."""

    def __init__(self, vt, ft, albedo, metallic, roughness):
        self.vt = np.ascontiguousarray(vt, np.float32)
        self.ft = np.ascontiguousarray(ft, np.int32)
        self.albedo = np.asarray(albedo, np.float32)
        self.metallic = np.asarray(metallic, np.float32)
        self.roughness = np.asarray(roughness, np.float32)
        if self.vt.ndim != 2 or self.vt.shape[1] != 2 or self.vt.shape[0] < 1:
            raise ValueError(f'vt has shape {self.vt.shape}; expected [N,2] with N >= 1')
        if self.ft.ndim != 2 or self.ft.shape[1] != 3:
            raise ValueError(f'ft has shape {self.ft.shape}; expected [T,3]')
        if self.ft.size and (self.ft.min() < 0 or self.ft.max() >= self.vt.shape[0]):
            raise ValueError(f'ft indexes [{self.ft.min()}, {self.ft.max()}] outside the {self.vt.shape[0]} uv vertices')
        if self.albedo.ndim != 3 or self.albedo.shape[2] != 3 or min(self.albedo.shape[:2]) < 1:
            raise ValueError(f'albedo map has shape {self.albedo.shape}; expected [H,W,3]')
        hw = self.albedo.shape[:2]
        for k in ('metallic', 'roughness'):
            a = getattr(self, k)
            if a.shape not in (hw, hw + (1,)):
                raise ValueError(f'{k} map has shape {a.shape}; the albedo map is {hw}')
        if not all(np.isfinite(a).all() for a in (self.vt, self.albedo, self.metallic, self.roughness)):
            raise ValueError('UV materials hold non-finite values')

    def texel_table(self):
        """[H,W,8] float32 texel rows (albedo rgb, metallic, roughness, 0, 0, 0), the layout nero_relight_render_textured
        reads."""
        H, W = self.albedo.shape[:2]
        t = np.zeros((H, W, 8), np.float32)
        t[..., :3], t[..., 3], t[..., 4] = self.albedo, self.metallic.reshape(H, W), self.roughness.reshape(H, W)
        return t


def _obj_error(path, what):
    return ValueError(f'{path}: {what}')


def _obj_index(tok, n, path, lineno, what):
    try:
        i = int(tok)
    except ValueError:
        raise _obj_error(path, f'line {lineno}: {what} index {tok!r} is not an integer') from None
    if not 1 <= i <= n:
        raise _obj_error(path, f'line {lineno}: {what} index {i} is out of range [1, {n}]')
    return i - 1


def _read_map(path, channels):
    """An 8-bit image file -> float32 [H,W,len(channels)] decoded with srgb_to_linear(k / 255); channels index RGB."""
    import cv2
    if not os.path.isfile(path):
        raise ValueError(f'{path}: texture file is missing')
    img = cv2.imread(path, cv2.IMREAD_COLOR)
    if img is None:
        raise ValueError(f'{path}: not an image OpenCV can read')
    rgb = img[..., ::-1]
    return srgb_to_linear(rgb[..., list(channels)].astype(np.float64) / 255).astype(np.float32)


def load_textured_obj(path):
    """Read the textured OBJ of tools/extract_materials_texture_map.py (or the reference's) ->
    (verts [V,3] float32, tris [T,3] int32, vt [N,2] float32 as written in the file, ft [T,3] int32,
    maps {'metallic' [H,W,1], 'roughness' [H,W,1], 'albedo' [H,W,3]} float32 linear, row 0 at the top).

    The OBJ gives v, vt, triangles `f a/b c/d e/f` (the a/b/n form too; normals are ignored) and `mtllib`; the MTL's
    `map_Kd` names the albedo file, and the metallic and roughness files are named alike with feat1_ and feat2_ in place of
    feat0_.  Images are read with OpenCV (PNG or JPEG); metallic and roughness come from the red channel.  Every value is
    decoded with srgb_to_linear(k / 255), as load_materials decodes its arrays.  Anything else raises ValueError naming the
    file: faces that are not triangles or lack uv indices, indices out of range, non-finite values, a missing MTL or texture
    file, or maps of different sizes."""
    verts, uvs, faces, mtllib = [], [], [], None
    with open(path) as f:
        lines = f.read().splitlines()
    for lineno, line in enumerate(lines, 1):
        tok = line.split()
        if not tok:
            continue
        if tok[0] == 'v':
            verts.append((lineno, tok[1:4]))
        elif tok[0] == 'vt':
            uvs.append((lineno, tok[1:3]))
        elif tok[0] == 'f':
            faces.append((lineno, tok[1:]))
        elif tok[0] == 'mtllib' and mtllib is None:
            mtllib = line.strip()[len('mtllib'):].strip()

    def floats(rows, k, what):
        out = np.zeros((len(rows), k), np.float64)
        for i, (lineno, t) in enumerate(rows):
            try:
                if len(t) < k:
                    raise ValueError
                out[i] = [float(x) for x in t[:k]]
            except ValueError:
                raise _obj_error(path, f'line {lineno}: {what} needs {k} numbers') from None
        if not np.isfinite(out).all():
            raise _obj_error(path, f'non-finite {what} coordinates')
        return out
    V, N = floats(verts, 3, 'vertex'), floats(uvs, 2, 'texture vertex')
    tris = np.zeros((len(faces), 3), np.int32)
    ft = np.zeros((len(faces), 3), np.int32)
    for i, (lineno, corners) in enumerate(faces):
        if len(corners) != 3:
            raise _obj_error(path, f'line {lineno}: a face with {len(corners)} corners (only triangles are supported)')
        for c, corner in enumerate(corners):
            parts = corner.split('/')
            if len(parts) < 2 or not parts[1]:
                raise _obj_error(path, f'line {lineno}: face corner {corner!r} has no uv index')
            tris[i, c] = _obj_index(parts[0], V.shape[0], path, lineno, 'vertex')
            ft[i, c] = _obj_index(parts[1], N.shape[0], path, lineno, 'uv')
    if not faces:
        raise _obj_error(path, 'no faces')
    if mtllib is None:
        raise _obj_error(path, 'no mtllib line')
    mtl_path = os.path.join(os.path.dirname(path), mtllib)
    if not os.path.isfile(mtl_path):
        raise ValueError(f'{mtl_path}: material file is missing')
    map_kd = None
    with open(mtl_path) as f:
        for line in f:
            if line.split()[:1] == ['map_Kd']:
                map_kd = line.strip()[len('map_Kd'):].strip()
                break
    if map_kd is None:
        raise ValueError(f'{mtl_path}: no map_Kd line')
    name = os.path.basename(map_kd)
    if 'feat0_' not in name:
        raise ValueError(f'{mtl_path}: map_Kd {map_kd!r} is not named feat0_*, so the metallic and roughness maps cannot be found')
    base = os.path.join(os.path.dirname(mtl_path), os.path.dirname(map_kd))
    files = {'albedo': os.path.join(base, name), 'metallic': os.path.join(base, name.replace('feat0_', 'feat1_', 1)),
             'roughness': os.path.join(base, name.replace('feat0_', 'feat2_', 1))}
    maps = {k: _read_map(files[k], (0, 1, 2) if k == 'albedo' else (0,)) for k in MATERIAL_NAMES}
    sizes = {k: m.shape[:2] for k, m in maps.items()}
    if len(set(sizes.values())) != 1:
        raise ValueError(f'{path}: texture maps differ in size: ' + ', '.join(f'{files[k]} {sizes[k][1]}x{sizes[k][0]}' for k in MATERIAL_NAMES))
    return V.astype(np.float32), tris, N.astype(np.float32), ft, maps


# ------------------------------------------------------------------------------------------------ environment maps
def load_env_map(path):
    """Read an HDR environment map -> float32 [H, W, 3] linear radiance, row 0 at the top.

    Radiance .hdr (RGBE, flat or new-style run-length scanlines) and OpenEXR scanline files with NONE, ZIPS or ZIP
    compression and half / float / uint channels named R, G, B.  Any other compression (PIZ, PXR24, B44, DWA, ...), tiled,
    deep or multi-part EXR raises ValueError.  It is not known whether the reference's example map
    (neon_photostudio_4k.exr) uses a supported compression; if it does not, convert it first, for example to .hdr or to an
    EXR with ZIP compression."""
    with open(path, 'rb') as f:
        data = f.read()
    if data[:4] == struct.pack('<i', 20000630):
        return _read_exr(data)
    if data[:2] == b'#?':
        return _read_hdr(data)
    raise ValueError(f'{path}: neither a Radiance .hdr nor an OpenEXR file')


def _read_hdr(data):
    pos = 0
    fmt = None
    while True:
        end = data.index(b'\n', pos)
        line = data[pos:end].strip()
        pos = end + 1
        if not line:
            break
        if line.startswith(b'FORMAT='):
            fmt = line[7:]
    if fmt not in (None, b'32-bit_rle_rgbe'):
        raise ValueError(f'.hdr pixel format {fmt.decode(errors="replace")} is not supported (only 32-bit_rle_rgbe)')
    end = data.index(b'\n', pos)
    tok = data[pos:end].split()
    pos = end + 1
    if len(tok) != 4 or tok[0] != b'-Y' or tok[2] != b'+X':
        raise ValueError(f'.hdr resolution line {b" ".join(tok).decode(errors="replace")} is not supported (only -Y H +X W)')
    H, W = int(tok[1]), int(tok[3])
    buf = np.frombuffer(data, np.uint8)
    rgbe = np.empty((H, W, 4), np.uint8)
    for y in range(H):
        if 8 <= W < 0x8000 and buf[pos] == 2 and buf[pos + 1] == 2 and (int(buf[pos + 2]) << 8 | int(buf[pos + 3])) == W:
            pos += 4
            for c in range(4):
                x = 0
                while x < W:
                    n = int(buf[pos])
                    if n > 128:
                        n -= 128
                        rgbe[y, x:x + n, c] = buf[pos + 1]
                        pos += 2
                    else:
                        rgbe[y, x:x + n, c] = buf[pos + 1:pos + 1 + n]
                        pos += 1 + n
                    if n == 0 or x + n > W:
                        raise ValueError('.hdr: corrupt run-length scanline')
                    x += n
        else:
            rgbe[y] = buf[pos:pos + 4 * W].reshape(W, 4)
            pos += 4 * W
    e = rgbe[..., 3].astype(np.int32)
    scale = np.where(e > 0, np.ldexp(1.0, e - 136), 0.0)
    return ((rgbe[..., :3] + 0.5) * scale[..., None]).astype(np.float32)


_EXR_COMPRESSION = {0: 'NONE', 1: 'RLE', 2: 'ZIPS', 3: 'ZIP', 4: 'PIZ', 5: 'PXR24', 6: 'B44', 7: 'B44A', 8: 'DWAA', 9: 'DWAB'}
_EXR_LINES = {0: 1, 2: 1, 3: 16}
_EXR_TYPES = {0: np.dtype('<u4'), 1: np.dtype('<f2'), 2: np.dtype('<f4')}


def _read_exr(data):
    version = struct.unpack_from('<i', data, 4)[0]
    if version & 0xff != 2:
        raise ValueError(f'OpenEXR version {version & 0xff} is not supported')
    for bit, what in ((0x200, 'tiled'), (0x800, 'deep'), (0x1000, 'multi-part')):
        if version & bit:
            raise ValueError(f'{what} OpenEXR files are not supported (scanline images only)')
    pos, attrs = 8, {}
    while data[pos] != 0:
        name_end = data.index(b'\0', pos)
        type_end = data.index(b'\0', name_end + 1)
        name, typ = data[pos:name_end].decode(), data[name_end + 1:type_end].decode()
        size = struct.unpack_from('<i', data, type_end + 1)[0]
        attrs[name] = (typ, data[type_end + 5:type_end + 5 + size])
        pos = type_end + 5 + size
    pos += 1
    comp = attrs['compression'][1][0]
    if comp not in _EXR_LINES:
        raise ValueError(f'OpenEXR compression {_EXR_COMPRESSION.get(comp, comp)} is not supported (NONE, ZIPS or ZIP only)')
    channels, raw, p = [], attrs['channels'][1], 0
    while raw[p] != 0:
        e = raw.index(b'\0', p)
        ptype, _, _, _, _, xs, ys = struct.unpack_from('<iBBBBii', raw, e + 1)
        if xs != 1 or ys != 1:
            raise ValueError('subsampled OpenEXR channels are not supported')
        channels.append((raw[p:e].decode(), _EXR_TYPES[ptype]))
        p = e + 1 + 16
    names = [c[0] for c in channels]
    if not all(c in names for c in 'RGB'):
        raise ValueError(f'OpenEXR file has channels {names}; R, G and B are needed')
    x0, y0, x1, y1 = struct.unpack('<4i', attrs['dataWindow'][1])
    W, H = x1 - x0 + 1, y1 - y0 + 1
    lines = _EXR_LINES[comp]
    n_chunks = (H + lines - 1) // lines
    offsets = np.frombuffer(data, '<u8', n_chunks, pos)
    line_bytes = sum(W * dt.itemsize for _, dt in channels)
    out = {c: np.zeros((H, W), np.float32) for c in 'RGB'}
    for off in offsets:
        y, size = struct.unpack_from('<ii', data, int(off))
        block = data[int(off) + 8:int(off) + 8 + size]
        n = min(lines, y1 + 1 - y)
        if comp != 0 and size < n * line_bytes:
            t = np.frombuffer(zlib.decompress(block), np.uint8).astype(np.int64)
            t[1:] -= 128
            t = (np.cumsum(t) & 0xff).astype(np.uint8)
            half = (t.size + 1) // 2
            block = np.empty_like(t)
            block[0::2], block[1::2] = t[:half], t[half:]
            block = block.tobytes()
        p = 0
        for r in range(n):
            for c, dt in channels:
                vals = np.frombuffer(block, dt, W, p)
                p += W * dt.itemsize
                if c in out:
                    out[c][y - y0 + r] = vals.astype(np.float32)
    return np.stack([out['R'], out['G'], out['B']], -1)


def env_tables(env):
    """Importance-sampling tables of an environment map [H,W,3] (row 0 at the top), computed in float64 and returned in the
    float32 layout nero_relight_render reads, rows from the bottom (v = 0) up:
      env [H,W,4] radiance, p [H,W] texel probabilities proportional to luminance * sin(polar angle at the row centre)
      (uniform in solid angle for a black map), cdf_rows [H+1] marginal CDF over rows, cdf_cols [H,W+1] CDF within each row."""
    e = np.asarray(env, np.float64)[::-1]
    H, W = e.shape[:2]
    ce = np.cos(((np.arange(H) + 0.5) / H - 0.5) * np.pi)[:, None]
    lum = np.maximum(0.2126 * e[..., 0] + 0.7152 * e[..., 1] + 0.0722 * e[..., 2], 0.0)
    w = np.nan_to_num(lum) * ce
    if not w.sum() > 0:
        w = np.broadcast_to(ce, (H, W)).copy()
    row = w.sum(1)
    cdf_rows = np.concatenate([[0.0], np.cumsum(row) / row.sum()])
    cdf_rows[-1] = 1.0
    safe = np.where(row > 0, row, 1.0)[:, None]
    cdf_cols = np.concatenate([np.zeros((H, 1)), np.cumsum(w, 1) / safe], 1)
    cdf_cols[row == 0] = np.linspace(0.0, 1.0, W + 1)
    cdf_cols[:, -1] = 1.0
    env4 = np.zeros((H, W, 4), np.float32)
    env4[..., :3] = e
    return {'env': env4, 'p': (w / w.sum()).astype(np.float32), 'cdf_rows': cdf_rows.astype(np.float32),
            'cdf_cols': cdf_cols.astype(np.float32)}


# ------------------------------------------------------------------------------------------------ cameras
def relight_poses(num, azimuth=0.0, elevation=45.0, cam_dist=3.0):
    """World -> camera poses [num,3,4] (OpenCV axes) of generate_relghting_poses (blender_utils.py:101-116) as placed in the
    Blender scene by set_camera_by_pose (blender_utils.py:48-68): camera centre dist (cos az cos el, sin az cos el, sin el),
    looking at the origin with up +z, az = azimuth + linspace(-90, 90, num) degrees."""
    az = np.deg2rad(azimuth) + np.linspace(-np.pi / 2, np.pi / 2, num)
    el = np.deg2rad(elevation)
    c = cam_dist * np.stack([np.cos(az) * np.cos(el), np.sin(az) * np.cos(el), np.full_like(az, np.sin(el))], -1)
    z = -c / np.linalg.norm(c, axis=-1, keepdims=True)
    up = np.asarray([0.0, 0.0, 1.0])
    y = -(up - (z @ up)[:, None] * z)
    y /= np.linalg.norm(y, axis=-1, keepdims=True)
    x = np.cross(y, z)
    R = np.stack([x, y, z], 1)
    t = -np.einsum('nij,nj->ni', R, c)
    return np.concatenate([R, t[..., None]], -1)


def blender_default_K(h, w):
    """Intrinsics of Blender's default camera (50 mm lens, 36 mm sensor, sensor fit auto) at h x w pixels."""
    f = 50.0 / 36.0 * max(h, w)
    return np.asarray([[f, 0.0, w / 2.0], [0.0, f, h / 2.0], [0.0, 0.0, 1.0]])


# ------------------------------------------------------------------------------------------------ output
def to_rgba8(img):
    """[h,w,4] premultiplied linear RGB + alpha -> uint8 RGBA with straight alpha and the plain sRGB transfer, clamped."""
    img = np.asarray(img, np.float64)
    a = img[..., 3:4]
    rgb = np.where(a > 0, img[..., :3] / np.where(a > 0, a, 1.0), 0.0)
    srgb = np.clip(linear_to_srgb(rgb), 0.0, 1.0)
    return np.round(np.concatenate([srgb, np.clip(a, 0.0, 1.0)], -1) * 255.0).astype(np.uint8)


def write_png(path, img):
    """Write uint8 [h,w,3] or [h,w,4] as an 8-bit RGB or RGBA PNG (stdlib zlib; no image library needed)."""
    img = np.ascontiguousarray(img, np.uint8)
    if img.ndim != 3 or img.shape[2] not in (3, 4):
        raise ValueError(f'expected [h,w,3] or [h,w,4] uint8, got {img.shape}')
    h, w, c = img.shape
    raw = np.concatenate([np.zeros((h, 1), np.uint8), img.reshape(h, c * w)], 1).tobytes()   # filter type 0 per row

    def chunk(tag, body):
        return struct.pack('>I', len(body)) + tag + body + struct.pack('>I', zlib.crc32(tag + body) & 0xffffffff)
    with open(path, 'wb') as f:
        f.write(b'\x89PNG\r\n\x1a\n' + chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, 6 if c == 4 else 2, 0, 0, 0)) +
                chunk(b'IDAT', zlib.compress(raw, 6)) + chunk(b'IEND', b''))


def write_png_rgba(path, rgba):
    """Write uint8 [h,w,4] as an 8-bit RGBA PNG."""
    rgba = np.asarray(rgba)
    if rgba.ndim != 3 or rgba.shape[2] != 4:
        raise ValueError(f'expected [h,w,4] uint8, got {rgba.shape}')
    write_png(path, rgba)


# ------------------------------------------------------------------------------------------------ renderer
class Relighter:
    """A mesh with per-vertex or UV-textured materials under one environment map, resident on the GPU.

    verts [V,3] (scene coordinates), tris [T,3]; materials = linear (decoded) {'metallic' [V,1], 'roughness' [V,1],
    'albedo' [V,3]} (see load_materials) or a UVMaterials (see load_textured_obj); env [H,W,3] radiance (load_env_map);
    geometry_type 'schlick' or 'ggx_smith'."""

    def __init__(self, verts, tris, materials, env, geometry_type='schlick', device='cuda'):
        import torch
        from . import ops
        ops.require_cuda(device, 'Relighter')
        if geometry_type not in ('schlick', 'ggx_smith'):
            raise ValueError(f'geometry_type {geometry_type!r}: expected schlick or ggx_smith')
        self.dev = torch.device(device)
        self.verts = np.ascontiguousarray(verts, np.float32)
        self.tris = np.ascontiguousarray(tris, np.int32)
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.dev)
        self.uv = materials if isinstance(materials, UVMaterials) else None
        if self.uv is not None:
            if self.uv.ft.shape != self.tris.shape:
                raise ValueError(f'ft has shape {self.uv.ft.shape} for tris of shape {self.tris.shape}')
            self.vmat, self.vmat_d = None, None
            self.tex = self.uv.texel_table()
            self.vt_d, self.ft_d, self.tex_d = up(self.uv.vt), up(self.uv.ft), up(self.tex)
        else:
            self.vmat = vertex_material_table(materials)
            if self.vmat.shape[0] != self.verts.shape[0]:
                raise ValueError(f'{self.vmat.shape[0]} material rows for {self.verts.shape[0]} vertices')
        self.ggx_smith = 1 if geometry_type == 'ggx_smith' else 0
        nodes, tri, ids = ops.bvh_build(self.verts, self.tris)
        self.nodes, self.tri, self.tri_ids, self.faces = up(nodes), up(tri), up(ids), up(self.tris)
        if self.uv is None:
            self.vmat_d = up(self.vmat)
        self.tables = env_tables(env)
        self.env_h, self.env_w = self.tables['p'].shape
        self.env_d = {k: up(v) for k, v in self.tables.items()}
        self.rays = torch.zeros(1, dtype=torch.int64, device=self.dev)

    def _params(self, pose, K, h, w, max_bounces, seed, accum):
        from . import ops
        e = self.env_d
        q = ops.RelightParams().set(nodes=self.nodes, tris=self.tri, tri_ids=self.tri_ids, faces=self.faces, vmat=self.vmat_d, env=e['env'],
                                    env_p=e['p'], cdf_rows=e['cdf_rows'], cdf_cols=e['cdf_cols'], accum=accum, rays=self.rays)
        q.pose[:] = [float(x) for x in np.asarray(pose, np.float64).reshape(12)]
        K = np.asarray(K, np.float64)
        q.K[:] = [K[0, 0], K[1, 1], K[0, 2], K[1, 2]]
        q.env_w, q.env_h, q.width, q.height = self.env_w, self.env_h, w, h
        q.max_bounces, q.ggx_smith, q.seed = max_bounces, self.ggx_smith, seed & 0xffffffff
        return q

    def render(self, pose, K, h, w, spp, max_bounces=4, seed=0, spp_per_launch=16, denoise=False):
        """One image -> CUDA float32 [h,w,4]: linear RGB premultiplied by coverage, alpha = fraction of camera samples that hit
        the mesh.  pose: world -> camera [3,4] (OpenCV axes), K: [3,3] pinhole intrinsics.  The samples are launched in
        chunks of spp_per_launch; the result does not depend on the chunking.  self.rays accumulates the rays traced.
        denoise=True traces with the feature buffers and returns the frame filtered by nero_b200.denoise.denoise (default
        settings; focal K[0,0]) in the same layout, with the same alpha."""
        import torch
        from . import ops
        if denoise:
            from .denoise import denoise as run_denoise
            accum, aov = self.render_sums(pose, K, h, w, spp, max_bounces, seed, spp_per_launch)
            return run_denoise(accum, aov, spp, float(np.asarray(K, np.float64)[0, 0]))
        if spp < 1 or max_bounces < 1 or spp_per_launch < 1:
            raise ValueError('spp, max_bounces and spp_per_launch must be positive')
        accum = torch.zeros(h * w, 4, device=self.dev)
        q = self._params(pose, K, h, w, max_bounces, seed, accum)
        for s0 in range(0, spp, spp_per_launch):
            q.spp0, q.spp = s0, min(spp_per_launch, spp - s0)
            if self.uv is None:
                ops.K('nero_relight_render', q)
            else:
                ops.K('nero_relight_render_textured', q, self.vt_d, self.ft_d, self.vt_d.shape[0], self.tex_d, self.tex.shape[1],
                      self.tex.shape[0])
        return (accum / spp).reshape(h, w, 4)

    def render_sums(self, pose, K, h, w, spp, max_bounces=4, seed=0, spp_per_launch=16):
        """The samples of render() traced by the AOV instances -> (accum [h,w,4], aov [h,w,16]) CUDA float32 sums over the
        samples: accum holds the bits render() divides by spp, aov the denoiser's feature sums (include/nero_denoise.h)."""
        import torch
        from . import ops
        from .denoise import AOV
        if spp < 1 or max_bounces < 1 or spp_per_launch < 1:
            raise ValueError('spp, max_bounces and spp_per_launch must be positive')
        accum = torch.zeros(h * w, 4, device=self.dev)
        aov = torch.zeros(h * w, AOV, device=self.dev)
        q = self._params(pose, K, h, w, max_bounces, seed, accum)
        for s0 in range(0, spp, spp_per_launch):
            q.spp0, q.spp = s0, min(spp_per_launch, spp - s0)
            if self.uv is None:
                ops.K('nero_relight_render_aov', q, aov)
            else:
                ops.K('nero_relight_render_textured_aov', q, self.vt_d, self.ft_d, self.vt_d.shape[0], self.tex_d, self.tex.shape[1],
                      self.tex.shape[0], aov)
        return accum.reshape(h, w, 4), aov.reshape(h, w, AOV)
