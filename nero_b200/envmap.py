"""Export of the learned environment light as an equirectangular HDR map on the GPU.

Reference being replaced (paths relative to the reference repository):
  network/field.py:836-854   MCShadingNetwork.predict_outer_lights   stage II: outer_light(IDE(d, 0) [| IDE(sphere point, 0)])
  network/field.py:554-589   AppShadingNetwork outer_light calls     stage I:  outer_light(IDE(d, k) [| IDE(sphere dir, k)])
  network/field.py:1020-1047 MCShadingNetwork.predict_outer_lights_pts / get_env_light (an unused 2:1 preview in another
                             convention; the map here is the one nero_b200.relight reads)

The protocol:
  * The map is width x height texels, row 0 at the top (load_env_map's layout), in relight's convention
    (nero_b200/relight.py): u = 0.5 - atan2(d_y, d_x) / 2pi, v = 0.5 + atan2(d_z, hypot(d_x, d_y)) / pi, v = 0 at the bottom.
    Each texel is sampled at ssaa x ssaa sub-sample centres, u = (x + (a + 1/2) / ssaa) / width, v = (j + (b + 1/2) / ssaa) /
    height with j = height - 1 - y; the direction is relight's inverse mapping in fp64, rotated by `frame` (fp64) and rounded to
    fp32 once (include/nero_envmap.h).  `frame` = MESH_TRANS^T gives the map tools/relight.py --trans expects: the scene
    direction d maps to the network's direction MESH_TRANS^T d.
  * The radiance of a sub-sample is the checkpoint's outer_light MLP on the reference's encoding of that direction (the
    fused chain, fp32 accumulation of split-bf16 products, ACT_EXPCLAMP at the config's light_exp_max):
      stage II (kappa_inv = 0):  [IDE(d, 0)], or with sphere_direction [IDE(d, 0) | IDE(c' + d t, 0)], c' = 0.999 c when
                                 |c| > 0.999, t = get_sphere_intersection(c', d), not normalised;
      stage I (kappa_inv = k):   [IDE(d, k)], or with sphere_direction [IDE(d, k) | IDE(normalize(offset_points_to_sphere(c)
                                 + d t), k)].  kappa_inv = 1 is the diffuse light of stage I, smaller values its pre-filtered
                                 specular light at roughness kappa_inv.
    c is one fixed point (`center`, the origin by default): a sphere_direction light depends on where it is seen from.
  * A texel is the solid-angle-weighted mean of its sub-samples, weight cos(elevation), summed in fp64 in sub-sample order and
    rounded to fp32: bit-identical from run to run and for any batch size.
  * Not in the map: the capturer's pose-dependent "human light" of real scenes and stage II's inner (indirect) light.
  * Files: Radiance .hdr (RGBE, new-style run-length scanlines, -Y H +X W), scanline OpenEXR (float, NONE or ZIP) and an
    8-bit sRGB PNG preview, clamped.
"""
import struct
import zlib

import numpy as np

MAX_ROWS = 1 << 19                # sub-sample rows per chain launch: ~3.7 KB of workspace per row (144-wide input), ~1.9 GB
STAGE1_KAPPA = (0.0, 0.1, 0.25, 0.5, 1.0)
_SPHERE = {None: 0, 'stage1': 1, 'stage2': 2}


def trans_frame(trans):
    """The frame of tools/relight.py --trans (MESH_TRANS^T: scene direction -> network direction), or None."""
    from .relight import MESH_TRANS
    return np.ascontiguousarray(MESH_TRANS.T) if trans else None


def _sphere_mode(sphere):
    if sphere not in _SPHERE:
        raise ValueError(f"sphere {sphere!r}: expected None, 'stage1' or 'stage2'")
    return _SPHERE[sphere]


def _check_size(width, height, ssaa):
    if width < 1 or height < 1 or not 1 <= ssaa <= 16:
        raise ValueError(f'a {width} x {height} map at ssaa {ssaa}: sizes must be positive and ssaa in [1, 16]')


def _frame_tensor(frame, dev):
    import torch
    if frame is None:
        return None
    f = np.asarray(frame, np.float64)
    if f.shape != (3, 3):
        raise ValueError(f'frame must be 3x3, got {f.shape}')
    return torch.from_numpy(np.ascontiguousarray(f.reshape(9))).to(dev)


def env_rows(row0, n, width, height, ssaa, *, kappa_inv=0.0, sphere=None, center=(0.0, 0.0, 0.0), frame=None, device='cuda'):
    """The MLP input rows [row0, row0 + n) -> (A [n, 128 or 192] CUDA float32, directions [n, 3] CUDA float32)."""
    import torch
    from . import ops
    from .engine import upload_ide_table
    ops.require_cuda(device, 'env_rows')
    _check_size(width, height, ssaa)
    mode = _sphere_mode(sphere)
    upload_ide_table()
    A = torch.empty(n, 192 if mode else 128, device=device)
    dirs = torch.empty(n, 3, device=device)
    F = _frame_tensor(frame, device)
    c = [float(x) for x in center]
    ops.K('nero_env_rows', row0, n, width, height, ssaa, F, float(kappa_inv), mode, c[0], c[1], c[2], A, A.shape[1], dirs)
    return A, dirs


class OuterLight:
    """The outer-light MLP of a checkpoint prepared for forward-only evaluation on environment maps.

    outer_light: the PredictorParams of MCShadingParams.outer_light (stage II) or ShadingParams.outer_light (stage I), on a
    CUDA device; its own operand images are built here (the training engines' copies are neither read nor touched)."""

    def __init__(self, outer_light, exp_max, sphere=None):
        from . import ops
        from .engine import Predictor, upload_ide_table
        self.dev = outer_light.layers()[0].weight_v.device
        ops.require_cuda(self.dev, 'outer_light_map')
        self.mode = _sphere_mode(sphere)
        self.k = 144 if self.mode else 72
        k_in = outer_light.layers()[0].weight_v.shape[1]
        if k_in != self.k:
            raise ValueError(f'outer_light reads {k_in} columns but sphere={sphere!r} encodes {self.k}')
        upload_ide_table()
        self.exp_max = float(exp_max)
        self.pred = Predictor(outer_light, self.dev, 3, ops.ACT_EXPCLAMP, self.exp_max, k_layout=self.k, t_cols=(0, self.k))
        self.lda = self.pred.layers[0].k_chunks * 64
        self.ws, self.cap = None, 0

    def _alloc(self, rows):
        import torch
        if self.cap < rows:
            self.ws = dict(A=torch.empty(rows, self.lda, device=self.dev), OUT=torch.empty(rows, 4, device=self.dev))
            self.cap = rows

    def _chain(self, n):
        from .ops import Mat, chain, chain_layer as CL, EK_BIAS_RELU, EK_BIAS_GENERIC, ACT_EXPCLAMP
        L = self.pred.layers
        chain(Mat(self.ws['A']), L[0].k_valid,
              [CL(L[0], EK_BIAS_RELU, 256), CL(L[1], EK_BIAS_RELU, 256), CL(L[2], EK_BIAS_RELU, 256),
               CL(L[3], EK_BIAS_GENERIC, 3, save=Mat(self.ws['OUT']), act=ACT_EXPCLAMP, act_param=self.exp_max)], None, n,
              tag='envmap_outer_light')

    def map(self, width, height, ssaa, kappa_inv=0.0, center=(0.0, 0.0, 0.0), frame=None, max_rows=MAX_ROWS):
        """-> CUDA float32 [height, width, 3] radiance, row 0 at the top."""
        import torch
        from . import ops
        _check_size(width, height, ssaa)
        s2 = ssaa * ssaa
        if self.mode == 2 and float(np.linalg.norm(np.asarray(center, np.float64))) >= 1.0:
            raise ValueError(f'stage II sees its sphere_direction light from inside the unit sphere; center {tuple(center)} is not')
        if max_rows < s2:
            raise ValueError(f'max_rows {max_rows} is less than one texel ({s2} sub-samples)')
        n_tex = width * height
        per = min(max_rows // s2, n_tex)            # whole texels per launch
        c = [float(x) for x in center]
        with torch.no_grad():
            self.pred.prep()
            self._alloc(per * s2)
            F = _frame_tensor(frame, self.dev)
            env = torch.empty(height, width, 3, device=self.dev)
            for t0 in range(0, n_tex, per):
                nt = min(per, n_tex - t0)
                n = nt * s2
                ops.K('nero_env_rows', t0 * s2, n, width, height, ssaa, F, float(kappa_inv), self.mode, c[0], c[1], c[2], self.ws['A'],
                      self.lda, None)
                self._chain(n)
                ops.K('nero_env_resolve', self.ws['OUT'], 4, t0, nt, width, height, ssaa, env)
        return env


def outer_light_map(outer_light, *, width, height, ssaa, kappa_inv=0.0, sphere=None, center=(0.0, 0.0, 0.0), frame=None, exp_max,
                    max_rows=MAX_ROWS):
    """The outer light of a checkpoint as a CUDA float32 [height, width, 3] map (see the module docstring).

    sphere: None (outer_light reads IDE(d) only), 'stage1' or 'stage2' (its sphere_direction input, at the fixed point
    `center`); frame: 3x3 applied to the map's directions before the query (trans_frame(True) for relight's --trans);
    max_rows bounds the sub-sample rows per launch and so the workspace."""
    return OuterLight(outer_light, exp_max, sphere).map(width, height, ssaa, kappa_inv, center, frame, max_rows)


def clamp_fraction(env, exp_max):
    """Fraction of texels whose largest channel is at the exp(exp_max) clamp of the MLP's output."""
    import torch
    top = torch.exp(torch.tensor(float(exp_max), dtype=torch.float32)).item()
    m = env.reshape(-1, 3).amax(1)
    return float((m >= top * (1 - 1e-6)).float().mean())


# ------------------------------------------------------------------------------------------------ files
def _host(env):
    env = env.detach().cpu().numpy() if hasattr(env, 'detach') else np.asarray(env)
    env = np.ascontiguousarray(env, np.float32)
    if env.ndim != 3 or env.shape[2] != 3:
        raise ValueError(f'expected an [H, W, 3] map, got {env.shape}')
    return env


def rgbe(env):
    """[H,W,3] float -> [H,W,4] uint8 Radiance RGBE: e = frexp(max channel) exponent, mantissa bytes floor(c / 2^e * 256);
    pixels whose largest channel is below 1e-32 (or not positive) are all zero."""
    e = np.asarray(env, np.float64)
    m = e.max(-1)
    ok = m > 1e-32
    mant, ex = np.frexp(np.where(ok, m, 1.0))
    scale = np.ldexp(256.0, -ex)
    q = np.clip(np.floor(np.maximum(e, 0.0) * scale[..., None]), 0, 255)
    out = np.zeros(e.shape[:2] + (4,), np.uint8)
    out[..., :3] = np.where(ok[..., None], q, 0).astype(np.uint8)
    out[..., 3] = np.where(ok, ex + 128, 0).astype(np.uint8)
    return out


def _rle(line):
    """New-style run-length encoding of one channel of one scanline (runs of 3 or more bytes, literals in chunks of 128)."""
    n = line.size
    cut = np.flatnonzero(line[1:] != line[:-1]) + 1
    starts = np.concatenate([[0], cut])
    lens = np.diff(np.concatenate([starts, [n]]))
    out = bytearray()
    lit = 0

    def literal(a, b):
        for p in range(a, b, 128):
            q = min(p + 128, b)
            out.append(q - p)
            out.extend(line[p:q].tobytes())
    for s, ln in zip(starts[lens >= 3].tolist(), lens[lens >= 3].tolist()):
        literal(lit, s)
        lit = s + ln
        v = int(line[s])
        while ln > 0:
            k = min(ln, 127)
            out += bytes((128 + k, v))
            ln -= k
    literal(lit, n)
    return bytes(out)


def write_hdr(path, env):
    """Radiance .hdr (32-bit_rle_rgbe, -Y H +X W, new-style run-length scanlines where the width allows it, flat otherwise)."""
    env = _host(env)
    H, W = env.shape[:2]
    px = rgbe(env)
    parts = [b'#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n', f'-Y {H} +X {W}\n'.encode()]
    rle = 8 <= W < 0x8000
    for y in range(H):
        if rle:
            parts.append(bytes((2, 2, W >> 8, W & 0xff)))
            parts.extend(_rle(np.ascontiguousarray(px[y, :, c])) for c in range(4))
        else:
            parts.append(px[y].tobytes())
    with open(path, 'wb') as f:
        f.write(b''.join(parts))


def _attr(name, typ, body):
    return name.encode() + b'\0' + typ.encode() + b'\0' + struct.pack('<i', len(body)) + body


def write_exr(path, env, compression='zip'):
    """Scanline OpenEXR with float R, G, B channels, NONE or ZIP (16-line blocks) compression."""
    env = _host(env)
    if compression not in ('none', 'zip'):
        raise ValueError(f"compression {compression!r}: expected 'none' or 'zip'")
    H, W = env.shape[:2]
    comp, lines = (3, 16) if compression == 'zip' else (0, 1)
    chlist = b''.join(c.encode() + b'\0' + struct.pack('<iBBBBii', 2, 0, 0, 0, 0, 1, 1) for c in 'BGR') + b'\0'
    box = struct.pack('<4i', 0, 0, W - 1, H - 1)
    header = (struct.pack('<ii', 20000630, 2) + _attr('channels', 'chlist', chlist) + _attr('compression', 'compression', bytes((comp,))) +
              _attr('dataWindow', 'box2i', box) + _attr('displayWindow', 'box2i', box) + _attr('lineOrder', 'lineOrder', b'\0') +
              _attr('pixelAspectRatio', 'float', struct.pack('<f', 1.0)) + _attr('screenWindowCenter', 'v2f', struct.pack('<ff', 0, 0)) +
              _attr('screenWindowWidth', 'float', struct.pack('<f', 1.0)) + b'\0')
    planar = np.ascontiguousarray(env[..., ::-1].transpose(0, 2, 1))     # [H, (B,G,R), W] = the scanline layout
    chunks = []
    for y in range(0, H, lines):
        raw = planar[y:y + lines].tobytes()
        data = raw
        if comp:
            b = np.frombuffer(raw, np.uint8)
            sp = np.concatenate([b[0::2], b[1::2]]).astype(np.int16)       # ZIP's byte split and delta predictor
            t = sp.copy()
            t[1:] = (sp[1:] - sp[:-1] + 128) & 0xff
            z = zlib.compress(t.astype(np.uint8).tobytes(), 6)
            if len(z) < len(raw):
                data = z
        chunks.append(struct.pack('<ii', y, len(data)) + data)
    offsets, pos = [], len(header) + 8 * len(chunks)
    for c in chunks:
        offsets.append(pos)
        pos += len(c)
    with open(path, 'wb') as f:
        f.write(header + struct.pack(f'<{len(offsets)}Q', *offsets) + b''.join(chunks))


def preview(env, exposure=0.0):
    """[H,W,3] uint8: the map times 2^exposure, plain sRGB transfer, clamped and rounded."""
    from .relight import linear_to_srgb
    e = _host(env).astype(np.float64) * 2.0 ** float(exposure)
    return np.round(np.clip(linear_to_srgb(e), 0.0, 1.0) * 255.0).astype(np.uint8)


def write_preview_png(path, env, exposure=0.0):
    from .relight import write_png
    write_png(path, preview(env, exposure))
