"""numpy restatement of the UV texture-map export (nero_b200/texmap.py, nero_b200/csrc/k_texmap.cu) for the tests.

  rasterize     the uv rasteriser with the kernel's fixed-point rule: uv snapped to 1/256 texel (round half to even of
                u * width * 256), exact integer edge functions, the top-left rule for either winding, zero-area triangles own
                nothing; owner = smallest covering triangle id (-1 = uncovered), count = covering triangles, barycentrics
                w_i / area rounded to fp32.  It stands in for nvdiffrast's rasterize / interpolate in make_golden_texmap.py.
  interpolate   sum_i b_i attr[f_i] in fp32, ((b0 a0 + b1 a1) + b2 a2).
  encode        the reference's float64 linear_to_srgb, x 255, astype(uint8) (extract_materials_texture_map.py:130-133).
  inpaint       lines 136-149 with the kernel's tie rule: Manhattan-32 dilation, Manhattan-3 erosion (border unmasked),
                nearest search texel by squared distance, then by row-major index.
  downsample    (a + b + c + d + 2) >> 2, OpenCV's INTER_LINEAR on an exact 2x uint8 shrink.
  obj_text      lines 170-197, loop for loop.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np
from scipy import ndimage

RADIUS, ERODE = 32, 3


def snap(vt, width, height):
    vt = np.asarray(vt, np.float32).astype(np.float64)
    return np.rint(vt[:, 0] * width * 256.0).astype(np.int64), np.rint(vt[:, 1] * height * 256.0).astype(np.int64)


def rasterize(vt, ft, width, height):
    """-> owner [h,w] int64 (-1 uncovered), count [h,w] int32, bary [h,w,3] float32 of the owner."""
    sx, sy = snap(vt, width, height)
    ft = np.asarray(ft, np.int64)
    owner = np.full((height, width), -1, np.int64)
    count = np.zeros((height, width), np.int32)
    bary = np.zeros((height, width, 3), np.float32)
    for t in range(ft.shape[0]):
        x, y = sx[ft[t]], sy[ft[t]]
        area = (x[1] - x[0]) * (y[2] - y[0]) - (y[1] - y[0]) * (x[2] - x[0])
        if area == 0:
            continue
        s = 1 if area > 0 else -1
        x0 = max(0, -((-(x.min() - 128)) // 256)); x1 = min(width - 1, (x.max() - 128) // 256)
        y0 = max(0, -((-(y.min() - 128)) // 256)); y1 = min(height - 1, (y.max() - 128) // 256)
        if x0 > x1 or y0 > y1:
            continue
        py, px = np.mgrid[y0:y1 + 1, x0:x1 + 1]
        px, py = 256 * px + 128, 256 * py + 128
        w, inside = [], np.ones(px.shape, bool)
        for i in range(3):
            a, b = (i + 1) % 3, (i + 2) % 3
            dx, dy = x[b] - x[a], y[b] - y[a]
            wi = s * (dx * (py - y[a]) - dy * (px - x[a]))
            tl = (s * dy < 0) or (s * dy == 0 and s * dx > 0)
            inside &= (wi > 0) | ((wi == 0) & tl)
            w.append(wi)
        ys, xs = np.nonzero(inside)
        ys, xs = ys + y0, xs + x0
        count[ys, xs] += 1
        first = owner[ys, xs] < 0
        ys, xs = ys[first], xs[first]          # triangles are visited in ascending order: the first owner is the smallest
        owner[ys, xs] = t
        for i in range(3):
            bary[ys, xs, i] = (w[i][inside][first].astype(np.float64) / float(s * area)).astype(np.float32)
    return owner, count, bary


def interpolate(attr, faces, owner, bary):
    """[h,w,C] float32: the attribute interpolated at every covered texel, 0 elsewhere."""
    attr = np.asarray(attr, np.float32)
    faces = np.asarray(faces, np.int64)
    out = np.zeros(owner.shape + (attr.shape[1],), np.float32)
    m = owner >= 0
    f = faces[owner[m]]
    b = bary[m]
    out[m] = (b[:, 0:1] * attr[f[:, 0]] + b[:, 1:2] * attr[f[:, 1]]) + b[:, 2:3] * attr[f[:, 2]]
    return out


def linear_to_srgb(linear):
    eps = np.finfo(np.float32).eps
    srgb0 = 323 / 25 * linear
    srgb1 = (211 * np.maximum(eps, linear) ** (5 / 12) - 11) / 200
    return np.where(linear <= 0.0031308, srgb0, srgb1)


def encode(mat, mask):
    """mat [n,5] float32 of the covered texels in row-major order, mask [h,w] -> [h,w,5] uint8."""
    feats = np.zeros(mask.shape + (5,))
    feats[mask] = np.asarray(mat, np.float32)
    return (linear_to_srgb(feats) * 255).astype(np.uint8)


def inpaint(img, mask, chunk=4096):
    """-> (out [h,w,5] uint8, src [h,w] int64 row-major index of the copied texel, -1 elsewhere)."""
    h, w = mask.shape
    cross = ndimage.generate_binary_structure(2, 1)
    region = ndimage.binary_dilation(mask, cross, iterations=RADIUS) & ~mask
    search = mask & ~ndimage.binary_erosion(mask, cross, iterations=ERODE, border_value=0)
    sy, sx = np.nonzero(search)
    sidx = sy * w + sx
    iy, ix = np.nonzero(region)
    src = np.full((h, w), -1, np.int64)
    for c0 in range(0, iy.shape[0], chunk):
        d2 = (iy[c0:c0 + chunk, None] - sy[None]) ** 2 + (ix[c0:c0 + chunk, None] - sx[None]) ** 2
        key = d2.astype(np.int64) * (h * w) + sidx[None]      # squared distance first, then row-major index
        src[iy[c0:c0 + chunk], ix[c0:c0 + chunk]] = sidx[np.argmin(key, 1)]
    out = img.copy()
    m = src >= 0
    out[m] = img.reshape(-1, img.shape[-1])[src[m]]
    return out, src


def downsample(img):
    a = img.astype(np.uint32)
    return ((a[0::2, 0::2] + a[0::2, 1::2] + a[1::2, 0::2] + a[1::2, 1::2] + 2) >> 2).astype(np.uint8)


def obj_text(v_np, f_np, vt_np, ft_np, cas=0):
    """(obj, mtl) text as extract_materials_texture_map.py:170-197 writes them (the reference's map_Kd names a .jpg)."""
    obj = [f'mtllib mesh_{cas}.mtl \n']
    for v in v_np:
        obj.append(f'v {v[0]} {v[1]} {v[2]} \n')
    for v in vt_np:
        obj.append(f'vt {v[0]} {1 - v[1]} \n')
    obj.append('usemtl defaultMat \n')
    for i in range(len(f_np)):
        obj.append(f"f {f_np[i, 0] + 1}/{ft_np[i, 0] + 1} {f_np[i, 1] + 1}/{ft_np[i, 1] + 1} {f_np[i, 2] + 1}/{ft_np[i, 2] + 1} \n")
    mtl = (f'newmtl defaultMat \nKa 1 1 1 \nKd 1 1 1 \nKs 0 0 0 \nTr 1 \nillum 1 \nNs 0 \nmap_Kd feat0_{cas}.jpg \n')
    return ''.join(obj), mtl
