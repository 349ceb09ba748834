"""numpy restatement of the ambient-occlusion bake (nero_b200/occlusion.py, k_occlusion.cu) for the tests.

  sampler   the rotated Hammersley set in float32, every operation rounded as numpy rounds it: r1, r2 bit for bit the
            kernel's.  The directions are nero_oracle_relight.sample_diffuse in float64 of those numbers.
  texels    the texel points, keys and flat outward normals: nero_oracle_texmap's rasteriser and fp32 interpolation (the
            kernel's bits), and for a detail mesh the normal bake's cage ray (nero_oracle_normalmap.cast in float64); the hit
            point there is o + t (-c) rounded once to float32 from the float64 t, so it may differ from the kernel's in the
            last bits.
  counts    the visibility test with nero_oracle_normalmap.cast in float64 with t in (0, distance), and per row the number of
            tie rays: rays cast flags as near ties, where fp32 and float64 arithmetic, or CUDA's cosf and numpy's cos, may
            decide differently.  A row whose cage ray is itself a near tie counts all its rays as ties.
TEST INFRASTRUCTURE ONLY.
"""
import numpy as np

import nero_oracle_normalmap as ON
import nero_oracle_relight as OR
import nero_oracle_texmap as OT

EPS = np.float32(OR.EPS)        # kRelightEps


def encode(counts, rays):
    """(510 c + N) div (2N) in integers."""
    c = np.asarray(counts, np.int64)
    return ((510 * c + rays) // (2 * rays)).astype(np.uint8)


def brev32(i):
    """__brev: the 32-bit reversal of each value."""
    i = np.asarray(i, np.uint64)
    r = np.zeros_like(i)
    for b in range(32):
        r |= ((i >> np.uint64(b)) & np.uint64(1)) << np.uint64(31 - b)
    return r


def sampler(seed, keys, rays):
    """-> (r1, r2) float32 [n, rays] for keys [n]."""
    keys = np.asarray(keys, np.int64)
    xi1 = OR.uniform(seed, keys, 0, 0, 0).astype(np.float32)[:, None]
    xi2 = OR.uniform(seed, keys, 0, 0, 1).astype(np.float32)[:, None]
    i = np.arange(rays, dtype=np.int64)
    a = (2 * i + 1).astype(np.float32) / np.float32(2 * rays) + xi1
    b = (brev32(i) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24) + xi2
    one = np.float32(1)
    return np.where(a < one, a, a - one), np.where(b < one, b, b - one)


def directions(normals, r1, r2):
    """Cosine-weighted directions about normals [n,3] -> float64 [n, rays, 3]."""
    n = np.asarray(normals, np.float32).astype(np.float64)[:, None, :]
    return OR.sample_diffuse(n, r1.astype(np.float64), r2.astype(np.float64))


def flat_normals32(e1, e2):
    """normalize(-cross(e1, e2)) in float32, component by component (the kernel's bits)."""
    e1, e2 = np.asarray(e1, np.float32), np.asarray(e2, np.float32)
    s = np.stack([-(e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]), -(e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]),
                  -(e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0])], -1)
    return ON.normalize32(s)


def counts(points, normals, occ_verts, occ_tris, rays, distance, seed, keys=None):
    """-> (counts [n] int64 unoccluded rays, ties [n] int64 tie rays).  A zero normal counts every ray, with no ties."""
    p, nrm = np.asarray(points, np.float32), np.asarray(normals, np.float32)
    n = p.shape[0]
    keys = np.arange(n) if keys is None else np.asarray(keys, np.int64)
    c, ties = np.full(n, rays, np.int64), np.zeros(n, np.int64)
    live = np.nonzero(nrm.any(1))[0]
    if live.size == 0:
        return c, ties
    o = p[live] + EPS * nrm[live]
    r1, r2 = sampler(seed, keys[live], rays)
    d = directions(nrm[live], r1, r2).reshape(-1, 3)
    oo = np.repeat(o.astype(np.float64), rays, axis=0)
    tri, _, _, _, tie = ON.cast(occ_verts, occ_tris, oo, d, float(np.float32(distance)))
    c[live] = rays - (tri >= 0).reshape(-1, rays).sum(1)
    ties[live] = tie.reshape(-1, rays).sum(1)
    return c, ties


def texels(verts, tris, vt, ft, width, height, dverts=None, dtris=None, cage_distance=0.02):
    """Per covered texel in row-major order -> dict texel / key [n], point / normal [n,3] float32 (where the rays start
    from, before the offset), hit [n] bool, cage_tie [n] bool, surface / cage [n,3] float32, owner [h,w]."""
    owner, _, bary = OT.rasterize(vt, ft, width, height)
    m = owner >= 0
    texel = np.nonzero(m.reshape(-1))[0]
    surface = OT.interpolate(verts, tris, owner, bary)[m]
    n = texel.size
    if dverts is None:
        V, T = np.asarray(verts, np.float32), np.asarray(tris, np.int64)[owner[m]]
        normal = flat_normals32(V[T[:, 1]] - V[T[:, 0]], V[T[:, 2]] - V[T[:, 0]])
        return dict(texel=texel, key=texel, point=surface, normal=normal, hit=np.ones(n, bool), cage_tie=np.zeros(n, bool),
                    surface=surface, cage=np.zeros((n, 3), np.float32), owner=owner)
    cage = ON.normalize32(OT.interpolate(ON.vertex_normals(verts, tris), tris, owner, bary)[m])
    d32 = np.float32(cage_distance)
    o = surface + d32 * cage
    tri, t, _, _, tie = ON.cast(dverts, dtris, o.astype(np.float64), -cage.astype(np.float64), 2.0 * float(d32))
    hit = (tri >= 0) & cage.any(1)
    point = np.where(hit[:, None], (o.astype(np.float64) - t[:, None] * cage.astype(np.float64)).astype(np.float32), surface)
    DV, DT = np.asarray(dverts, np.float32), np.asarray(dtris, np.int64)[np.maximum(tri, 0)]
    normal = np.where(hit[:, None], flat_normals32(DV[DT[:, 1]] - DV[DT[:, 0]], DV[DT[:, 2]] - DV[DT[:, 0]]), np.float32(0))
    return dict(texel=texel, key=texel, point=point, normal=normal.astype(np.float32), hit=hit, cage_tie=tie, surface=surface,
                cage=cage, owner=owner)


def bake_texels(verts, tris, vt, ft, width, height, dverts=None, dtris=None, rays=256, distance=0.25, seed=0, cage_distance=0.02):
    """texels() plus counts [n], ties [n] (all rays of a row with a cage tie) and img [h,w,5] uint8 (before inpainting)."""
    b = texels(verts, tris, vt, ft, width, height, dverts, dtris, cage_distance)
    occ = (verts, tris) if dverts is None else (dverts, dtris)
    c, ties = counts(b['point'], b['normal'], occ[0], occ[1], rays, distance, seed, b['key'])
    ties = np.where(b['cage_tie'], rays, ties)
    img = np.zeros((height * width, 5), np.uint8)
    img[b['texel'], :3] = encode(c, rays)[:, None]
    b.update(counts=c, ties=ties, img=img.reshape(height, width, 5))
    return b


def bake(verts, tris, vt, ft, size, dverts=None, dtris=None, ssaa=2, rays=256, distance=0.25, seed=0, cage_distance=0.02):
    """occlusion.bake restated -> (img uint8 [h0,w0,3], stats, bake_texels' dict)."""
    h0, w0 = (size, size) if np.isscalar(size) else size
    b = bake_texels(verts, tris, vt, ft, w0 * ssaa, h0 * ssaa, dverts, dtris, rays, distance, seed, cage_distance)
    img, _ = OT.inpaint(b['img'], b['owner'] >= 0)
    if ssaa == 2:
        img = OT.downsample(img)
    n = b['texel'].size
    hits = int(b['hit'].sum())
    return img[..., :3], {'covered': n, 'hits': hits, 'misses': n - hits, 'mean': float(b['counts'].sum()) / (n * rays)}, b
