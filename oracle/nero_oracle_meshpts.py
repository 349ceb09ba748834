"""numpy / fp64 restatement of the mesh clean-up and surface sampling of k_meshpts.cu (include/nero_meshpts.h), in the GPU's
order, so the kernels must match it bit for bit.

There is no reference code to pin against: the reference protocol cleans the mesh by hand in MeshLab and samples it with
CloudCompare, neither of which is in the reference tree.  This file states what the kernels compute instead:
  areas       a = 0.5 sqrt((cx cx + cy cy) + cz cz), c = (v1 - v0) x (v2 - v0), fp64 from the fp32 vertices
  crop        a triangle is kept iff its three vertices lie inside the sphere and / or the box (fp64 tests)
  components  triangles sharing a vertex index; label = smallest vertex index of the component
  selection   component area = np.add.at sum in ascending triangle index; kept iff area >= f * largest area
  compaction  kept triangles and referenced vertices in original order, indices remapped
  sampling    blocked fp64 prefix of the areas, counter-based hash, binary search, barycentric point
"""
import numpy as np

CHUNK = 256          # NERO_MESHPTS_CHUNK: triangles per sequential chunk of the cumulative areas
_M32 = np.uint64(0xffffffff)


def areas(verts, tris):
    """fp64 [T] triangle areas, 0 for a triangle with an index outside [0, V)."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    ok = ((t >= 0) & (t < v.shape[0])).all(1)
    tt = np.where(ok[:, None], t, 0)
    p0, p1, p2 = v[tt[:, 0]], v[tt[:, 1]], v[tt[:, 2]]
    e1, e2 = p1 - p0, p2 - p0
    cx = e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1]
    cy = e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2]
    cz = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    a = 0.5 * np.sqrt((cx * cx + cy * cy) + cz * cz)
    return np.where(ok, a, 0.0)


def crop(verts, tris, sphere=None, box=None):
    """bool [T]: indices in range and all three vertices inside the sphere (cx, cy, cz, r) and / or the box (x0, y0, z0,
    x1, y1, z1)."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    ok = ((t >= 0) & (t < v.shape[0])).all(1)
    inside = np.ones(v.shape[0], bool)
    if sphere is not None:
        c = np.asarray(sphere, np.float64)
        d = v - c[:3]
        inside &= (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2] <= c[3] * c[3]
    if box is not None:
        b = np.asarray(box, np.float64)
        inside &= ((v >= b[:3]) & (v <= b[3:])).all(1)
    tt = np.where(ok[:, None], t, 0)
    return ok & inside[tt].all(1)


def components(tris, keep, V):
    """int64 [T] label of each kept triangle (smallest vertex index of its component), V for the others.  Union-find by
    hooking each root to the smaller root of its neighbours, then jumping pointers to the roots, until no edge joins two
    trees."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)[np.asarray(keep, bool)]
    a = np.concatenate([t[:, 0], t[:, 0]])
    b = np.concatenate([t[:, 1], t[:, 2]])
    parent = np.arange(V, dtype=np.int64)
    while True:
        ra, rb = parent[a], parent[b]
        lo, hi = np.minimum(ra, rb), np.maximum(ra, rb)
        m = lo != hi
        if not m.any():
            break
        np.minimum.at(parent, hi[m], lo[m])
        while True:
            g = parent[parent]
            if (g == parent).all():
                break
            parent = g
    label = np.full(np.asarray(tris).reshape(-1, 3).shape[0], V, np.int64)
    label[np.asarray(keep, bool)] = parent[t[:, 0]]
    return label


def component_areas(area, label, V):
    """(labels [m] ascending, areas [m]): fp64 sums by np.add.at over the kept triangles in ascending triangle index."""
    kept = label < V
    labs = np.unique(label[kept])
    idx = np.searchsorted(labs, label[kept])
    s = np.zeros(labs.shape[0], np.float64)
    np.add.at(s, idx, np.asarray(area, np.float64)[kept])
    return labs, s


def select(comp_area, frac):
    """bool [m]: area >= frac * largest area."""
    return comp_area >= frac * comp_area.max()


def compact(verts, tris, tri_keep):
    """(verts [V',3] float32, tris [T',3] int32): kept triangles in order, referenced vertices in order, remapped."""
    t = np.asarray(tris, np.int64).reshape(-1, 3)[tri_keep]
    used = np.zeros(np.asarray(verts).shape[0], bool)
    used[t.ravel()] = True
    remap = np.cumsum(used) - 1
    return np.asarray(verts, np.float32)[used], remap[t].astype(np.int32)


def clean(verts, tris, sphere=None, box=None, min_component=0.0):
    """Everything clean_mesh computes: dict of area, keep (crop), label, comp_label, comp_area, comp_keep, verts, tris."""
    V = np.asarray(verts).shape[0]
    a = areas(verts, tris)
    keep = crop(verts, tris, sphere, box)
    label = components(tris, keep, V)
    labs, carea = component_areas(a, label, V)
    ck = select(carea, min_component)
    tri_keep = keep & np.isin(label, labs[ck])
    cv, ct = compact(verts, tris, tri_keep)
    return dict(area=a, keep=keep, label=label, comp_label=labs, comp_area=carea, comp_keep=ck, tri_keep=tri_keep, verts=cv,
                tris=ct)


def cdf(area):
    """Inclusive prefix of the areas: sequential sums per 256-triangle chunk, a sequential prefix of the chunk sums, and
    the chunk's offset added to each partial sum."""
    a = np.asarray(area, np.float64)
    T = a.shape[0]
    n = (T + CHUNK - 1) // CHUNK
    part = np.empty(T, np.float64)
    s = np.empty(n, np.float64)
    for c in range(n):
        part[c * CHUNK:(c + 1) * CHUNK] = np.cumsum(a[c * CHUNK:(c + 1) * CHUNK])
        s[c] = part[min((c + 1) * CHUNK, T) - 1]
    off = np.concatenate([[0.0], np.cumsum(s)[:-1]])
    return off[np.arange(T) // CHUNK] + part


def _mix(x):
    x = x ^ (x >> np.uint32(16))
    x = x * np.uint32(0x85ebca6b)
    x = x ^ (x >> np.uint32(13))
    x = x * np.uint32(0xc2b2ae35)
    return x ^ (x >> np.uint32(16))


def bits(seed, i, dim):
    """uint32 hash of (seed, sample index i (uint64 array), dim), the rl_mix chain of k_meshpts.cu."""
    i = np.asarray(i, np.uint64)
    h = _mix(np.full(i.shape, np.uint32(seed), np.uint32) * np.uint32(0x9e3779b9) + np.uint32(0x7f4a7c15))
    h = _mix(h ^ (i & _M32).astype(np.uint32))
    h = _mix(h ^ (i >> np.uint64(32)).astype(np.uint32))
    return _mix(h ^ np.uint32(dim))


def uniforms(seed, i):
    """(u0 with 53 random bits, r1, r2 with 32 bits each) of samples i."""
    h = [bits(seed, i, d).astype(np.float64) for d in range(4)]
    u0 = (np.floor(h[0] / 32.0) * 67108864.0 + np.floor(h[1] / 64.0)) * 2.0 ** -53
    return u0, h[2] * 2.0 ** -32, h[3] * 2.0 ** -32


def sample(verts, tris, n, seed=0, i0=0):
    """(points float64 [n,3], triangle of each sample) of samples i0 .. i0 + n - 1."""
    v = np.asarray(verts, np.float32).astype(np.float64)
    t = np.asarray(tris, np.int64).reshape(-1, 3)
    c = cdf(areas(verts, tris))
    i = np.arange(i0, i0 + n, dtype=np.uint64)
    u0, r1, r2 = uniforms(seed, i)
    tri = np.minimum(np.searchsorted(c, u0 * c[-1], side='right'), t.shape[0] - 1)
    s = np.sqrt(r1)
    b = np.stack([1.0 - s, s * (1.0 - r2), s * r2], 1)
    p = v[t[tri]]
    return (b[:, 0:1] * p[:, 0] + b[:, 1:2] * p[:, 1]) + b[:, 2:3] * p[:, 2], tri


# ------------------------------------------------------------------------------------------------ test meshes
def reversed_strip(n):
    """A strip of n triangles along x whose vertex indices run against its adjacency: triangle k (in order along the strip)
    uses vertices N-1-k, N-2-k, N-3-k of N = n + 2.  Hooking each triangle to the smaller root in triangle order builds one
    chain of depth ~N, the worst case for label propagation."""
    N = n + 2
    j = np.arange(N)
    pos = np.stack([(j // 2) * 0.01, (j % 2) * 0.01, np.zeros(N)], 1).astype(np.float32)
    verts = pos[::-1].copy()                 # vertex N-1-j sits at position j
    k = np.arange(n)
    tris = np.stack([N - 1 - k, N - 2 - k, N - 3 - k], 1).astype(np.int32)
    return verts, tris


def floater_scene(subdiv=2):
    """The two-sphere scene of nero_oracle_mat.test_scene plus two floaters: a small sphere near the object and a quad far
    from it (outside the unit sphere), with vertices that no triangle uses and a zero-area triangle on the main sphere."""
    import nero_oracle_mat as OM
    v, f = OM.test_scene(subdiv)
    fv, ff = OM.icosphere(1, 0.05)
    fv = fv + np.asarray([-0.1, 0.75, 0.2], np.float32)
    quad = np.asarray([[1.2, -1.0, -0.5], [1.6, -1.0, -0.5], [1.6, -0.6, -0.5], [1.2, -0.6, -0.5]], np.float32)
    spare = np.asarray([[5.0, 5.0, 5.0], [0.0, 0.0, 0.0]], np.float32)    # referenced by no triangle
    V0, V1 = v.shape[0], v.shape[0] + fv.shape[0]
    verts = np.concatenate([v, fv, quad, spare], 0)
    tris = np.concatenate([f, ff + V0, np.asarray([[0, 1, 2], [0, 2, 3]]) + V1,
                           np.asarray([[f[0, 0], f[0, 0], f[0, 1]]])], 0).astype(np.int32)   # last: zero area
    return np.ascontiguousarray(verts), np.ascontiguousarray(tris)
