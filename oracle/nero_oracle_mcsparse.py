"""CPU oracle for brick-wise marching cubes on a narrow band (nero_b200/csrc/k_mcsparse.cu, nero_b200.mesh.extract_sparse).

TEST INFRASTRUCTURE ONLY -- never imported by the product path.  A numpy restatement of the protocol on a callable field:
coarse pass at the brick corners, seeding by the Lipschitz test, filling the listed bricks, growth across brick faces with a
sign-change edge until no brick is added, then marching cubes per brick (nero_oracle_mesh.marching_cubes on the brick's
(B+1)^3 values gives its triangles), global int64 keys, and a sort by key.  The brick list has the kernels' order (seeds in
ascending brick index, then each round's additions in ascending index), so the statistics can be compared too.

`field(points [M,3] float32) -> values [M]`.  With dtype=np.float64 the vertices are computed as nero_oracle_mesh computes them
(the result equals its marching_cubes on the dense field exactly); with dtype=np.float32 as the kernels compute them.
"""
import numpy as np

import nero_oracle_mesh as OMesh

SQRT3_HALF = 0.8660254037844386
MAX_TRI = 5


def _points(axes, idx):
    return np.stack([np.asarray(axes[a], np.float32)[idx[a]] for a in range(3)], -1)


def dense_field(field, axes, outside=None):
    """The whole grid, with the override: what the dense path samples."""
    n = [len(a) for a in axes]
    idx = np.stack(np.meshgrid(*[np.arange(m) for m in n], indexing='ij'), -1).reshape(-1, 3).T
    pts = _points(axes, idx)
    val = np.asarray(field(pts), np.float32)
    if outside is not None:
        val = np.where(np.linalg.norm(pts, axis=-1) >= 1.0, np.float32(outside), val)
    return val.reshape(n)


def extract_sparse(field, axes, iso=0.0, brick=8, lipschitz=2.0, outside=None, dtype=np.float64, tables=None):
    """-> (verts dtype [V,3] in index space, tris int64 [T,3], stats) in the canonical order of nero_oracle_mesh."""
    if brick not in (4, 8, 16):
        raise ValueError(f'brick must be 4, 8 or 16, got {brick!r}')
    if len(axes) != 3 or any(np.ndim(a) != 1 or len(a) < 2 for a in axes):
        raise ValueError('three 1-D axes with at least 2 points each are needed')
    tables = tables if tables is not None else OMesh.load_tables()
    edge_corner, ntri, tri = tables
    axes = [np.asarray(a, np.float32) for a in axes]
    n = np.array([len(a) for a in axes])
    B, B1 = brick, brick + 1
    P = B1 ** 3
    nb = (n - 2) // B + 1
    iso32 = np.float32(iso)
    h = max(abs(float(a[-1]) - float(a[0])) / (len(a) - 1) for a in axes)
    margin = np.float32(float(lipschitz) * SQRT3_HALF * B * h)

    # 1. coarse pass: every B-th grid point and the last one per axis
    cidx = np.stack(np.meshgrid(*[np.minimum(np.arange(m + 1) * B, k - 1) for m, k in zip(nb, n)], indexing='ij'), -1)
    cpts = _points(axes, cidx.reshape(-1, 3).T)
    cval = np.asarray(field(cpts), np.float32).reshape(nb + 1)
    # 2. seeds
    d = np.stack([(cval - iso32)[q & 1:nb[0] + (q & 1), q >> 1 & 1:nb[1] + (q >> 1 & 1), q >> 2 & 1:nb[2] + (q >> 2 & 1)]
                  for q in range(8)])
    seed = np.abs(d).min(0) <= margin
    if outside is not None:
        out = (np.linalg.norm(cpts, axis=-1) >= 1.0).reshape(nb + 1)
        n_out = sum(out[q & 1:nb[0] + (q & 1), q >> 1 & 1:nb[1] + (q >> 1 & 1), q >> 2 & 1:nb[2] + (q >> 2 & 1)].astype(int)
                    for q in range(8))
        seed |= (n_out > 0) & (n_out < 8) & (d.min(0) <= margin)
    blist = list(np.nonzero(seed.reshape(-1))[0])
    n_seed = len(blist)
    listed = seed.copy()

    loc = np.stack(np.meshgrid(np.arange(B1), np.arange(B1), np.arange(B1), indexing='ij'), -1).reshape(-1, 3)

    def fill(b):
        o = np.array(np.unravel_index(b, nb)) * B
        g = np.minimum(o[None, :] + loc, n[None, :] - 1)
        pts = _points(axes, g.T)
        val = np.asarray(field(pts), np.float32)
        if outside is not None:
            val = np.where(np.linalg.norm(pts, axis=-1) >= 1.0, np.float32(outside), val)
        return val.reshape(B1, B1, B1)

    # 3. / 4. fill, and grow across faces with a sign-change edge
    pool, first, rounds, added = [], 0, 0, 0
    while first < len(blist):
        last = len(blist)
        new = set()
        for j in range(first, last):
            u = fill(blist[j])
            pool.append(u)
            bc = np.array(np.unravel_index(blist[j], nb))
            for a in range(3):
                for hi in (0, 1):
                    nc = bc.copy()
                    nc[a] += 1 if hi else -1
                    if nc[a] < 0 or nc[a] >= nb[a] or listed[tuple(nc)]:
                        continue
                    below = np.take(u, B if hi else 0, axis=a) <= iso32
                    if (below[1:] != below[:-1]).any() or (below[:, 1:] != below[:, :-1]).any():
                        new.add(int(np.ravel_multi_index(nc, nb)))
        first = last
        if new:
            rounds, added = rounds + 1, added + len(new)
            for b in sorted(new):
                blist.append(b)
                listed[np.unravel_index(b, nb)] = True

    # 5. cubes per brick
    vkeys, vpos, tkeys, tedges = [], [], [], []
    cubes = 0
    c0 = edge_corner[:, 0]
    for b, u in zip(blist, pool):
        o = np.array(np.unravel_index(b, nb)) * B
        e = np.minimum(B, n - 1 - o) + 1                       # real points of this brick per axis
        sub = u[:e[0], :e[1], :e[2]]
        cubes += int(np.prod(e - 1))
        _, lt = OMesh.marching_cubes(sub, iso32, tables)
        below = sub <= iso32
        # this brick's sign-change edges in the order of marching_cubes' vertices (local key), with their global keys
        lk, gk, own, pos = [], [], [], []
        for a in range(3):
            lo = tuple(slice(0, m - 1) if dd == a else slice(None) for dd, m in enumerate(sub.shape))
            hi = tuple(slice(1, m) if dd == a else slice(None) for dd, m in enumerate(sub.shape))
            idx = np.nonzero(below[lo] != below[hi])
            li = np.stack(idx, -1)
            gi = li + o[None, :]
            lk.append(3 * np.ravel_multi_index(idx, sub.shape).astype(np.int64) + a)
            gk.append(3 * np.ravel_multi_index(tuple(gi.T), n).astype(np.int64) + a)
            own.append(((li < B) | (gi == n[None, :] - 1)).all(-1))
            u0, u1 = sub[lo][idx], sub[hi][idx]
            p = gi.astype(dtype)
            if dtype == np.float32:
                p[:, a] += (iso32 - u0) / (u1 - u0)
            else:
                u0, u1 = u0.astype(np.float64), u1.astype(np.float64)
                p[:, a] += (np.float64(iso32) - u0) / (u1 - u0)
            pos.append(p)
        order = np.argsort(np.concatenate(lk), kind='stable')
        gk, own, pos = np.concatenate(gk)[order], np.concatenate(own)[order], np.concatenate(pos)[order]
        vkeys.append(gk[own])
        vpos.append(pos[own])
        # triangles: every cube of the sub-volume is owned; cube order = local linear index, as marching_cubes lists them
        cs = np.zeros(tuple(e - 1), np.int64)
        for c in range(8):
            ox, oy, oz = c & 1, c >> 1 & 1, c >> 2 & 1
            cs |= below[ox:ox + e[0] - 1, oy:oy + e[1] - 1, oz:oz + e[2] - 1].astype(np.int64) << c
        cube = np.nonzero(ntri[cs])
        nt = ntri[cs[cube]]
        assert nt.sum() == lt.shape[0]
        lin = np.ravel_multi_index(tuple((np.stack(cube, -1) + o[None, :]).T), n).astype(np.int64)
        rep = np.repeat(np.arange(len(nt)), nt)
        slot = np.arange(rep.shape[0]) - np.repeat(np.cumsum(nt) - nt, nt)
        tkeys.append(MAX_TRI * lin[rep] + slot)
        tedges.append(gk[lt])
    stats = dict(coarse_points=int(np.prod(nb + 1)), seed_bricks=n_seed, grow_rounds=rounds, bricks_added=added, bricks=len(blist),
                 points_evaluated=len(blist) * P, points_owned=len(blist) * B ** 3, cubes_visited=cubes, vertices=0, triangles=0)
    if not blist or sum(len(k) for k in vkeys) == 0:
        return np.zeros((0, 3), dtype), np.zeros((0, 3), np.int64), stats
    vkeys, vpos = np.concatenate(vkeys), np.concatenate(vpos)
    assert np.unique(vkeys).shape[0] == vkeys.shape[0], 'an edge has two owners'
    order = np.argsort(vkeys)
    vkeys, verts = vkeys[order], vpos[order]
    tkeys, tedges = np.concatenate(tkeys), np.concatenate(tedges).reshape(-1, 3)
    tedges = tedges[np.argsort(tkeys)]
    tris = np.searchsorted(vkeys, tedges)
    assert (vkeys[np.minimum(tris, len(vkeys) - 1)] == tedges).all(), 'a triangle uses an edge no listed brick owns'
    stats['vertices'], stats['triangles'] = int(verts.shape[0]), int(tris.shape[0])
    return verts.reshape(-1, 3), tris.astype(np.int64).reshape(-1, 3), stats
