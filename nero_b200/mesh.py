"""Meshes from SDF grids: marching cubes on the GPU (k_mcubes.cu) and a binary PLY writer.

`marching_cubes(volume, isovalue)` takes the arguments of `mcubes.marching_cubes` (PyMCubes, called by the reference at
network/field.py:1110) and returns the same kind of result: float64 [V,3] vertices in index space and int64 [T,3] triangles.
Differences from PyMCubes: the isovalue is rounded to float32 (the grid is float32); vertex positions are computed in float32;
connectivity inside cubes with an ambiguous face, and the diagonal chosen in quads, follow this project's generated table
(tools/gen_mc_tables.py), which separates the below corners of every ambiguous face.  Triangles are wound so that
cross(v1-v0, v2-v0) points to the below side (u <= iso: inside the solid for an SDF).  The output order is fixed by the input
alone: vertices by (grid point, axis) of their edge, triangles by cube, so the same volume gives bit-identical arrays.

`extract_sparse(query, axes, isovalue)` gives the arrays `marching_cubes_cuda` gives on the dense field, bit for bit, from field
values in a narrow band of bricks around the surface only (k_mcsparse.cu), so that 1024^3 and 2048^3 grids fit one card.

`write_ply(path, verts, tris)` writes binary little-endian `float x y z` / `list uchar int vertex_indices`, readable by
`material.read_ply`.  It writes the arrays as given; trimesh's default processing (the reference exports through trimesh)
would also merge vertices at identical positions, which marching cubes only produces where a grid value equals the isovalue.
"""
import time

import numpy as np
import torch

from . import ops

_TILE = 1024            # grid points per block of k_mcubes.cu (nblk in include/nero_b200.h); NERO_MCSPARSE_TILE too
_INT32_MAX = 2 ** 31 - 1


def _check_shape(shape):
    if len(shape) != 3 or min(shape) < 2:
        raise ValueError(f'marching cubes needs a 3-D volume with every dimension >= 2, got shape {tuple(shape)}')


def marching_cubes_cuda(u, isovalue=0.0):
    """Marching cubes of a CUDA tensor u [nx,ny,nz]: (verts float32 [V,3] in index space, tris int32 [T,3]) on u's device.
    Reads the two totals back once to size the outputs."""
    _check_shape(u.shape)
    ops.require_cuda(u.device, 'marching_cubes')
    u = u.to(torch.float32).contiguous()
    nx, ny, nz = u.shape
    n = nx * ny * nz
    nblk = ops.ceil_div(n, _TILE)
    dev = u.device
    with torch.cuda.device(dev):
        blk_cnt = torch.empty(2 * nblk, dtype=torch.int32, device=dev)
        blk_off = torch.empty(2 * nblk, dtype=torch.int64, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)
        ops.K('nero_mcubes_count', u, nx, ny, nz, isovalue, blk_cnt, blk_off, totals, launches=2)
        V, T = totals.tolist()
        if V > _INT32_MAX or T > _INT32_MAX:
            raise RuntimeError(f'marching cubes: {V} vertices / {T} triangles do not fit int32 indices')
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        tris = torch.empty(T, 3, dtype=torch.int32, device=dev)
        emap = torch.empty(3 * n if V else 0, dtype=torch.int32, device=dev)
        ops.K('nero_mcubes_emit', u, nx, ny, nz, isovalue, blk_off, V, T, emap, verts, tris, launches=(V > 0) + (T > 0))
    return verts, tris


_BRICKS = (4, 8, 16)
SPARSE_CHUNK_POINTS = 1 << 22     # points per call of `query`
_SQRT3_HALF = 0.8660254037844386


def _sparse_args(axes, brick):
    if brick not in _BRICKS:
        raise ValueError(f'extract_sparse: brick must be one of {_BRICKS}, got {brick!r}')
    if len(axes) != 3 or any(getattr(a, 'ndim', 0) != 1 for a in axes):
        raise ValueError('extract_sparse needs three 1-D axis tensors')
    _check_shape(tuple(int(a.shape[0]) for a in axes))


def extract_sparse(query, axes, isovalue, brick=8, lipschitz=2.0, outside=None, profile=False):
    """Marching cubes of the field `query` on the grid axes[0] x axes[1] x axes[2] without sampling the whole grid.

    query maps CUDA points [M,3] (float32) to values [M]; a point's value must not depend on the batch it comes in.  axes are
    three 1-D float32 CUDA tensors.  outside: None, or the constant the field takes at points with norm >= 1 (the test is
    torch.norm(points, dim=-1) >= 1.0 on the rows handed to `query`); it must lie above the isovalue for the seeding to see
    the surface this cut makes.  Returns (verts float32 [V,3] in index space, tris int32 [T,3], stats): the arrays
    marching_cubes_cuda returns for the dense field, bit for bit, in the same order.

    The grid is cut into bricks of brick^3 cubes.  The field is sampled at the brick corners; a brick is a seed if
    min |value - isovalue| over its corners is at most lipschitz * (sqrt(3)/2) * brick * h (h the largest grid spacing), or, with
    `outside`, if it straddles the unit sphere and min (value - isovalue) is at most that.  Seed bricks are sampled in full,
    then bricks are added across every brick face on which a grid edge changes side, until none is added, and the cube
    tables run on the listed bricks only.  The growth makes the result independent of `lipschitz` for every sheet of the
    surface that crosses a seed brick.
    Limit: a connected piece of surface that crosses no seed brick is not found -- a closed component smaller than a brick,
    between brick corners, in a field steeper than `lipschitz`.  Raise `lipschitz` or lower `brick` for such fields.

    stats: coarse_points, seed_bricks, grow_rounds, bricks_added, bricks, points_evaluated (bricks * (brick+1)^3: apron points
    shared by neighbours are evaluated by each), points_owned (bricks * brick^3), cubes_visited, vertices, triangles; with
    profile=True also 'ms', the host-clock milliseconds of the phases coarse / fill / grow / cubes / sort, each ended by a
    device synchronise."""
    _sparse_args(axes, brick)
    dev = axes[0].device
    ops.require_cuda(dev, 'extract_sparse')
    axes = [a.to(dev, torch.float32).contiguous() for a in axes]
    n = [int(a.shape[0]) for a in axes]
    B, P = brick, (brick + 1) ** 3
    nb = [ops.ceil_div(m - 1, B) for m in n]
    n_bricks_all, n_coarse = nb[0] * nb[1] * nb[2], (nb[0] + 1) * (nb[1] + 1) * (nb[2] + 1)
    if n_bricks_all > _INT32_MAX:
        raise RuntimeError(f'extract_sparse: {n_bricks_all} bricks do not fit int32 indices')
    ends = [(float(a[0]), float(a[-1])) for a in axes]
    h = max(abs(e1 - e0) / (m - 1) for (e0, e1), m in zip(ends, n))
    margin = float(lipschitz) * _SQRT3_HALF * B * h
    if not margin >= 0.0:
        raise ValueError(f'extract_sparse: lipschitz must be >= 0, got {lipschitz!r}')
    grid = (n[0], n[1], n[2], B)
    ms = {k: 0.0 for k in ('coarse', 'fill', 'grow', 'cubes', 'sort')}
    clock = [0.0]

    def lap(phase):
        if profile:
            torch.cuda.synchronize(dev)
            t = time.perf_counter()
            if phase is not None:
                ms[phase] += (t - clock[0]) * 1e3
            clock[0] = t

    def values(rows):
        val = query(rows)
        if val.shape != (rows.shape[0],):
            raise ValueError(f'extract_sparse: query returned shape {tuple(val.shape)} for {rows.shape[0]} points')
        return val.to(torch.float32)

    with torch.cuda.device(dev):
        lap(None)
        cval = torch.empty(n_coarse, dtype=torch.float32, device=dev)
        cout = torch.empty(n_coarse, dtype=torch.uint8, device=dev) if outside is not None else None
        for c0 in range(0, n_coarse, SPARSE_CHUNK_POINTS):
            m = min(SPARSE_CHUNK_POINTS, n_coarse - c0)
            rows = torch.empty(m, 3, dtype=torch.float32, device=dev)
            ops.K('nero_mcsparse_coarse_points', *axes, *grid, c0, m, rows)
            cval[c0:c0 + m] = values(rows)
            if cout is not None:
                cout[c0:c0 + m] = torch.norm(rows, dim=-1) >= 1.0
        flag = torch.empty(n_bricks_all, dtype=torch.uint8, device=dev)
        ops.K('nero_mcsparse_seed', cval, cout, *grid, isovalue, margin, flag)
        del cval, cout
        slot = torch.full((n_bricks_all,), -1, dtype=torch.int32, device=dev)
        nblk = ops.ceil_div(n_bricks_all, _TILE)
        blk_cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
        blk_off = torch.empty(nblk, dtype=torch.int64, device=dev)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        blist = torch.empty(0, dtype=torch.int32, device=dev)
        pool = torch.empty(0, P, dtype=torch.float32, device=dev)

        def append(blist):
            """the flagged bricks, in ascending order, appended to the list; one read of their count"""
            ops.K('nero_mcsparse_compact_count', flag, n_bricks_all, blk_cnt, blk_off, total, launches=2)
            add = int(total.item())
            if add:
                grown = torch.empty(blist.shape[0] + add, dtype=torch.int32, device=dev)
                grown[:blist.shape[0]] = blist
                ops.K('nero_mcsparse_compact_emit', flag, n_bricks_all, blk_off, blist.shape[0], grown, slot)
                blist = grown
            return blist, add

        blist, seeds = append(blist)
        lap('coarse')
        first, rounds, added = 0, 0, 0
        per_call = max(1, SPARSE_CHUNK_POINTS // P)
        while first < blist.shape[0]:
            last = blist.shape[0]
            new = torch.empty(last - first, P, dtype=torch.float32, device=dev)
            for j0 in range(first, last, per_call):
                m = min(per_call, last - j0)
                rows = torch.empty(m * P, 3, dtype=torch.float32, device=dev)
                ops.K('nero_mcsparse_brick_points', *axes, *grid, blist, j0, m, rows)
                val = values(rows)
                if outside is not None:
                    val = torch.where(torch.norm(rows, dim=-1) >= 1.0, torch.full_like(val, float(outside)), val)
                new[j0 - first:j0 - first + m] = val.view(m, P)
            del rows, val
            pool = torch.cat([pool, new]) if first else new
            del new
            lap('fill')
            ops.K('nero_mcsparse_grow', pool, blist, first, last - first, slot, *grid, isovalue, flag)
            blist, add = append(blist)
            first = last
            if add:
                rounds, added = rounds + 1, added + add
            lap('grow')
        del slot, flag
        nbr = blist.shape[0]
        stats = dict(coarse_points=n_coarse, seed_bricks=seeds, grow_rounds=rounds, bricks_added=added, bricks=nbr,
                     points_evaluated=nbr * P, points_owned=nbr * B ** 3, cubes_visited=0, vertices=0, triangles=0)
        if profile:
            stats['ms'] = ms
        verts = torch.empty(0, 3, dtype=torch.float32, device=dev)
        tris = torch.empty(0, 3, dtype=torch.int32, device=dev)
        if nbr == 0:
            return verts, tris, stats
        b = blist.long()
        ext = [torch.clamp(m - 1 - c * B, max=B) for m, c in zip(n, (b // (nb[1] * nb[2]), b // nb[2] % nb[1], b % nb[2]))]
        stats['cubes_visited'] = int((ext[0] * ext[1] * ext[2]).sum())
        cnt = torch.empty(2 * nbr, dtype=torch.int32, device=dev)
        off = torch.empty(2 * nbr, dtype=torch.int64, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)
        ops.K('nero_mcsparse_count', pool, blist, nbr, *grid, isovalue, cnt, off, totals, launches=2)
        V, T = totals.tolist()
        if V > _INT32_MAX or T > _INT32_MAX:
            raise RuntimeError(f'extract_sparse: {V} vertices / {T} triangles do not fit int32 indices')
        stats['vertices'], stats['triangles'] = V, T
        if V == 0:
            lap('cubes')
            return verts, tris, stats
        vkey = torch.empty(V, dtype=torch.int64, device=dev)
        vpos = torch.empty(V, 3, dtype=torch.float32, device=dev)
        tkey = torch.empty(T, dtype=torch.int64, device=dev)
        tedge = torch.empty(T, 3, dtype=torch.int64, device=dev)
        ops.K('nero_mcsparse_emit', pool, blist, nbr, *grid, isovalue, off, vkey, vpos, tkey, tedge)
        del pool
        lap('cubes')
        vkey, order = torch.sort(vkey)          # keys are unique, so the order does not depend on the sort's stability
        verts = vpos[order]
        del vpos
        if T:
            order = torch.sort(tkey)[1]
            tedge = tedge[order]
            del tkey, order
            tris = torch.empty(T, 3, dtype=torch.int32, device=dev)
            lap('sort')
            ops.K('nero_mcsparse_lookup', vkey, V, tedge, 3 * T, tris)
            lap('cubes')
        else:
            lap('sort')
    return verts, tris, stats


def marching_cubes(volume, isovalue):
    """Drop-in for mcubes.marching_cubes(volume, isovalue): volume is a numpy array or a CUDA tensor [nx,ny,nz];
    returns (float64 [V,3] vertices in index space, int64 [T,3] triangles) as numpy arrays."""
    if torch.is_tensor(volume):
        _check_shape(volume.shape)
        u = volume.detach()
        if u.device.type != 'cuda':
            u = u.cuda()
    else:
        arr = np.asarray(volume)
        _check_shape(arr.shape)
        u = torch.from_numpy(np.ascontiguousarray(arr, np.float32)).cuda()
    v, t = marching_cubes_cuda(u, isovalue)
    return v.cpu().numpy().astype(np.float64), t.cpu().numpy().astype(np.int64)


def write_ply(path, verts, tris, colors=None, quality=None):
    """Binary little-endian PLY: `float x y z` per vertex, `list uchar int vertex_indices` per triangle.  Optional per-vertex
    colors [V,3] uint8 (`uchar red green blue`) and quality [V] (`float quality`, the scalar field MeshLab and CloudCompare
    show) follow x y z in that order; without them the file is exactly the plain layout."""
    verts = np.ascontiguousarray(verts, '<f4')
    tris = np.asarray(tris)
    if verts.ndim != 2 or verts.shape[1] != 3 or tris.ndim != 2 or tris.shape[1] != 3:
        raise ValueError(f'write_ply needs verts [V,3] and tris [T,3], got {verts.shape} and {tris.shape}')
    if tris.size and (tris.min() < 0 or tris.max() >= verts.shape[0]):
        raise ValueError('write_ply: triangle index out of range')
    fields, props = [('p', '<f4', (3,))], 'property float x\nproperty float y\nproperty float z\n'
    if colors is not None:
        colors = np.asarray(colors)
        if colors.shape != verts.shape or colors.dtype != np.uint8:
            raise ValueError(f'write_ply: colors must be uint8 [{verts.shape[0]},3], got {colors.dtype} {colors.shape}')
        fields.append(('c', 'u1', (3,)))
        props += 'property uchar red\nproperty uchar green\nproperty uchar blue\n'
    if quality is not None:
        quality = np.asarray(quality)
        if quality.shape != (verts.shape[0],):
            raise ValueError(f'write_ply: quality must be [{verts.shape[0]}], got {quality.shape}')
        fields.append(('q', '<f4'))
        props += 'property float quality\n'
    vrec = np.empty(verts.shape[0], dtype=fields)
    vrec['p'] = verts
    if colors is not None:
        vrec['c'] = colors
    if quality is not None:
        vrec['q'] = quality
    face = np.empty(tris.shape[0], dtype=[('n', 'u1'), ('v', '<i4', (3,))])
    face['n'] = 3
    face['v'] = tris
    header = (f'ply\nformat binary_little_endian 1.0\nelement vertex {verts.shape[0]}\n{props}'
              f'element face {tris.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n')
    with open(path, 'wb') as f:
        f.write(header.encode('ascii'))
        f.write(vrec.tobytes())
        f.write(face.tobytes())
