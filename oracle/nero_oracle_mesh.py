"""CPU oracle for marching cubes (nero_b200/csrc/k_mcubes.cu, nero_b200.mesh.marching_cubes).

TEST INFRASTRUCTURE ONLY -- never imported by the product path.  A plain numpy restatement, in float64, of the algorithm the
kernels implement, with the same canonical order: one vertex per sign-change grid edge (p, p+e_a), a corner being below iff
u <= iso (iso rounded to float32, as the kernels see it), at p + t e_a with t = (iso-u(p)) / (u(p+e_a)-u(p)); vertices sorted
by (linear index of p, a); triangles sorted by the linear index of their cube, then by table order.  The case table is read
from nero_b200/csrc/mc_tables.cuh (the tests check the table itself through its properties), so this checks classification,
scan, interpolation, vertex sharing and ordering.

PARITY UNPINNED against PyMCubes (the reference's mcubes.marching_cubes, network/field.py:1110): PyMCubes is not available
here.  Its vertex set is the same by construction (one vertex per sign-change edge, linear interpolation); connectivity
inside cubes with an ambiguous face, and the diagonal chosen in quads, may differ from its hand-made table.
"""
import os
import re

import numpy as np

TABLES = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'nero_b200', 'csrc', 'mc_tables.cuh')


def load_tables(path=TABLES):
    """(edge corners [12,2], triangles per case [256], triangle edges [256, 3*max_tri] padded with -1) from mc_tables.cuh."""
    txt = open(path).read()

    def arr(name):
        body = re.search(name + r'\[[^=]*=\s*\{(.*?)\};', txt, re.S).group(1)
        body = re.sub(r'//[^\n]*', '', body)
        return np.array([int(x) for x in re.findall(r'-?\d+', body)], np.int64)
    max_tri = int(re.search(r'kMcMaxTri = (\d+)', txt).group(1))
    return arr('kMcEdgeCorner').reshape(12, 2), arr('kMcNumTri'), arr('kMcTri').reshape(256, 3 * max_tri)


def marching_cubes(u, iso=0.0, tables=None):
    """u [nx,ny,nz] -> (verts float64 [V,3] in index space, tris int64 [T,3]) in the kernels' canonical order."""
    edge_corner, ntri, tri = tables if tables is not None else load_tables()
    u = np.asarray(u, np.float32)
    assert u.ndim == 3 and min(u.shape) >= 2, u.shape
    shape = u.shape
    nx, ny, nz = shape
    iso32 = np.float32(iso)
    below = u <= iso32
    u64, iso64 = u.astype(np.float64), np.float64(iso32)
    keys, pos = [], []
    for a in range(3):
        lo = tuple(slice(0, n - 1) if d == a else slice(None) for d, n in enumerate(shape))
        hi = tuple(slice(1, n) if d == a else slice(None) for d, n in enumerate(shape))
        idx = np.nonzero(below[lo] != below[hi])
        u0 = u64[lo][idx]
        u1 = u64[hi][idx]
        p = np.stack(idx, -1).astype(np.float64)
        p[:, a] += (iso64 - u0) / (u1 - u0)
        keys.append(3 * np.ravel_multi_index(idx, shape).astype(np.int64) + a)
        pos.append(p)
    keys = np.concatenate(keys)
    order = np.argsort(keys, kind='stable')
    keys, verts = keys[order], np.concatenate(pos)[order]

    cs = np.zeros((nx - 1, ny - 1, nz - 1), np.int64)
    for c in range(8):
        ox, oy, oz = c & 1, c >> 1 & 1, c >> 2 & 1
        cs |= below[ox:ox + nx - 1, oy:oy + ny - 1, oz:oz + nz - 1].astype(np.int64) << c
    cube = np.nonzero(ntri[cs])                          # C order = ascending cube linear index
    cases = cs[cube]
    lin = np.ravel_multi_index(cube, shape).astype(np.int64)
    nt = ntri[cases]
    rep = np.repeat(np.arange(len(cases)), nt)
    slot = np.arange(rep.shape[0]) - np.repeat(np.cumsum(nt) - nt, nt)
    edges = tri[cases[rep][:, None], 3 * slot[:, None] + np.arange(3)[None, :]]
    c0 = edge_corner[:, 0]
    eoff = (c0 & 1) * ny * nz + (c0 >> 1 & 1) * nz + (c0 >> 2 & 1)
    ekey = 3 * (lin[rep][:, None] + eoff[edges]) + (edges >> 2)
    tris = np.searchsorted(keys, ekey)
    assert (keys[np.minimum(tris, len(keys) - 1)] == ekey).all(), 'a triangle uses an edge without a sign change'
    return verts.reshape(-1, 3), tris.astype(np.int64).reshape(-1, 3)
