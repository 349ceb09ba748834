"""Meshes from SDF grids: marching cubes on the GPU (k_mcubes.cu) and a binary PLY writer.

`marching_cubes(volume, isovalue)` takes the arguments of `mcubes.marching_cubes` (PyMCubes, called by the reference at
network/field.py:1110) and returns the same kind of result: float64 [V,3] vertices in index space and int64 [T,3] triangles.
Differences from PyMCubes: the isovalue is rounded to float32 (the grid is float32); vertex positions are computed in float32;
connectivity inside cubes with an ambiguous face, and the diagonal chosen in quads, follow this project's generated table
(tools/gen_mc_tables.py), which separates the below corners of every ambiguous face.  Triangles are wound so that
cross(v1-v0, v2-v0) points to the below side (u <= iso: inside the solid for an SDF).  The output order is fixed by the input
alone: vertices by (grid point, axis) of their edge, triangles by cube, so the same volume gives bit-identical arrays.

`write_ply(path, verts, tris)` writes binary little-endian `float x y z` / `list uchar int vertex_indices`, readable by
`material.read_ply`.  It writes the arrays as given; trimesh's default processing (the reference exports through trimesh)
would also merge vertices at identical positions, which marching cubes only produces where a grid value equals the isovalue.
"""
import ctypes

import numpy as np
import torch

from . import ops

_TILE = 1024            # grid points per block of k_mcubes.cu (nblk in include/nero_b200.h)
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
    iso = ctypes.c_float(float(isovalue))
    with torch.cuda.device(dev):
        blk_cnt = torch.empty(2 * nblk, dtype=torch.int32, device=dev)
        blk_off = torch.empty(2 * nblk, dtype=torch.int64, device=dev)
        totals = torch.empty(2, dtype=torch.int64, device=dev)
        ops._check(ops.lib.nero_mcubes_count(ops._ptr(u), nx, ny, nz, iso, ops._ptr(blk_cnt), ops._ptr(blk_off), ops._ptr(totals),
                                             ops._stream()), 'nero_mcubes_count')
        ops.launch_count += 2
        V, T = totals.tolist()
        if V > _INT32_MAX or T > _INT32_MAX:
            raise RuntimeError(f'marching cubes: {V} vertices / {T} triangles do not fit int32 indices')
        verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
        tris = torch.empty(T, 3, dtype=torch.int32, device=dev)
        emap = torch.empty(3 * n if V else 0, dtype=torch.int32, device=dev)
        ops._check(ops.lib.nero_mcubes_emit(ops._ptr(u), nx, ny, nz, iso, ops._ptr(blk_off), ctypes.c_longlong(V), ctypes.c_longlong(T),
                                            ops._ptr(emap), ops._ptr(verts), ops._ptr(tris), ops._stream()), 'nero_mcubes_emit')
        ops.launch_count += (V > 0) + (T > 0)
    return verts, tris


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


def write_ply(path, verts, tris):
    """Binary little-endian PLY: `float x y z` per vertex, `list uchar int vertex_indices` per triangle."""
    verts = np.ascontiguousarray(verts, '<f4')
    tris = np.asarray(tris)
    if verts.ndim != 2 or verts.shape[1] != 3 or tris.ndim != 2 or tris.shape[1] != 3:
        raise ValueError(f'write_ply needs verts [V,3] and tris [T,3], got {verts.shape} and {tris.shape}')
    if tris.size and (tris.min() < 0 or tris.max() >= verts.shape[0]):
        raise ValueError('write_ply: triangle index out of range')
    face = np.empty(tris.shape[0], dtype=[('n', 'u1'), ('v', '<i4', (3,))])
    face['n'] = 3
    face['v'] = tris
    header = (f'ply\nformat binary_little_endian 1.0\nelement vertex {verts.shape[0]}\nproperty float x\nproperty float y\n'
              f'property float z\nelement face {tris.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n')
    with open(path, 'wb') as f:
        f.write(header.encode('ascii'))
        f.write(verts.tobytes())
        f.write(face.tobytes())
