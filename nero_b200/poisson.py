"""Mesh an oriented point cloud on the GPU: screened Poisson surface reconstruction on a regular grid (k_poisson.cu,
include/nero_poisson.h), iso-surface extraction with marching_cubes_cuda and an optional trim of poorly sampled surface.

COLMAP ends its dense pipeline with poisson_mesher.  This module gives the custom-object workflow the same last step on the
GPU: dense_points.py --normals -> poisson_mesh.py.  It solves the same kind of energy as screened Poisson reconstruction
(Kazhdan and Hoppe 2013), but on a regular grid rather than an adaptive octree, so its result is not pinned to PoissonRecon's
or COLMAP's output.

Protocol
--------
  * Inputs (checked on the host before any kernel runs, ValueError otherwise): points [n,3] and normals [n,3] finite, n >= 16,
    every normal non-zero (renormalised in fp64, then rounded to fp32), resolution N in RESOLUTIONS, screen > 0, scale > 1,
    tol > 0, max_iters >= 1, trim >= 0.
  * Grid.  N = 2^k + 1 nodes per axis over the points' bounding cube scaled by `scale` about its centre: side = scale
    max(hi - lo), h = side / (N - 1), origin = (lo + hi) / 2 - side / 2 (fp64).  Grid coordinates q = fp32((p - origin) / h),
    clamped to [0, N - 1] (nero_poisson_keys), binned to cells and sorted by cell key with a stable sort (torch.sort); start
    gives each cell's first sample (nero_poisson_cell_starts).  Every later kernel reads the samples in that order.
  * sigma = 1.5 n / (occupied cells), in fp64, the samples per unit area (a plane crossing a unit cell has mean area 2/3 in
    it).  ws = fp32(screen / sigma), the screening weight per sample.
  * Normal field (nero_poisson_edge_splat): each normal component splatted with trilinear (hat) weights onto the midpoints of
    the edges along that axis, divided by fp32(sigma): v_e, a jump of 1 across a sampled surface.
  * Energy E(chi) = sum_e (chi_b - chi_a - v_e)^2 + ws sum_i chi(p_i)^2, chi(p) the trilinear interpolation of the nodes,
    edges only inside the grid (Neumann boundary).  Its minimiser solves A chi = G^T v, A = L + ws S^T S, L = G^T G the
    7-point Laplacian, S the interpolation at the samples (nero_poisson_rhs, nero_poisson_matvec).  screen > 0 makes A SPD.
  * Solver (pcg(), shared with the oracle): conjugate gradients on A from chi = 0, preconditioned by one V-cycle.  The V-cycle
    runs on s L + diag(d) per level: level 0 has s = 1 and d = ws diag(S^T S) (nero_poisson_node_splat); level l + 1 has
    N_(l+1) = (N_l - 1) / 2 + 1, s = 2^(l+1) (the rediscretised Laplacian) and d restricted from level l, down to N = 5.
    Each level: SMOOTH red-black Gauss-Seidel sweeps (red then black), the residual restricted by the transpose of
    trilinear prolongation (full weighting times 8), the coarse correction from zero, prolongation, then SMOOTH sweeps in
    reverse (black then red).  The coarsest level gets COARSE_SWEEPS / 2 forward and COARSE_SWEEPS / 2 reversed sweeps.  The
    cycle is symmetric, so PCG applies.  Vectors are fp32; dot products are fp64 block partials (nero_poisson_dot) summed by
    nero_align_reduce; alpha = rz / pAp and beta = rz' / rz in fp64 on the host, passed as fp32 to nero_poisson_update and
    nero_poisson_direction.  The run stops when |r| / |b| <= tol or after max_iters; the history of |r| / |b| is returned.
  * Iso value: the mean of chi at the samples, their fp64 sum in sorted order (nero_poisson_interp, nero_poisson_dot) over n.
    chi grows along the normals, so it is below the iso value inside; marching_cubes_cuda(chi, iso) then winds the
    triangles as extract_mesh.py's meshes are wound (cross(e1, e2) points inside).  Vertices are mapped back to world
    coordinates in fp64 (origin + h v) and rounded to fp32.
  * Trim: the splat density (sum of the samples' hat weights per node) restricted twice (to spacing 4h), interpolated at
    each vertex (at v / 4) and divided by its median over the vertices (those with a non-zero density).  With trim t > 0, triangles with a vertex below t are
    dropped (nero_poisson_trim) and unreferenced vertices removed by the ordered compaction of evaluate.clean_mesh_cuda.

Two runs give bit-identical outputs.  SMOOTH, COARSE_SWEEPS, MAX_ITERS and the defaults are choices, not tuned values.
"""
import numpy as np

RESOLUTIONS = (33, 65, 129, 257, 513)
BLOCK = 256               # NERO_POISSON_BLOCK (include/nero_poisson.h)
MIN_POINTS = 16
COARSEST = 5              # nodes per axis of the coarsest multigrid level
SMOOTH = 2                # red-black sweeps before and after each coarse correction
COARSE_SWEEPS = 8         # sweeps on the coarsest level
MAX_ITERS = 200
SCREEN = 4.0              # PoissonRecon's default point weight
SCALE = 1.1
TOL = 1e-5


def _torch():
    import torch
    return torch


def _ops():
    from . import ops
    return ops


def _host(a, what):
    torch = _torch()
    if torch.is_tensor(a):
        a = a.detach().cpu().numpy()
    a = np.asarray(a, np.float64)
    if a.ndim != 2 or a.shape[1] != 3:
        raise ValueError(f'{what} must be [n,3], got shape {a.shape}')
    return a


def check_inputs(points, normals, resolution=513, screen=SCREEN, scale=SCALE, tol=TOL, max_iters=MAX_ITERS, trim=0.0):
    """(points fp64 [n,3], unit normals fp32 [n,3]) on the host, or ValueError."""
    p, nrm = _host(points, 'points'), _host(normals, 'normals')
    if p.shape[0] != nrm.shape[0]:
        raise ValueError(f'{p.shape[0]} points but {nrm.shape[0]} normals')
    if p.shape[0] < MIN_POINTS:
        raise ValueError(f'need at least {MIN_POINTS} points, got {p.shape[0]}')
    if p.shape[0] >= 2 ** 31:
        raise ValueError(f'{p.shape[0]} points do not fit int32 indices')
    if not np.isfinite(p).all():
        raise ValueError('points must be finite')
    if not np.isfinite(nrm).all():
        raise ValueError('normals must be finite')
    length = np.linalg.norm(nrm, axis=1)
    if not (length > 0).all():
        raise ValueError(f'{int((length <= 0).sum())} normals are zero')
    if resolution not in RESOLUTIONS:
        raise ValueError(f'resolution must be one of {RESOLUTIONS}, got {resolution}')
    if not (np.isfinite(screen) and screen > 0):
        raise ValueError(f'screen must be positive, got {screen}')
    if not (np.isfinite(scale) and scale > 1):
        raise ValueError(f'scale must be > 1, got {scale}')
    if not tol > 0 or int(max_iters) < 1:
        raise ValueError(f'need tol > 0 and max_iters >= 1, got {tol}, {max_iters}')
    if not (np.isfinite(trim) and trim >= 0):
        raise ValueError(f'trim must be >= 0, got {trim}')
    if not (p.max(0) - p.min(0)).max() > 0:
        raise ValueError('the points all coincide')
    return p, (nrm / length[:, None]).astype(np.float32)


def frame(points, N, scale=SCALE):
    """(origin fp64 [3], h) of the grid over the points' bounding cube scaled by `scale`."""
    lo, hi = points.min(0), points.max(0)
    side = scale * float((hi - lo).max())
    return (lo + hi) / 2 - side / 2, side / (N - 1)


def levels(N):
    """Nodes per axis of the multigrid levels, finest first, down to COARSEST."""
    out = [N]
    while out[-1] > COARSEST:
        out.append((out[-1] - 1) // 2 + 1)
    return out


def weights(n, occupied, screen):
    """(sigma fp64, fp32(sigma), ws = fp32(screen / sigma))."""
    sigma = 1.5 * n / occupied
    return sigma, np.float32(sigma), np.float32(screen / sigma)


def vcycle(be, L, b, x):
    """x = one V-cycle applied to b (level 0).  L: per level dict(N, s, d, x, b, r), the x, b, r of level 0 unused."""
    last = len(L) - 1
    for l, lv in enumerate(L):
        bl, xl = (b, x) if l == 0 else (lv['b'], lv['x'])
        be.zero(xl)
        if l == last:
            for _ in range(COARSE_SWEEPS // 2):
                be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 0)
                be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 1)
            for _ in range(COARSE_SWEEPS // 2):
                be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 1)
                be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 0)
            break
        for _ in range(SMOOTH):
            be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 0)
            be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 1)
        be.residual(xl, bl, lv['d'], lv['N'], lv['s'], lv['r'])
        be.restrict(lv['r'], lv['N'], L[l + 1]['b'])
    for l in range(last - 1, -1, -1):
        lv = L[l]
        bl, xl = (b, x) if l == 0 else (lv['b'], lv['x'])
        be.prolong(L[l + 1]['x'], L[l + 1]['N'], xl)
        for _ in range(SMOOTH):
            be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 1)
            be.smooth(xl, bl, lv['d'], lv['N'], lv['s'], 0)


def pcg(be, L, b, tol=TOL, max_iters=MAX_ITERS, trace=None):
    """Preconditioned conjugate gradients from x = 0 -> (x, history of |r| / |b|, iterations).  be: the kernels (the CUDA
    ones below, or the oracle's); trace (a list) gets per iteration dict(x, r, p, alpha, beta, rz, pap) as host copies."""
    x, r, z, p, ap = be.vec(), be.vec(), be.vec(), be.vec(), be.vec()
    be.zero(x)
    be.copy(b, r)
    bb = be.dot(b, b)
    hist = [1.0]
    if bb == 0.0:
        return x, hist, 0
    bnorm = np.sqrt(bb)
    vcycle(be, L, r, z)
    be.copy(z, p)
    rz = be.dot(r, z)
    it = 0
    while it < max_iters:
        be.matvec(p, ap)
        pap = be.dot(p, ap)
        alpha = rz / pap
        be.update(x, r, p, ap, np.float32(alpha))
        it += 1
        hist.append(float(np.sqrt(be.dot(r, r)) / bnorm))
        rec = None if trace is None else dict(alpha=alpha, rz=rz, pap=pap)
        if hist[-1] <= tol or it == max_iters:
            if rec is not None:
                trace.append(dict(rec, x=be.host(x), r=be.host(r), p=be.host(p), beta=None))
            break
        vcycle(be, L, r, z)
        rz_new = be.dot(r, z)
        beta = rz_new / rz
        be.direction(p, z, np.float32(beta))
        rz = rz_new
        if rec is not None:
            trace.append(dict(rec, x=be.host(x), r=be.host(r), p=be.host(p), beta=beta))
    return x, hist, it


class _Cuda:
    """The kernels of include/nero_poisson.h on flat CUDA fp32 vectors of the finest level."""

    def __init__(self, N, q, start, ws):
        torch = _torch()
        self.ops, self.torch = _ops(), torch
        self.N, self.q, self.start, self.ws, self.n = N, q, start, float(ws), q.shape[0]
        self.sx = torch.empty(self.n, dtype=torch.float32, device=q.device)
        self.out = torch.empty(1, dtype=torch.float64, device=q.device)

    def vec(self, N=None):
        N = self.N if N is None else N
        return self.torch.empty(N ** 3, dtype=self.torch.float32, device=self.q.device)

    def zero(self, x):
        x.zero_()

    def copy(self, a, b):
        b.copy_(a)

    def host(self, a):
        return a.cpu().numpy()

    def matvec(self, x, y):
        self.ops.K('nero_poisson_matvec', x, self.N, self.q, self.n, self.start, self.ws, self.sx, y, launches=2)

    def smooth(self, x, b, d, N, s, colour):
        self.ops.K('nero_poisson_smooth', x, b, d, N, float(s), colour)

    def residual(self, x, b, d, N, s, r):
        self.ops.K('nero_poisson_residual', x, b, d, N, float(s), r)

    def restrict(self, fine, Nf, coarse):
        self.ops.K('nero_poisson_restrict', fine, Nf, coarse)

    def prolong(self, coarse, Nc, fine):
        self.ops.K('nero_poisson_prolong', coarse, Nc, fine)

    def interp(self, grid, N, q):
        out = self.torch.empty(q.shape[0], dtype=self.torch.float32, device=q.device)
        self.ops.K('nero_poisson_interp', grid, N, q, q.shape[0], out)
        return out

    def total(self, a, b=None):
        """The fp64 fixed-order sum of a b (of a when b is None)."""
        m = a.numel()
        blocks = self.ops.ceil_div(m, BLOCK)
        partial = self.torch.empty(blocks, dtype=self.torch.float64, device=a.device)
        self.ops.K('nero_poisson_dot', a, b, m, partial)
        self.ops.K('nero_align_reduce', partial, 1, blocks, 1, self.out)
        return float(self.out.item())

    def dot(self, a, b):
        return self.total(a, b)

    def update(self, x, r, p, ap, alpha):
        self.ops.K('nero_poisson_update', x, r, p, ap, float(alpha), x.numel())

    def direction(self, p, z, beta):
        self.ops.K('nero_poisson_direction', p, z, float(beta), p.numel())


def setup(points, normals, N, screen=SCREEN, scale=SCALE):
    """Binning and splats on the GPU from checked host inputs -> dict(origin, h, q, nrm, keys, order, start, occupied, sigma,
    sigma32, ws, v (vx, vy, vz), b, density, diag) with CUDA tensors, the samples in sorted order."""
    torch = _torch()
    ops = _ops()
    dev = torch.device('cuda')
    n = points.shape[0]
    origin, h = frame(points, N, scale)
    p = torch.from_numpy(np.ascontiguousarray(points)).to(dev)
    q = torch.empty(n, 3, dtype=torch.float32, device=dev)
    keys = torch.empty(n, dtype=torch.int32, device=dev)
    ops.K('nero_poisson_keys', p, n, float(origin[0]), float(origin[1]), float(origin[2]), float(h), N, q, keys)
    skeys, order = torch.sort(keys, stable=True)           # plumbing: stable, so each cell keeps its samples in input order
    q = q[order].contiguous()
    nrm = torch.from_numpy(np.ascontiguousarray(normals)).to(dev)[order].contiguous()
    cells = (N - 1) ** 3
    start = torch.empty(cells + 1, dtype=torch.int32, device=dev)
    ops.K('nero_poisson_cell_starts', skeys, n, cells, start)
    occupied = int((skeys[1:] != skeys[:-1]).sum()) + 1
    sigma, sigma32, ws = weights(n, occupied, screen)
    E = (N - 1) * N * N
    v = tuple(torch.empty(E, dtype=torch.float32, device=dev) for _ in range(3))
    ops.K('nero_poisson_edge_splat', q, nrm, n, start, N, float(sigma32), *v, launches=3)
    b = torch.empty(N ** 3, dtype=torch.float32, device=dev)
    ops.K('nero_poisson_rhs', *v, N, b)
    density = torch.empty(N ** 3, dtype=torch.float32, device=dev)
    diag = torch.empty(N ** 3, dtype=torch.float32, device=dev)
    ops.K('nero_poisson_node_splat', q, n, start, N, density, diag)
    return dict(origin=origin, h=h, q=q, nrm=nrm, keys=skeys, order=order, start=start, occupied=occupied, sigma=sigma,
                sigma32=sigma32, ws=ws, v=v, b=b, density=density, diag=diag)


def hierarchy(be, N, diag, ws):
    """The multigrid levels: dict(N, s, d, x, b, r) per level, d = ws diag on level 0 and restricted below."""
    L, Ns = [], levels(N)
    for l, Nl in enumerate(Ns):
        if l == 0:
            d = diag * float(ws)
        else:
            d = be.vec(Nl)
            be.restrict(L[-1]['d'], L[-1]['N'], d)
        L.append(dict(N=Nl, s=float(2 ** l), d=d, x=be.vec(Nl) if l else None, b=be.vec(Nl) if l else None,
                      r=be.vec(Nl) if l < len(Ns) - 1 else None))
    return L


def reconstruct(points, normals, resolution=513, screen=SCREEN, scale=SCALE, tol=TOL, max_iters=MAX_ITERS, trim=0.0, trace=None):
    """The screened Poisson surface of an oriented cloud: points [n,3], normals [n,3] (numpy or tensors) -> (verts CUDA fp32
    [V,3] in world coordinates, tris CUDA int32 [T,3], info).  info: origin, h, resolution, sigma, ws, occupied, iso, history
    (|r| / |b| per iteration, 1 first), iterations, density (per output vertex, over the median), triangles_before,
    triangles_after.  trace (a dict) gets the setup tensors (setup()), chi, the levels and the PCG iterates (pcg())."""
    p, nrm = check_inputs(points, normals, resolution, screen, scale, tol, max_iters, trim)
    N = resolution
    S = setup(p, nrm, N, screen, scale)
    be = _Cuda(N, S['q'], S['start'], S['ws'])
    L = hierarchy(be, N, S['diag'], S['ws'])
    iters = None if trace is None else []
    chi, hist, it = pcg(be, L, S['b'], tol, int(max_iters), iters)
    world, tris, dens, iso, T0 = extract(be, S, L, chi, trim)
    if trace is not None:
        trace.update(S, chi=chi, levels=L, iterates=iters)
    info = dict(origin=S['origin'], h=S['h'], resolution=N, sigma=S['sigma'], ws=float(S['ws']), occupied=S['occupied'], iso=iso,
                history=hist, iterations=it, density=dens, triangles_before=T0, triangles_after=int(tris.shape[0]))
    return world, tris, info


def extract(be, S, L, chi, trim=0.0):
    """The iso-surface of the solution chi and its trim -> (verts world fp32, tris, vertex densities, iso, triangles before
    the trim)."""
    torch = _torch()
    N = L[0]['N']
    iso = be.total(be.interp(chi, N, S['q'])) / S['q'].shape[0]
    verts, tris = _mesh().marching_cubes_cuda(chi.view(N, N, N), iso)
    T0 = tris.shape[0]
    dens = torch.zeros(0, dtype=torch.float32, device=chi.device)
    if T0:
        # the splat density two levels down (spacing 4h) at v / 4, over its median
        D1 = be.vec(L[1]['N'])
        be.restrict(S['density'], N, D1)
        D2 = be.vec(L[2]['N'])
        be.restrict(D1, L[1]['N'], D2)
        dv = be.interp(D2, L[2]['N'], (verts * 0.25).contiguous())
        dens = dv / median_density(dv)
        if trim > 0:
            verts, tris, dens = _trim(verts, tris, dens, trim)
    world = (verts.to(torch.float64) * S['h'] + torch.from_numpy(S['origin']).to(verts.device)).to(torch.float32)
    return world, tris, dens, iso, T0


def median_density(dv):
    """The median (torch's lower median) of the non-zero vertex densities: a large unsampled part of a closed surface must
    not make it zero."""
    pos = dv[dv > 0]
    return pos.median() if pos.numel() else dv.new_ones(())


def _mesh():
    from . import mesh
    return mesh


def _trim(verts, tris, dens, t):
    """Drop the triangles with a vertex density below t; the ordered compaction of evaluate.clean_mesh_cuda removes the
    vertices no kept triangle references -> (verts, tris, dens)."""
    torch = _torch()
    ops = _ops()
    V, T = verts.shape[0], tris.shape[0]
    dev = verts.device
    keep = torch.empty(T, dtype=torch.uint8, device=dev)
    ops.K('nero_poisson_trim', dens, V, tris, T, float(t), keep)
    label = torch.zeros(T, dtype=torch.int32, device=dev)    # one component: the trim alone decides
    root_keep = torch.ones(V, dtype=torch.uint8, device=dev)
    nbt, nbv = ops.ceil_div(T, BLOCK), ops.ceil_div(V, BLOCK)
    tri_flag = torch.empty(T, dtype=torch.uint8, device=dev)
    vert_flag = torch.empty(V, dtype=torch.uint8, device=dev)
    blk_cnt = torch.empty(nbt + nbv, dtype=torch.int32, device=dev)
    blk_off = torch.empty(nbt + nbv, dtype=torch.int64, device=dev)
    totals = torch.empty(2, dtype=torch.int64, device=dev)
    ops.K('nero_meshpts_compact_count', tris, T, keep, label, root_keep, V, tri_flag, vert_flag, blk_cnt, blk_off, totals, launches=5)
    nv, nt = totals.tolist()
    remap = torch.empty(V, dtype=torch.int32, device=dev)
    vo = torch.empty(nv, 3, dtype=torch.float32, device=dev)
    to = torch.empty(nt, 3, dtype=torch.int32, device=dev)
    ops.K('nero_meshpts_compact_emit', verts, V, tris, T, tri_flag, vert_flag, blk_off, nv, nt, remap, vo, to, launches=2)
    return vo, to, dens[vert_flag.bool()]
