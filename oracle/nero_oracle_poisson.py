"""numpy restatement of include/nero_poisson.h: the cell keys, the gather splats of the normal field and the density, the
right-hand side, the operator, red-black Gauss-Seidel, residual, restriction, prolongation, interpolation, the fp64 dot
partials and the CG updates, in fp32 with the kernels' operation order, so the product's arrays are compared bit for bit.
Backend() runs nero_b200/poisson.py's own vcycle() and pcg() on them.  numpy rounds every float32 operation correctly and
never contracts a * b + c.

assemble() builds A = G^T G + ws S^T S and G^T v with scipy.sparse in fp64 for the exact solution."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import nero_oracle_align as OA
from nero_b200 import poisson as P

F = np.float32
ONE, HALF = F(1.0), F(0.5)


def keys(points, origin, h, N):
    """(q fp32 [n,3], keys int32 [n])."""
    q = ((np.asarray(points, np.float64) - origin) / h).astype(F)
    q = np.minimum(np.maximum(q, F(0)), F(N - 1))
    c = np.minimum(np.floor(q).astype(np.int64), N - 2)
    return q, ((c[:, 0] * (N - 1) + c[:, 1]) * (N - 1) + c[:, 2]).astype(np.int32)


def cell_starts(skeys, cells):
    return np.searchsorted(skeys, np.arange(cells + 1), 'left').astype(np.int32)


def hat(q, c):
    return ONE - np.abs(q - c)


def _gather(centres, ranges, q, start, N, terms):
    """The gather of include/nero_poisson.h: for lattice points at centres [E,3] fp32 and per axis the cell offsets `ranges`
    (relative to the point's index, ascending), acc_j = acc_j + terms(w, sample)[j] over the support cells (x outermost) and
    their samples in sorted order.  centres' integer parts are the indices the offsets apply to."""
    E = centres.shape[0]
    idx = np.floor(centres).astype(np.int64)
    M = N - 1
    accs = None
    for dx in ranges[0]:
        for dy in ranges[1]:
            for dz in ranges[2]:
                c = idx + np.asarray([dx, dy, dz])
                ok = ((c >= 0) & (c <= N - 2)).all(1)
                key = np.where(ok, (c[:, 0] * M + c[:, 1]) * M + c[:, 2], 0)
                s0, s1 = start[key], start[key + 1]
                cnt = np.where(ok, s1 - s0, 0)
                for t in range(int(cnt.max()) if E else 0):
                    live = t < cnt
                    s = np.where(live, s0 + t, 0)
                    w3 = [hat(q[s, a], centres[:, a]) for a in range(3)]
                    live = live & (w3[0] > 0) & (w3[1] > 0) & (w3[2] > 0)
                    w = (w3[0] * w3[1]) * w3[2]
                    vals = terms(w, s)
                    if accs is None:
                        accs = [np.zeros(E, F) for _ in vals]
                    for j, v in enumerate(vals):
                        accs[j] = np.where(live, accs[j] + v, accs[j])
    return accs


def _nodes(N):
    i, j, k = np.meshgrid(np.arange(N), np.arange(N), np.arange(N), indexing='ij')
    return np.stack([i.ravel(), j.ravel(), k.ravel()], 1)


def edge_splat(q, nrm, start, N, sigma32):
    """(vx, vy, vz) fp32 on the three edge lattices."""
    out = []
    for a in range(3):
        dims = [N - 1 if b == a else N for b in range(3)]
        i, j, k = np.meshgrid(*[np.arange(d) for d in dims], indexing='ij')
        e = np.stack([i.ravel(), j.ravel(), k.ravel()], 1).astype(F)
        e[:, a] += HALF
        ranges = [(-1, 0, 1) if b == a else (-1, 0) for b in range(3)]
        acc = _gather(e, ranges, q, start, N, lambda w, s: [w * nrm[s, a]])
        out.append(acc[0] / F(sigma32) if acc is not None else np.zeros(e.shape[0], F))
    return tuple(out)


def node_splat(q, start, N):
    """(density, diag) fp32 [N^3]."""
    acc = _gather(_nodes(N).astype(F), [(-1, 0)] * 3, q, start, N, lambda w, s: [w, w * w])
    return acc[0], acc[1]


def rhs(vx, vy, vz, N):
    vx, vy, vz = vx.reshape(N - 1, N, N), vy.reshape(N, N - 1, N), vz.reshape(N, N, N - 1)
    acc = np.zeros((N, N, N), F)
    for a, v in enumerate((vx, vy, vz)):
        sl = [slice(None)] * 3
        end = np.zeros((N, N, N), F)
        sl[a] = slice(1, None)
        end[tuple(sl)] = v                        # the edge ending at the node
        has = np.zeros((N, N, N), bool)
        has[tuple(sl)] = True
        acc = np.where(has, acc + end, acc)
        beg = np.zeros((N, N, N), F)
        sl[a] = slice(0, N - 1)
        beg[tuple(sl)] = v                        # the edge starting at it
        has = np.zeros((N, N, N), bool)
        has[tuple(sl)] = True
        acc = np.where(has, acc - beg, acc)
    return acc.ravel()


def interp(grid, N, q):
    g = grid.reshape(-1)
    c = np.clip(np.floor(q).astype(np.int64), 0, N - 2)
    acc = np.zeros(q.shape[0], F)
    for a in range(2):
        for b in range(2):
            for e in range(2):
                node = c + np.asarray([a, b, e])
                w3 = [hat(q[:, d], node[:, d].astype(F)) for d in range(3)]
                live = (w3[0] > 0) & (w3[1] > 0) & (w3[2] > 0)
                val = g[(node[:, 0] * N + node[:, 1]) * N + node[:, 2]]
                acc = np.where(live, acc + ((w3[0] * w3[1]) * w3[2]) * val, acc)
    return acc


def stencil(x, N):
    """(m, lap, deg) of every node: the neighbours' sum, the sum of (x_n - x_m) and their number, in stencil order."""
    x = x.reshape(N, N, N)
    m, lap, deg = np.zeros_like(x), np.zeros_like(x), np.zeros(x.shape, np.int64)
    for a in range(3):
        for step in (-1, 1):
            nb = np.zeros_like(x)
            has = np.zeros(x.shape, bool)
            dst = [slice(None)] * 3
            src = [slice(None)] * 3
            if step < 0:
                dst[a], src[a] = slice(1, None), slice(0, N - 1)
            else:
                dst[a], src[a] = slice(0, N - 1), slice(1, None)
            nb[tuple(dst)] = x[tuple(src)]
            has[tuple(dst)] = True
            m = np.where(has, m + nb, m)
            lap = np.where(has, lap + (x - nb), lap)
            deg = deg + has
    return m.ravel(), lap.ravel(), deg.ravel()


def _colour(N):
    n = _nodes(N)
    return n.sum(1) & 1


def matvec(x, N, q, start, ws):
    sx = interp(x, N, q)
    t = _gather(_nodes(N).astype(F), [(-1, 0)] * 3, q, start, N, lambda w, s: [w * sx[s]])[0]
    return stencil(x, N)[1] + F(ws) * t


def smooth(x, b, d, N, s, colour):
    m, _, deg = stencil(x, N)
    s = F(s)
    new = (b + s * m) / (s * deg.astype(F) + d)
    return np.where(_colour(N) == colour, new, x)


def residual(x, b, d, N, s):
    return b - (F(s) * stencil(x, N)[1] + d * x)


def restrict(fine, Nf):
    Nc = (Nf - 1) // 2 + 1
    f = fine.reshape(Nf, Nf, Nf)
    I = _nodes(Nc)
    acc = np.zeros(I.shape[0], F)
    for dx in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dz in (-1, 0, 1):
                p = 2 * I + np.asarray([dx, dy, dz])
                ok = ((p >= 0) & (p < Nf)).all(1)
                pc = np.clip(p, 0, Nf - 1)
                w = (F(1 if dx == 0 else 0.5) * F(1 if dy == 0 else 0.5)) * F(1 if dz == 0 else 0.5)
                acc = np.where(ok, acc + w * f[pc[:, 0], pc[:, 1], pc[:, 2]], acc)
    return acc


def prolong(coarse, Nc, fine):
    Nf = 2 * (Nc - 1) + 1
    c = coarse.reshape(Nc, Nc, Nc)
    n = _nodes(Nf)
    odd = n & 1
    w = (np.where(odd[:, 0], HALF, ONE) * np.where(odd[:, 1], HALF, ONE)) * np.where(odd[:, 2], HALF, ONE)
    acc = np.zeros(n.shape[0], F)
    for a in range(2):
        for b in range(2):
            for e in range(2):
                live = (a <= odd[:, 0]) & (b <= odd[:, 1]) & (e <= odd[:, 2])
                p = np.minimum(n // 2 + np.asarray([a, b, e]), Nc - 1)
                acc = np.where(live, acc + w * c[p[:, 0], p[:, 1], p[:, 2]], acc)
    return fine + acc


def total(a, b=None):
    v = a.astype(np.float64) if b is None else a.astype(np.float64) * b.astype(np.float64)
    return float(OA.reduce(OA.block_partials(v[:, None])[None])[0, 0])


class Backend:
    """The numpy kernels behind nero_b200.poisson.vcycle / pcg (vectors are flat fp32 arrays, updated in place)."""

    def __init__(self, N, q, start, ws):
        self.N, self.q, self.start, self.ws = N, q, start, F(ws)

    def vec(self, N=None):
        return np.zeros((self.N if N is None else N) ** 3, F)

    def zero(self, x):
        x[:] = 0

    def copy(self, a, b):
        b[:] = a

    def host(self, a):
        return a.copy()

    def matvec(self, x, y):
        y[:] = matvec(x, self.N, self.q, self.start, self.ws)

    def smooth(self, x, b, d, N, s, colour):
        x[:] = smooth(x, b, d, N, s, colour)

    def residual(self, x, b, d, N, s, r):
        r[:] = residual(x, b, d, N, s)

    def restrict(self, fine, Nf, coarse):
        coarse[:] = restrict(fine, Nf)

    def prolong(self, coarse, Nc, fine):
        fine[:] = prolong(coarse, Nc, fine)

    def dot(self, a, b):
        return total(a, b)

    def update(self, x, r, p, ap, alpha):
        x[:] = x + F(alpha) * p
        r[:] = r - F(alpha) * ap

    def direction(self, p, z, beta):
        p[:] = z + F(beta) * p


def setup(points, normals, N, screen=P.SCREEN, scale=P.SCALE):
    """nero_b200.poisson.setup in numpy from checked host inputs (poisson.check_inputs)."""
    n = points.shape[0]
    origin, h = P.frame(points, N, scale)
    q, k = keys(points, origin, h, N)
    order = np.argsort(k, kind='stable')
    q, nrm, sk = q[order], np.asarray(normals, F)[order], k[order]
    start = cell_starts(sk, (N - 1) ** 3)
    occupied = int((sk[1:] != sk[:-1]).sum()) + 1
    sigma, sigma32, ws = P.weights(n, occupied, screen)
    v = edge_splat(q, nrm, start, N, sigma32)
    density, diag = node_splat(q, start, N)
    return dict(origin=origin, h=h, q=q, nrm=nrm, keys=sk, order=order, start=start, occupied=occupied, sigma=sigma, sigma32=sigma32,
                ws=ws, v=v, b=rhs(*v, N), density=density, diag=diag)


def hierarchy(N, diag, ws):
    """nero_b200.poisson.hierarchy with numpy arrays."""
    L, Ns = [], P.levels(N)
    for l, Nl in enumerate(Ns):
        d = diag * F(ws) if l == 0 else restrict(L[-1]['d'], L[-1]['N'])
        z = lambda: np.zeros(Nl ** 3, F)
        L.append(dict(N=Nl, s=float(2 ** l), d=d, x=z() if l else None, b=z() if l else None, r=z() if l < len(Ns) - 1 else None))
    return L


def solve(S, N, tol=P.TOL, max_iters=P.MAX_ITERS, trace=None):
    """pcg() of nero_b200.poisson on the numpy kernels -> (chi, history, iterations)."""
    be = Backend(N, S['q'], S['start'], S['ws'])
    return P.pcg(be, hierarchy(N, S['diag'], S['ws']), S['b'].copy(), tol, max_iters, trace)


# ------------------------------------------------------------------------------------------------ exact system (scipy)
def assemble(q, ws, N):
    """(G [edges, N^3], S [n, N^3]) in fp64 from the fp32 grid coordinates; A = G^T G + ws S^T S."""
    idx = np.arange(N ** 3).reshape(N, N, N)
    rows = []
    for a in range(3):
        lo = [slice(None)] * 3
        hi = [slice(None)] * 3
        lo[a], hi[a] = slice(0, N - 1), slice(1, None)
        rows.append((idx[tuple(lo)].ravel(), idx[tuple(hi)].ravel()))
    ia = np.concatenate([r[0] for r in rows])
    ib = np.concatenate([r[1] for r in rows])
    E = ia.shape[0]
    G = sp.csr_matrix((np.concatenate([-np.ones(E), np.ones(E)]), (np.tile(np.arange(E), 2), np.concatenate([ia, ib]))), shape=(E, N ** 3))
    q = np.asarray(q, np.float64)
    c = np.clip(np.floor(q).astype(np.int64), 0, N - 2)
    f = q - c
    data, ri, ci = [], [], []
    for a in range(2):
        for b in range(2):
            for e in range(2):
                w = np.where(a, f[:, 0], 1 - f[:, 0]) * np.where(b, f[:, 1], 1 - f[:, 1]) * np.where(e, f[:, 2], 1 - f[:, 2])
                node = c + np.asarray([a, b, e])
                data.append(w)
                ri.append(np.arange(q.shape[0]))
                ci.append((node[:, 0] * N + node[:, 1]) * N + node[:, 2])
    S = sp.csr_matrix((np.concatenate(data), (np.concatenate(ri), np.concatenate(ci))), shape=(q.shape[0], N ** 3))
    return G, S


def exact(S, N):
    """The fp64 solution of A chi = G^T v for the setup S (oracle or GPU, as host arrays)."""
    G, Sm = assemble(S['q'], float(S['ws']), N)
    A = (G.T @ G + float(S['ws']) * (Sm.T @ Sm)).tocsc()
    v = np.concatenate([np.asarray(x, np.float64) for x in S['v']])
    return spla.spsolve(A, G.T @ v)


def mesh(points, normals, N, screen=P.SCREEN, scale=P.SCALE):
    """The exact fp64 surface: (verts world fp64, tris, chi, iso, setup) with the repository's marching-cubes oracle."""
    import nero_oracle_mesh as OMesh
    S = setup(points, normals, N, screen, scale)
    chi = exact(S, N)
    G, Sm = assemble(S['q'], float(S['ws']), N)
    iso = float((Sm @ chi).mean())
    v, t = OMesh.marching_cubes(chi.reshape(N, N, N).astype(np.float32), iso)
    return S['origin'] + S['h'] * v, t, chi, iso, S
