"""Mesh simplification on the GPU: deterministic parallel quadric edge collapse (k_simplify.cu, include/nero_simplify.h).

Marching cubes spends triangles evenly over the surface; quadric error metrics (Garland-Heckbert) spend them where it
curves.  `simplify_cuda(verts, tris, faces)` reduces a mesh to about `faces` triangles in rounds of independent edge
collapses; `simplify(...)` is the same on numpy arrays.  oracle/nero_oracle_simplify.py restates the protocol in numpy and
the kernels match it bit for bit (DESIGN §4n lists the sizes the tests show it at).

Protocol
--------
Input.  float32 verts [V,3] and int32 tris [T,3] and a target face count F >= 4.  A ValueError names the first offender of:
an index outside [0, V) (smallest triangle), a triangle that repeats an index (smallest triangle), an undirected edge used
by more than two triangles, an edge used twice in the same direction (inconsistent winding) (smallest edge (a, b)).
Zero-area triangles with distinct indices are accepted.  Unreferenced vertices are dropped from the output; the winding of
every surviving triangle is preserved.

Locked vertices.  A vertex on a boundary edge (an edge with one triangle) is locked, and so is a vertex whose triangles do
not form a single fan: the walk around it from its lowest-index triangle, across the edges it shares with the next
triangle, reaches fewer triangles than it has.  An edge with a locked endpoint never collapses, so boundaries come out as
they went in.

Quadrics (fp64, every operation rounded on its own).  Per triangle n = (v1 - v0) x (v2 - v0) from the input positions, and
the quadric A p p^T with p = (n/|n|, -(n/|n|).v0), A = |n|/2; a zero-area triangle contributes 0.  Q_v is the sum of the
quadrics of v's triangles from 0.0 in ascending triangle order (10 entries xx xy xz xw yy yz yw zz zw ww).  A collapse of b
into a sets Q_a <- Q_a + Q_b; quadrics are never recomputed from the current faces.

One round.
 1. Edges: the unique undirected edges (a < b) of the current triangles sorted by (a, b); the rank is the edge id.  The
    vertex adjacency (CSR, ascending rows) and each vertex's triangles (ascending) come from the same sorts.
 2. Placement and cost: Q = Q_a + Q_b with 3x3 block M, vector g, scalar c.  x = -adj(M) g / det M is accepted when
    |det M| > 1e-10 ||M||_F^3 and x lies in the edge's bounding box grown by the edge length on every side; otherwise x is
    the cheapest of a, b and the midpoint, ties in that order.  cost = x^T M x + 2 g^T x + c, clamped at 0.
 3. Validity: neither endpoint locked; a and b have exactly two common neighbours (the link condition); both have valence
    >= 4; deg a + deg b - 4 >= 3; and every other triangle around a or b, with the moved corner at x, keeps
    n_new . n_old > 0 where n_old != 0 and never gets n_new = 0.  These keep a closed 2-manifold closed, manifold and of the
    same topology.
 4. Selection: key = float32(cost) bits << 32 | edge id (KEY_INF for an invalid edge).  vmin[v] = the smallest key of the
    edges at v (a 64-bit atomicMin: the minimum does not depend on the order); rmin[v] = the smallest vmin over v and its
    neighbours.  An edge is selected iff key == rmin[a] == rmin[b].
 5. Quality guard and budget: only selected edges whose key is at most the ceil(E_valid GUARD)-th smallest valid key
    collapse (GUARD = 1/4), so the rounds stay close to greedy order; at most floor((T - F) / 2) collapse, the smallest keys
    first.
 6. Collapse: a, the lower index, moves to x and takes Q_a + Q_b, b is renamed a in every triangle; the two triangles that
    held both are dropped, and the rest are compacted in triangle order.
Rounds stop when T <= F or when a round collapses nothing.  A closed mesh ends with exactly F triangles for even F, F or
F + 1 for odd F; when the rules leave nothing to collapse the result has more than F triangles, which the stats show.

Why the selected collapses of a round commute.  Let e = (a, b) and f = (c, d) be two selected edges.  key_e = rmin[a] is at
most vmin[w] for every w in the closed 1-ring of a, and vmin[a] <= key_e because e is at a.  If c were a or a neighbour of
a, then key_f = rmin[c] <= vmin[a] <= key_e and key_e = rmin[a] <= vmin[c] <= key_f, so key_e = key_f and e = f (the
edge id makes keys unique).  Hence no endpoint of one edge lies in the closed 1-ring of an endpoint of the other: no
triangle touches both edges, so the triangles each collapse rewrites or drops are disjoint, and so are the vertices whose
position, quadric or adjacency it changes, except that a vertex w opposite to both edges loses one neighbour to each.  Such
a w has a and b, and c and d, as consecutive neighbours with no edge between the pairs, so its valence is at least 6 and
stays >= 4 after either collapse.  Every test made for one edge therefore still holds after the others, and the round's
result does not depend on the order in which its collapses are applied.

Output.  float32 verts (the fp64 working positions rounded once) of the referenced vertices in index order, and int32 tris.
stats: rounds, collapses (per round), vertices, triangles, max_cost (the largest collapsed cost), locked (vertices).
Determinism: no floating-point atomics and every sum in a fixed order, so two runs give the same bytes.
"""
import time

import torch

from . import ops

GUARD = 0.25                               # collapse only within the cheapest quarter of a round's valid keys
KEY_INF = 0x7fffffffffffffff               # NERO_SIMPLIFY_KEY_INF
_BLOCK = 256                               # NERO_SIMPLIFY_BLOCK
_INT32_MAX = 2 ** 31 - 1


def _mesh(verts, tris):
    """(verts float32 [V,3], tris int32 [T,3], tris as given in int64) on the GPU; shapes, integer indices and finiteness
    checked."""
    v, t = torch.as_tensor(verts).detach(), torch.as_tensor(tris).detach()
    if v.ndim != 2 or v.shape[1] != 3 or t.ndim != 2 or t.shape[1] != 3:
        raise ValueError(f'simplify needs verts [V,3] and tris [T,3], got {tuple(v.shape)} and {tuple(t.shape)}')
    if v.shape[0] < 1 or t.shape[0] < 1:
        raise ValueError(f'simplify: the mesh is empty ({v.shape[0]} vertices, {t.shape[0]} triangles)')
    if t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f'simplify: triangle indices must be integers, got {t.dtype}')
    if v.shape[0] > _INT32_MAX or 6 * t.shape[0] > _INT32_MAX:
        raise ValueError(f'simplify: {v.shape[0]} vertices / {t.shape[0]} triangles do not fit the int32 rows of the kernels')
    dev = v.device if v.device.type == 'cuda' else t.device if t.device.type == 'cuda' else torch.device('cuda')
    ops.require_cuda(dev, 'simplify')
    v = v.to(dev, torch.float32).contiguous()
    t64 = t.to(dev, torch.int64)
    if not bool(torch.isfinite(v).all()):
        raise ValueError('simplify: vertex coordinates must be finite')
    t = t64.clamp(-1, v.shape[0]).to(torch.int32).contiguous()      # out-of-range indices stay out of range in int32
    return v, t, t64


def _vertex_triangles(t, V):
    """CSR of each vertex's triangles in ascending index: (ptr int32 [V+1], tri int32 [3T])."""
    flat = t.view(-1)
    corner = torch.sort(flat, stable=True)[1]
    ptr = torch.zeros(V + 1, dtype=torch.int32, device=t.device)
    ptr[1:] = torch.cumsum(torch.bincount(flat, minlength=V), 0)
    return ptr, (corner // 3).to(torch.int32)


def _edges(t, V):
    """Unique edges a < b sorted by (a, b) and the adjacency CSR with ascending rows: (ea, eb, adj_ptr, adj), int32."""
    src, dst = t.view(-1).long(), t[:, [1, 2, 0]].reshape(-1).long()
    k = torch.unique(torch.cat([src * V + dst, dst * V + src]))      # sorted
    s, d = k // V, k % V
    ptr = torch.zeros(V + 1, dtype=torch.int32, device=t.device)
    ptr[1:] = torch.cumsum(torch.bincount(s, minlength=V), 0)
    m = s < d
    return s[m].to(torch.int32), d[m].to(torch.int32), ptr, d.to(torch.int32)


def _threshold(key, selected, budget):
    """The largest key that may collapse this round, as a one-element int64 tensor on key's device: the
    ceil(E_valid GUARD)-th smallest valid key, lowered to the budget-th smallest selected key at or under it.  Plumbing:
    two sorts, no read-back.  The rank is computed in fp64, where E_valid GUARD is exact (GUARD is a power of two and
    E_valid < 2^53); the default float32 would round it for E_valid > 2^24."""
    inf = torch.full((), KEY_INF, dtype=torch.int64, device=key.device)
    nvalid = (key != inf).sum()
    rank = torch.clamp(torch.ceil(nvalid.to(torch.float64) * GUARD).to(torch.int64) - 1, min=0)
    thr = torch.sort(key).values[rank]
    cand = torch.where(selected.bool() & (key <= thr), key, inf)
    return torch.minimum(thr, torch.sort(cand).values[min(budget, key.shape[0]) - 1]).reshape(1)


def _check(v, t, t64):
    """The input checks of the protocol -> the half-edge twins [3T] (int32).  t64: the indices as given, for the messages."""
    V, T = v.shape[0], t.shape[0]
    err = torch.empty(4, dtype=torch.int64, device=v.device)
    ops.K('nero_simplify_check_tris', t, T, V, err, launches=2)
    e = err.tolist()
    if e[0] != KEY_INF:
        raise ValueError(f'simplify: triangle {e[0]} has an index outside [0, {V}): {tuple(t64[e[0]].tolist())}')
    if e[1] != KEY_INF:
        raise ValueError(f'simplify: triangle {e[1]} repeats an index: {tuple(t[e[1]].tolist())}')
    src, dst = t.view(-1).long(), t[:, [1, 2, 0]].reshape(-1).long()
    hkey = (torch.minimum(src, dst) * V + torch.maximum(src, dst)) * 2 + (src > dst).long()
    hkey, hidx = torch.sort(hkey, stable=True)
    twin = torch.empty(3 * T, dtype=torch.int32, device=v.device)
    ops.K('nero_simplify_check_edges', hkey, hidx, 3 * T, twin, err)
    e = err.tolist()
    for slot, what in ((2, 'is used by more than two triangles'), (3, 'is used twice in the same direction (inconsistent winding)')):
        if e[slot] != KEY_INF:
            ek = int(hkey[e[slot]]) >> 1
            raise ValueError(f'simplify: edge ({ek // V}, {ek % V}) {what}')
    return twin


def simplify_cuda(verts, tris, faces, trace=None, profile=False):
    """Simplify a mesh to about `faces` triangles (see the module docstring).  verts [V,3] / tris [T,3] as numpy arrays or
    tensors -> (verts CUDA float32 [V',3], tris CUDA int32 [T',3], stats).  Reads back one count per round.

    trace (a list) gets one dict of numpy arrays per round: tris [T,3] (the round's input), edges [E,2], key [E], selected [E] (the independent set),
    collapsed [E], x [E,3], cost [E].  profile=True adds stats['ms'], the host-clock milliseconds of the phases check /
    prepare / edges / cost / select / collapse / output, each ended by a device synchronise."""
    if int(faces) != faces or faces < 4:
        raise ValueError(f'simplify: the target face count must be an integer >= 4, got {faces}')
    faces = int(faces)
    v, t, t64 = _mesh(verts, tris)
    V, T = v.shape[0], t.shape[0]
    dev = v.device
    ms = {k: 0.0 for k in ('check', 'prepare', 'edges', 'cost', 'select', 'collapse', 'output')}
    clock = [0.0]

    def lap(phase):
        if profile:
            torch.cuda.synchronize(dev)
            now = time.perf_counter()
            if phase is not None:
                ms[phase] += (now - clock[0]) * 1e3
            clock[0] = now

    with torch.cuda.device(dev):
        lap(None)
        twin = _check(v, t, t64)
        del t64
        lap('check')
        vt_ptr, vt_tri = _vertex_triangles(t, V)
        tri_q = torch.empty(T, 10, dtype=torch.float64, device=dev)
        pos = torch.empty(V, 3, dtype=torch.float64, device=dev)
        Q = torch.empty(V, 10, dtype=torch.float64, device=dev)
        locked = torch.empty(V, dtype=torch.uint8, device=dev)
        ops.K('nero_simplify_prepare', v, V, t, T, vt_ptr, vt_tri, twin, tri_q, pos, Q, locked, launches=2)
        del tri_q, twin
        n_locked = int(locked.sum())
        lap('prepare')
        vmin = torch.empty(V, dtype=torch.int64, device=dev)
        rmin = torch.empty(V, dtype=torch.int64, device=dev)
        remap = torch.empty(V, dtype=torch.int32, device=dev)
        max_cost = torch.zeros((), dtype=torch.float64, device=dev)
        per_round = []
        while T > faces:
            budget = (T - faces) // 2
            if budget == 0:
                break
            ea, eb, adj_ptr, adj = _edges(t, V)
            vt_ptr, vt_tri = _vertex_triangles(t, V)
            E = ea.shape[0]
            lap('edges')
            x = torch.empty(E, 3, dtype=torch.float64, device=dev)
            cost = torch.empty(E, dtype=torch.float64, device=dev)
            key = torch.empty(E, dtype=torch.int64, device=dev)
            ops.K('nero_simplify_edges', pos, Q, locked, V, t, T, adj_ptr, adj, vt_ptr, vt_tri, ea, eb, E, x, cost, key)
            lap('cost')
            sel = torch.empty(E, dtype=torch.uint8, device=dev)
            ops.K('nero_simplify_select', ea, eb, E, key, adj_ptr, adj, V, vmin, rmin, sel, launches=4)
            thr = _threshold(key, sel, budget)
            lap('select')
            flag = torch.empty(E, dtype=torch.uint8, device=dev)
            ops.K('nero_simplify_collapse', ea, eb, E, key, sel, thr, x, V, pos, Q, remap, flag, launches=2)
            nblk = ops.ceil_div(T, _BLOCK)
            blk_cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
            blk_off = torch.empty(nblk, dtype=torch.int64, device=dev)
            total = torch.empty(1, dtype=torch.int64, device=dev)
            ops.K('nero_simplify_rewrite_count', t, T, remap, blk_cnt, blk_off, total, launches=2)
            if trace is not None:
                trace.append(dict(tris=t.cpu().numpy(), edges=torch.stack([ea, eb], 1).long().cpu().numpy(), key=key.cpu().numpy(),
                                  selected=sel.bool().cpu().numpy(), collapsed=flag.bool().cpu().numpy(),
                                  x=x.cpu().numpy(), cost=cost.cpu().numpy()))
            nt = int(total.item())
            n = (T - nt) // 2
            if n == 0:
                lap('collapse')
                break
            max_cost = torch.maximum(max_cost, torch.where(flag.bool(), cost, 0.0).max())
            out = torch.empty(nt, 3, dtype=torch.int32, device=dev)
            ops.K('nero_simplify_rewrite_emit', t, T, remap, blk_off, nt, out)
            t, T = out, nt
            per_round.append(n)
            lap('collapse')
        nblk = ops.ceil_div(V, _BLOCK)
        vflag = torch.empty(V, dtype=torch.uint8, device=dev)
        blk_cnt = torch.empty(nblk, dtype=torch.int32, device=dev)
        blk_off = torch.empty(nblk, dtype=torch.int64, device=dev)
        total = torch.empty(1, dtype=torch.int64, device=dev)
        ops.K('nero_simplify_output_count', t, T, V, vflag, blk_cnt, blk_off, total, launches=3)
        nv = int(total.item())
        vo = torch.empty(nv, 3, dtype=torch.float32, device=dev)
        to = torch.empty(T, 3, dtype=torch.int32, device=dev)
        ops.K('nero_simplify_output_emit', pos, V, t, T, vflag, blk_off, nv, remap, vo, to, launches=2)
        stats = dict(rounds=len(per_round), collapses=per_round, vertices=nv, triangles=T, max_cost=float(max_cost),
                     locked=n_locked)
        lap('output')
    if profile:
        stats['ms'] = ms
    return vo, to, stats


def simplify(verts, tris, faces):
    """simplify_cuda on numpy arrays: -> (verts float32 [V',3], tris int32 [T',3], stats) as numpy arrays."""
    v, t, stats = simplify_cuda(verts, tris, faces)
    return v.cpu().numpy(), t.cpu().numpy(), stats


def stats_line(stats):
    """One printable line of the statistics of simplify / simplify_cuda."""
    c = stats['collapses']
    per = ', '.join(map(str, c)) if len(c) <= 6 else ', '.join(map(str, c[:3])) + ', ..., ' + ', '.join(map(str, c[-2:]))
    return (f'simplify: {stats["rounds"]} rounds, collapses per round [{per}], {stats["vertices"]} vertices, '
            f'{stats["triangles"]} triangles, largest collapsed cost {stats["max_cost"]:.3e}, {stats["locked"]} locked vertices')
