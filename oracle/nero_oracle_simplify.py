"""numpy / fp64 restatement of the mesh simplification of k_simplify.cu (include/nero_simplify.h), in the GPU's order, so
the kernels must match it bit for bit.  The protocol is stated in nero_b200/simplify.py; in short:
  input       float32 verts [V,3], int32 tris [T,3]; indices in [0, V), three distinct per triangle, every undirected edge in
              at most two triangles, never twice in the same direction
  locks       an endpoint of a boundary edge, or a vertex whose fan walk from its lowest-index triangle reaches fewer
              triangles than its degree
  quadrics    per triangle A p p^T, p = (n/|n|, -(n/|n|).v0), A = |n|/2, n = (v1 - v0) x (v2 - v0); Q_v = the sum over v's
              triangles in ascending index; 10 entries xx xy xz xw yy yz yw zz zw ww
  one round   unique edges (a < b) sorted; placement by the adjugate or the cheapest of a, b, midpoint; validity (locks, link
              condition, valences, no flip); key = float32(cost) bits << 32 | edge id; vmin / rmin selection; the quarter
              guard and the budget floor((T - F) / 2); collapse b into a; drop the two triangles of the edge
  output      the referenced vertices in index order, rounded once to float32, and the remapped triangles
Every product and sum is one IEEE fp64 operation, written out in the order the kernels use (numpy does not contract).
"""
import numpy as np

GUARD = 0.25                    # collapse only keys within the cheapest quarter of the round's valid keys
DET_EPS = 1e-10                 # accept the adjugate solve when |det M| > DET_EPS ||M||_F^3
KEY_INF = np.int64(2 ** 63 - 1)   # the key of an edge that may not collapse


def check(verts, tris):
    """Refuse a mesh the protocol does not accept (ValueError naming the first offending triangle or edge); return the
    half-edge twins: twin[3 t + k] = the half-edge running the other way along tris[t][k] -> tris[t][(k+1) % 3], or -1."""
    V, T = verts.shape[0], tris.shape[0]
    t = tris.astype(np.int64)
    bad = ((t < 0) | (t >= V)).any(1)
    if bad.any():
        i = int(np.argmax(bad))
        raise ValueError(f'simplify: triangle {i} has an index outside [0, {V}): {tuple(int(x) for x in t[i])}')
    rep = (t[:, 0] == t[:, 1]) | (t[:, 1] == t[:, 2]) | (t[:, 0] == t[:, 2])
    if rep.any():
        i = int(np.argmax(rep))
        raise ValueError(f'simplify: triangle {i} repeats an index: {tuple(int(x) for x in t[i])}')
    src, dst = t.reshape(-1), t[:, [1, 2, 0]].reshape(-1)
    hkey = (np.minimum(src, dst) * V + np.maximum(src, dst)) * 2 + (src > dst)
    order = np.argsort(hkey, kind='stable')
    sk = hkey[order]
    ek = sk >> 1
    start = np.ones(sk.shape[0], bool)
    start[1:] = ek[1:] != ek[:-1]
    first = np.flatnonzero(start)
    n = np.diff(np.append(first, sk.shape[0]))
    over = first[n >= 3]
    if over.size:
        e = int(ek[over[0]])
        raise ValueError(f'simplify: edge ({e // V}, {e % V}) is used by more than two triangles')
    two = first[n == 2]
    same = two[(sk[two] & 1) == (sk[two + 1] & 1)]
    if same.size:
        e = int(ek[same[0]])
        raise ValueError(f'simplify: edge ({e // V}, {e % V}) is used twice in the same direction (inconsistent winding)')
    twin = np.full(3 * T, -1, np.int64)
    twin[order[two]] = order[two + 1]
    twin[order[two + 1]] = order[two]
    return twin


def vertex_triangles(tris, V):
    """CSR of each vertex's triangles in ascending index: (ptr [V+1], tri [3T])."""
    corner = np.argsort(tris.reshape(-1), kind='stable')
    ptr = np.zeros(V + 1, np.int64)
    ptr[1:] = np.cumsum(np.bincount(tris.reshape(-1), minlength=V))
    return ptr, corner // 3


def locks(tris, V, twin):
    """bool [V]: on a boundary edge, or a fan walk that does not reach every triangle of the vertex."""
    T = tris.shape[0]
    ptr, vt = vertex_triangles(tris, V)
    deg = np.diff(ptr)
    lock = np.zeros(V, bool)
    open_ = np.flatnonzero(twin < 0)
    lock[tris.reshape(-1)[open_]] = True
    lock[tris[:, [1, 2, 0]].reshape(-1)[open_]] = True
    vs = np.flatnonzero(deg > 0)
    t0 = vt[ptr[vs]]
    k0 = np.argmax(tris[t0] == vs[:, None], axis=1)
    h = 3 * t0 + k0
    cnt = np.ones(vs.shape[0], np.int64)
    live = np.ones(vs.shape[0], bool)
    for _ in range(int(deg.max()) + 1 if T else 0):
        if not live.any():
            break
        tw = twin[h]
        stop = live & (tw < 0)
        live &= ~stop
        nt = np.where(live, tw // 3, t0)
        back = live & (nt == t0)
        live &= ~back
        cnt += live
        live &= cnt <= deg[vs]
        h = np.where(live, 3 * (tw // 3) + (tw % 3 + 1) % 3, h)
    lock[vs] |= cnt != deg[vs]
    return lock


def _cross(p0, p1, p2):
    e1, e2 = p1 - p0, p2 - p0
    return np.stack([e1[:, 1] * e2[:, 2] - e1[:, 2] * e2[:, 1], e1[:, 2] * e2[:, 0] - e1[:, 0] * e2[:, 2],
                     e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]], 1)


def triangle_quadrics(pos, tris):
    n = _cross(pos[tris[:, 0]], pos[tris[:, 1]], pos[tris[:, 2]])
    ln = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    ok = ln > 0
    safe = np.where(ok, ln, 1.0)
    nh = n / safe[:, None]
    v0 = pos[tris[:, 0]]
    d = -((nh[:, 0] * v0[:, 0] + nh[:, 1] * v0[:, 1]) + nh[:, 2] * v0[:, 2])
    p = [nh[:, 0], nh[:, 1], nh[:, 2], d]
    A = ln * 0.5
    q = np.stack([A * (p[i] * p[j]) for i in range(4) for j in range(i, 4)], 1)
    return np.where(ok[:, None], q, 0.0)


def vertex_quadrics(pos, tris):
    """Q [V,10]: each vertex's triangle quadrics added from 0.0 in ascending triangle index."""
    V = pos.shape[0]
    tq = triangle_quadrics(pos, tris)
    ptr, vt = vertex_triangles(tris, V)
    deg = np.diff(ptr)
    Q = np.zeros((V, 10))
    for j in range(int(deg.max()) if tris.shape[0] else 0):
        m = deg > j
        Q[m] = Q[m] + tq[vt[ptr[:-1][m] + j]]
    return Q


def quadric_cost(q, x):
    """x^T M x + 2 g^T x + c of quadrics q [n,10] at points x [n,3]."""
    mx0 = (q[:, 0] * x[:, 0] + q[:, 1] * x[:, 1]) + q[:, 2] * x[:, 2]
    mx1 = (q[:, 1] * x[:, 0] + q[:, 4] * x[:, 1]) + q[:, 5] * x[:, 2]
    mx2 = (q[:, 2] * x[:, 0] + q[:, 5] * x[:, 1]) + q[:, 7] * x[:, 2]
    xmx = (x[:, 0] * mx0 + x[:, 1] * mx1) + x[:, 2] * mx2
    gx = (q[:, 3] * x[:, 0] + q[:, 6] * x[:, 1]) + q[:, 8] * x[:, 2]
    return (xmx + 2.0 * gx) + q[:, 9]


def placement(q, pa, pb):
    """(x [n,3], cost [n]) of edges with summed quadrics q and endpoints pa, pb (fp64)."""
    c00 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5]
    c01 = q[:, 2] * q[:, 5] - q[:, 1] * q[:, 7]
    c02 = q[:, 1] * q[:, 5] - q[:, 2] * q[:, 4]
    c11 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2]
    c12 = q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5]
    c22 = q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
    det = (q[:, 0] * c00 + q[:, 1] * c01) + q[:, 2] * c02
    fro = np.sqrt(((q[:, 0] * q[:, 0] + q[:, 4] * q[:, 4]) + q[:, 7] * q[:, 7])
                  + 2.0 * ((q[:, 1] * q[:, 1] + q[:, 2] * q[:, 2]) + q[:, 5] * q[:, 5]))
    g0, g1, g2 = q[:, 3], q[:, 6], q[:, 8]
    with np.errstate(divide='ignore', invalid='ignore'):
        xs = np.stack([-((c00 * g0 + c01 * g1) + c02 * g2) / det, -((c01 * g0 + c11 * g1) + c12 * g2) / det,
                       -((c02 * g0 + c12 * g1) + c22 * g2) / det], 1)
    d = pb - pa
    ln = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    lo, hi = np.minimum(pa, pb) - ln[:, None], np.maximum(pa, pb) + ln[:, None]
    ok = (np.abs(det) > DET_EPS * ((fro * fro) * fro)) & ((xs >= lo) & (xs <= hi)).all(1)
    mid = (pa + pb) * 0.5
    ca, cb, cm = quadric_cost(q, pa), quadric_cost(q, pb), quadric_cost(q, mid)
    use_b = cb < ca
    best, cbest = np.where(use_b[:, None], pb, pa), np.where(use_b, cb, ca)
    use_m = cm < cbest
    best, cbest = np.where(use_m[:, None], mid, best), np.where(use_m, cm, cbest)
    with np.errstate(invalid='ignore'):
        cs = quadric_cost(q, np.where(ok[:, None], xs, 0.0))
    x = np.where(ok[:, None], xs, best)
    cost = np.where(ok, cs, cbest)
    return x, np.where(cost > 0, cost, 0.0)


def edges(tris, V):
    """(ea, eb) unique undirected edges a < b sorted by (a, b), and the adjacency CSR (ptr [V+1], nbr) with ascending rows."""
    src, dst = tris.reshape(-1).astype(np.int64), tris[:, [1, 2, 0]].reshape(-1).astype(np.int64)
    k = np.unique(np.concatenate([src * V + dst, dst * V + src]))
    s, d = k // V, k % V
    ptr = np.zeros(V + 1, np.int64)
    ptr[1:] = np.cumsum(np.bincount(s, minlength=V))
    m = s < d
    return s[m], d[m], ptr, d, k


def validity(pos, tris, lock, ea, eb, x, ptr, nbr, akeys):
    V = pos.shape[0]
    E = ea.shape[0]
    val = np.diff(ptr)
    ok = ~lock[ea] & ~lock[eb]
    common = np.zeros(E, np.int64)
    low_opp = np.zeros(E, bool)
    for j in range(int(val.max())):
        m = val[ea] > j
        w = np.where(m, nbr[np.minimum(ptr[ea] + j, nbr.shape[0] - 1)], 0)
        kb = eb * V + w
        i = np.minimum(np.searchsorted(akeys, kb), akeys.shape[0] - 1)
        hit = m & (akeys[i] == kb)
        common += hit
        low_opp |= hit & (val[w] < 4)
    ok &= (common == 2) & ~low_opp & (val[ea] + val[eb] - 4 >= 3)
    vptr, vt = vertex_triangles(tris, V)
    deg = np.diff(vptr)
    for me, other in ((ea, eb), (eb, ea)):
        for j in range(int(deg.max())):
            m = ok & (deg[me] > j)
            t = tris[vt[np.minimum(vptr[me] + j, vt.shape[0] - 1)]]
            m &= ~(t == other[:, None]).any(1)
            p = [pos[t[:, c]] for c in range(3)]
            no = _cross(*p)
            pn = [np.where((t[:, c] == me)[:, None], x, p[c]) for c in range(3)]
            nn = _cross(*pn)
            dot = (nn[:, 0] * no[:, 0] + nn[:, 1] * no[:, 1]) + nn[:, 2] * no[:, 2]
            bad = (nn == 0).all(1) | ((no != 0).any(1) & ~(dot > 0))
            ok &= ~(m & bad)
    return ok


def keys(cost, ok):
    bits = np.asarray(cost, np.float32).view(np.uint32).astype(np.int64)
    return np.where(ok, (bits << 32) | np.arange(cost.shape[0], dtype=np.int64), KEY_INF)


def select(key, ea, eb, V, adj_src, nbr):
    """Selected edges: key == rmin[a] == rmin[b] (and not KEY_INF)."""
    vmin = np.full(V, KEY_INF, np.int64)
    np.minimum.at(vmin, ea, key)
    np.minimum.at(vmin, eb, key)
    rmin = vmin.copy()
    np.minimum.at(rmin, adj_src, vmin[nbr])
    return (key != KEY_INF) & (key == rmin[ea]) & (key == rmin[eb])


def threshold(key, selected, budget):
    """The largest key that may collapse this round: the ceil(E_valid GUARD)-th smallest valid key, lowered to the
    budget-th smallest selected key at or under it."""
    s = np.sort(key)
    nvalid = int((key != KEY_INF).sum())
    thr = s[max(int(np.ceil(nvalid * GUARD)) - 1, 0)]
    cand = np.sort(np.where(selected & (key <= thr), key, KEY_INF))
    return min(thr, cand[min(budget, key.shape[0]) - 1])


def prepare(verts, tris):
    """The checks, locks, fp64 positions and vertex quadrics of an input mesh: (lock [V], pos [V,3], Q [V,10])."""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64)
    lock = locks(tris, verts.shape[0], check(verts, tris))
    pos = verts.astype(np.float64)
    return lock, pos, vertex_quadrics(pos, tris)


def one_round(pos, Q, tris, lock, budget):
    """The selection of one round on the current triangles (nothing is collapsed): a dict of tris [T,3] (int32), edges
    [E,2], key [E], selected [E] (the independent set), collapsed [E] (the edges the round collapses), x [E,3], cost [E]."""
    V = pos.shape[0]
    ea, eb, ptr, nbr, akeys = edges(tris, V)
    x, cost = placement(Q[ea] + Q[eb], pos[ea], pos[eb])
    ok = validity(pos, tris, lock, ea, eb, x, ptr, nbr, akeys)
    key = keys(cost, ok)
    sel = select(key, ea, eb, V, np.repeat(np.arange(V), np.diff(ptr)), nbr)
    col = sel & (key <= threshold(key, sel, budget))
    return dict(tris=tris.astype(np.int32), edges=np.stack([ea, eb], 1), key=key, selected=sel, collapsed=col, x=x, cost=cost)


def simplify(verts, tris, faces, trace=None):
    """-> (verts float32 [V',3], tris int32 [T',3], stats).  trace (a list) gets one_round's dict for every round."""
    verts = np.asarray(verts, np.float32)
    tris = np.asarray(tris, np.int64)
    if faces < 4:
        raise ValueError(f'simplify: the target face count must be >= 4, got {faces}')
    V = verts.shape[0]
    lock, pos, Q = prepare(verts, tris)
    per_round, max_cost = [], 0.0
    while tris.shape[0] > faces:
        T = tris.shape[0]
        budget = (T - faces) // 2
        if budget == 0:
            break
        r = one_round(pos, Q, tris, lock, budget)
        if trace is not None:
            trace.append(r)
        col, x, cost = r['collapsed'], r['x'], r['cost']
        n = int(col.sum())
        if n == 0:
            break
        a, b = r['edges'][col, 0], r['edges'][col, 1]
        pos[a] = x[col]
        Q[a] = Q[a] + Q[b]
        remap = np.arange(V)
        remap[b] = a
        t = remap[tris]
        keep = (t[:, 0] != t[:, 1]) & (t[:, 1] != t[:, 2]) & (t[:, 0] != t[:, 2])
        tris = t[keep]
        per_round.append(n)
        max_cost = max(max_cost, float(cost[col].max()))
    used = np.zeros(V, bool)
    used[tris.reshape(-1)] = True
    new = np.cumsum(used) - 1
    out_v = pos[used].astype(np.float32)
    out_t = new[tris].astype(np.int32)
    stats = dict(rounds=len(per_round), collapses=per_round, vertices=int(out_v.shape[0]), triangles=int(out_t.shape[0]),
                 max_cost=max_cost, locked=int(lock.sum()))
    return out_v, out_t, stats
