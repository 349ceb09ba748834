"""numpy restatement of the sparse-feature kernels of k_sift.cu, k_match.cu and k_verify.cu (include/nero_features.h), in
the protocol of nero_b200/features.py: the scale space in fp32 with the kernels' operation order (so it must match bit for
bit), the keypoint refinement, orientation and descriptor in fp64 (the kernels' fp32 library functions agree with it to
rounding), the matcher in int64 and RANSAC in fp64 with the kernels' hash stream.

There is no reference code to pin the kernels against: the reference workflow runs COLMAP's feature_extractor and
exhaustive_matcher.  This file states what the kernels compute instead.
"""
import math

import numpy as np

import nero_oracle_objprep as OOp

f32 = np.float32
BORDER = 5
INT_MAX = 2 ** 31 - 1


# ------------------------------------------------------------------------------------------------ scale space
def blur(img, taps):
    """Separable pass along rows, then columns, clamp to edge: acc = t0 x0, then acc + t_k (x_-k + x_+k)."""
    img = np.asarray(img, f32)
    h, w = img.shape
    r = taps.shape[0] - 1
    xs, ys = np.arange(w), np.arange(h)
    acc = taps[0] * img
    for k in range(1, r + 1):
        acc = acc + taps[k] * (img[:, np.clip(xs - k, 0, w - 1)] + img[:, np.clip(xs + k, 0, w - 1)])
    tmp = acc
    acc = taps[0] * tmp
    for k in range(1, r + 1):
        acc = acc + taps[k] * (tmp[np.clip(ys - k, 0, h - 1)] + tmp[np.clip(ys + k, 0, h - 1)])
    return acc


def scale_space(grey, taps, sizes, scales):
    """(gauss, dog) per octave as fp32 stacks; taps: the level_sigmas taps, sizes: octave_sizes."""
    gauss, dog = [], []
    for o, (w, h) in enumerate(sizes):
        G = [blur(grey, taps[0]) if o == 0 else gauss[-1][scales][0:2 * h:2, 0:2 * w:2][:h, :w]]
        for l in range(1, scales + 3):
            G.append(blur(G[-1], taps[l]))
        G = np.stack(G)
        gauss.append(G)
        dog.append(G[1:] - G[:-1])
    return gauss, dog


def extrema(D, thr):
    """int32 [n, 3] (x, y, level) of the candidates of one DoG stack, in (level, row, column) order."""
    L, h, w = D.shape
    out = []
    thr = f32(thr)
    for l in range(1, L - 1):
        c = D[l, BORDER:h - BORDER, BORDER:w - BORDER]
        mx = np.ones_like(c, bool)
        mn = np.ones_like(c, bool)
        for dl in (-1, 0, 1):
            for dy in (-1, 0, 1):
                for dx in (-1, 0, 1):
                    if dl == dy == dx == 0:
                        continue
                    u = D[l + dl, BORDER + dy:h - BORDER + dy, BORDER + dx:w - BORDER + dx]
                    mx &= c > u
                    mn &= c < u
        ys, xs = np.nonzero((np.abs(c) > thr) & (mx | mn))
        out.append(np.stack([xs + BORDER, ys + BORDER, np.full_like(xs, l)], 1))
    return np.concatenate(out, 0).astype(np.int32) if out else np.zeros((0, 3), np.int32)


def refine(D, cand, octave, sigma0, peak, edge):
    """Refined records [n, 8] (x, y, sigma, response, octave, level, fractional level, ok), fp64."""
    L, h, w = D.shape
    S = L - 2
    out = np.zeros((len(cand), 8))
    for i, (x, y, l) in enumerate(np.asarray(cand, np.int64)):
        ok = True
        for it in range(6):
            A = lambda dl, dy, dx: float(D[l + dl, y + dy, x + dx])
            Dv = A(0, 0, 0)
            g = np.array([0.5 * (A(0, 0, 1) - A(0, 0, -1)), 0.5 * (A(0, 1, 0) - A(0, -1, 0)), 0.5 * (A(1, 0, 0) - A(-1, 0, 0))])
            H = np.zeros((3, 3))
            H[0, 0] = A(0, 0, 1) + A(0, 0, -1) - 2 * Dv
            H[1, 1] = A(0, 1, 0) + A(0, -1, 0) - 2 * Dv
            H[2, 2] = A(1, 0, 0) + A(-1, 0, 0) - 2 * Dv
            H[0, 1] = H[1, 0] = 0.25 * (A(0, 1, 1) - A(0, 1, -1) - A(0, -1, 1) + A(0, -1, -1))
            H[0, 2] = H[2, 0] = 0.25 * (A(1, 0, 1) - A(1, 0, -1) - A(-1, 0, 1) + A(-1, 0, -1))
            H[1, 2] = H[2, 1] = 0.25 * (A(1, 1, 0) - A(1, -1, 0) - A(-1, 1, 0) + A(-1, -1, 0))
            det = np.linalg.det(H)
            if not abs(det) > 1e-300:
                ok = False
                break
            b = -np.linalg.solve(H, g)
            if it == 5:
                break
            dx = 1 if (b[0] > 0.6 and x < w - BORDER - 1) else (-1 if (b[0] < -0.6 and x > BORDER) else 0)
            dy = 1 if (b[1] > 0.6 and y < h - BORDER - 1) else (-1 if (b[1] < -0.6 and y > BORDER) else 0)
            if not dx and not dy:
                break
            x, y = x + dx, y + dy
        val = Dv + 0.5 * g @ b
        tr, d2 = H[0, 0] + H[1, 1], H[0, 0] * H[1, 1] - H[0, 1] ** 2
        ok = ok and bool(np.all(np.abs(b) < 1.5)) and abs(val) >= peak and d2 > 0 and tr * tr * edge < (edge + 1) ** 2 * d2
        s = l + b[2]
        out[i] = (x + b[0], y + b[1], sigma0 * 2.0 ** (s / S), val, octave, l, s, 1.0 if ok else 0.0)
    return out


def _grad(img, xx, yy):
    gx = 0.5 * (img[yy, xx + 1].astype(np.float64) - img[yy, xx - 1])
    gy = 0.5 * (img[yy + 1, xx].astype(np.float64) - img[yy - 1, xx])
    a = np.arctan2(gy, gx)
    return np.sqrt(gx * gx + gy * gy), np.where(a < 0, a + 2 * np.pi, a)


def describe(kp, gauss):
    """(angle [n, 2], desc uint8 [n, 2, 128], nori [n], hist [n, 36] smoothed) of keypoint records on the Gaussian stacks."""
    n = len(kp)
    angle, desc, nori, hists = np.zeros((n, 2)), np.zeros((n, 2, 128), np.uint8), np.zeros(n, np.int32), np.zeros((n, 36))
    for i, k in enumerate(np.asarray(kp, np.float64)):
        x, y, sigma, o, l = k[0], k[1], k[2], int(k[4]), int(k[5])
        img = gauss[o][l]
        h, w = img.shape
        xi, yi = int(math.floor(float(f32(x) + f32(0.5)))), int(math.floor(float(f32(y) + f32(0.5))))
        sw = 1.5 * sigma
        R = max(1, int(math.floor(3 * sw)))
        yy, xx = np.mgrid[max(1, yi - R):min(h - 2, yi + R) + 1, max(1, xi - R):min(w - 2, xi + R) + 1]
        dx, dy = xx - x, yy - y
        r2 = dx * dx + dy * dy
        m = r2 < R * R + 0.6
        mag, ang = _grad(img, xx[m], yy[m])
        b = np.floor(36 * ang / (2 * np.pi)).astype(np.int64) % 36
        hist = np.bincount(b, mag * np.exp(-r2[m] / (2 * sw * sw)), 36)
        for _ in range(6):
            hist = (np.roll(hist, 1) + hist + np.roll(hist, -1)) / 3
        hists[i] = hist
        hm, hp = np.roll(hist, 1), np.roll(hist, -1)
        peaks = [(hist[j], j) for j in range(36) if hist[j] > hm[j] and hist[j] > hp[j] and hist[j] >= 0.8 * hist.max()]
        peaks = sorted(peaks, key=lambda p: (-p[0], p[1]))[:2]
        nori[i] = len(peaks)
        sbp = 3 * sigma
        W = int(math.floor(math.sqrt(2) * sbp * 2.5 + 0.5))
        yy, xx = np.mgrid[max(1, yi - W):min(h - 2, yi + W) + 1, max(1, xi - W):min(w - 2, xi + W) + 1]
        yy, xx = yy.reshape(-1), xx.reshape(-1)
        mag, ang = _grad(img, xx, yy)
        for a, (h0, j) in enumerate(peaks):
            di = -0.5 * (hp[j] - hm[j]) / (hp[j] + hm[j] - 2 * h0)
            th = 2 * np.pi * (j + di + 0.5) / 36
            angle[i, a] = th
            c, s = np.cos(th), np.sin(th)
            dx, dy = xx - x, yy - y
            nx, ny = (c * dx + s * dy) / sbp, (-s * dx + c * dy) / sbp
            bx, by = nx + 1.5, ny + 1.5
            sel = (bx > -1) & (bx < 4) & (by > -1) & (by < 4)
            rel = np.mod(ang - th, 2 * np.pi)
            nt = 8 * rel / (2 * np.pi)
            v = mag * np.exp(-(nx * nx + ny * ny) / 8)
            x0, y0, t0 = np.floor(bx), np.floor(by), np.floor(nt)
            fx, fy, ft = bx - x0, by - y0, nt - t0
            d = np.zeros(128)
            for ey in (0, 1):
                for ex in (0, 1):
                    for et in (0, 1):
                        yb, xb, tb = y0.astype(np.int64) + ey, x0.astype(np.int64) + ex, (t0.astype(np.int64) + et) % 8
                        ok = sel & (yb >= 0) & (yb <= 3) & (xb >= 0) & (xb <= 3)
                        wgt = v * (fy if ey else 1 - fy) * (fx if ex else 1 - fx) * (ft if et else 1 - ft)
                        np.add.at(d, ((yb * 4 + xb) * 8 + tb)[ok], wgt[ok])
            nrm = np.sqrt((d * d).sum())
            d = np.minimum(d / nrm if nrm > 0 else d, 0.2)
            nrm = np.sqrt((d * d).sum())
            d = d / nrm if nrm > 0 else d
            d = np.sqrt(d / d.sum()) if d.sum() > 0 else d
            desc[i, a] = np.minimum(255, np.floor(512 * d + 0.5)).astype(np.uint8)
    return angle, desc, nori, hists


# ------------------------------------------------------------------------------------------------ matcher
def row_best(A, B):
    """(index, d1, d2) int64 per row of A against B (uint8 descriptors): exact squared distances, ties to the lower index."""
    A, B = np.asarray(A, np.int64), np.asarray(B, np.int64)
    if B.shape[0] == 0:
        return np.full(A.shape[0], -1), np.full(A.shape[0], INT_MAX), np.full(A.shape[0], INT_MAX)
    D = (A * A).sum(1)[:, None] + (B * B).sum(1)[None, :] - 2 * A @ B.T
    i1 = D.argmin(1)
    d1 = D[np.arange(A.shape[0]), i1]
    if B.shape[0] == 1:
        return i1, d1, np.full(A.shape[0], INT_MAX)
    D[np.arange(A.shape[0]), i1] = np.iinfo(np.int64).max
    return i1, d1, D.min(1)


def match(A, B, ratio=(16, 25), max_d1=128450):
    """int64 [m, 2] mutual matches (row of A, row of B) in row order."""
    i1, d1, d2 = row_best(A, B)
    j1 = row_best(B, A)[0]
    r = np.arange(np.asarray(A).shape[0])
    keep = (i1 >= 0) & (ratio[1] * d1 < ratio[0] * d2) & (d1 <= max_d1)
    keep &= np.where(i1 >= 0, j1[np.maximum(i1, 0)] if j1.shape[0] else -1, -1) == r
    return np.stack([r[keep], i1[keep]], 1)


# ------------------------------------------------------------------------------------------------ RANSAC
def _mix(x):
    return OOp._mix(x)


def draw_key(seed, pair, hyp, draw):
    with np.errstate(over='ignore'):
        h = _mix(np.uint32(np.uint32(seed) * np.uint32(0x9e3779b9) + np.uint32(0x7f4a7c15)))
        h = _mix(h ^ np.uint32(pair))
        h = _mix(np.asarray(hyp, np.uint32) ^ h)
        return _mix(h ^ np.uint32(draw))


def jacobi(A, sweeps):
    """Batched cyclic Jacobi of symmetric [B, n, n] in the kernel's order -> (diagonalised A, V)."""
    A = np.array(A, np.float64)
    B, n, _ = A.shape
    V = np.broadcast_to(np.eye(n), A.shape).copy()
    for _ in range(sweeps):
        for p in range(n - 1):
            for q in range(p + 1, n):
                apq = A[:, p, q].copy()
                nz = apq != 0
                with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
                    theta = (A[:, q, q] - A[:, p, p]) / (2 * apq)
                    t = np.where(theta >= 0, 1.0, -1.0) / (np.abs(theta) + np.sqrt(theta * theta + 1))
                    c = 1 / np.sqrt(t * t + 1)
                    s = t * c
                c, s = np.where(nz, c, 1.0)[:, None], np.where(nz, s, 0.0)[:, None]
                akp, akq = A[:, :, p].copy(), A[:, :, q].copy()
                A[:, :, p], A[:, :, q] = c * akp - s * akq, s * akp + c * akq
                apk, aqk = A[:, p, :].copy(), A[:, q, :].copy()
                A[:, p, :], A[:, q, :] = c * apk - s * aqk, s * apk + c * aqk
                vkp, vkq = V[:, :, p].copy(), V[:, :, q].copy()
                V[:, :, p], V[:, :, q] = c * vkp - s * vkq, s * vkp + c * vkq
    return A, V


def _rows(P, nm):
    x1, y1 = (P[..., 0] - nm[0]) * nm[2], (P[..., 1] - nm[1]) * nm[2]
    x2, y2 = (P[..., 2] - nm[3]) * nm[5], (P[..., 3] - nm[4]) * nm[5]
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones_like(x1)], -1)


def solve_F(M, nm):
    """[B, 9] unit F with the largest |entry| positive from normal matrices M [B, 9, 9]."""
    A, V = jacobi(M, 12)
    m = np.argmin(np.diagonal(A, 0, 1, 2), 1)
    f = V[np.arange(len(M)), :, m].reshape(-1, 3, 3)
    A3, V3 = jacobi(np.einsum('bkr,bkc->brc', f, f), 8)
    s = np.argmin(np.diagonal(A3, 0, 1, 2), 1)
    v = V3[np.arange(len(M)), :, s]
    f = f - np.einsum('brc,bc->br', f, v)[:, :, None] * v[:, None, :]
    T1 = np.array([[nm[2], 0, -nm[2] * nm[0]], [0, nm[2], -nm[2] * nm[1]], [0, 0, 1]])
    T2 = np.array([[nm[5], 0, -nm[5] * nm[3]], [0, nm[5], -nm[5] * nm[4]], [0, 0, 1]])
    F = (T2.T @ f @ T1).reshape(-1, 9)
    big = F[np.arange(len(F)), np.abs(F).argmax(1)]
    return F * (np.where(big < 0, -1.0, 1.0) / np.sqrt((F * F).sum(1)))[:, None]


def inliers(F, P, max_err2):
    """bool [B, m] of F [B, 9] on points [m, 4]."""
    F = F.reshape(-1, 3, 3)
    x1 = np.stack([P[:, 0], P[:, 1], np.ones(len(P))], 1)
    x2 = np.stack([P[:, 2], P[:, 3], np.ones(len(P))], 1)
    l = np.einsum('brc,mc->bmr', F, x1)
    mm = np.einsum('brc,mr->bmc', F, x2)
    e = (x2[None] * l).sum(-1)
    return e * e <= max_err2 * (l[..., 0] ** 2 + l[..., 1] ** 2 + mm[..., 0] ** 2 + mm[..., 1] ** 2)


def ransac(P, pair, hypotheses, seed, max_err2):
    """(F [9], best hypothesis, its count, final inlier mask) of one pair's points [n, 4], as the kernel computes them."""
    P = np.asarray(P, np.float64)
    n = P.shape[0]
    if n < 8:
        return np.zeros(9), -1, 0, np.zeros(n, bool)
    c = P.mean(0)
    c = np.array([P[:, 0].sum() / n, P[:, 1].sum() / n, P[:, 2].sum() / n, P[:, 3].sum() / n])
    d1 = np.sqrt((P[:, 0] - c[0]) ** 2 + (P[:, 1] - c[1]) ** 2).sum()
    d2 = np.sqrt((P[:, 2] - c[2]) ** 2 + (P[:, 3] - c[3]) ** 2).sum()
    nm = (c[0], c[1], math.sqrt(2) * n / d1 if d1 > 0 else 1.0, c[2], c[3], math.sqrt(2) * n / d2 if d2 > 0 else 1.0)
    hs = np.arange(hypotheses)
    idx = np.full((hypotheses, 8), -1)
    k = np.zeros(hypotheses, np.int64)
    for d in range(64):
        m = (draw_key(seed, pair, hs, d) % np.uint32(n)).astype(np.int64)
        dup = (idx == m[:, None]).any(1)
        take = (k < 8) & ~dup
        idx[hs[take], k[take]] = m[take]
        k += take
    valid = k == 8
    hv = hs[valid]
    a = _rows(P[idx[valid]], nm)                        # [B, 8, 9]
    M = np.zeros((len(hv), 9, 9))
    for j in range(8):
        M = M + a[:, j, :, None] * a[:, j, None, :]
    F = solve_F(M, nm)
    cnt = inliers(F, P, max_err2).sum(1)
    w = int(np.argmax(cnt))                              # first maximum: the lowest hypothesis
    Fw, bh, bc = F[w], int(hv[w]), int(cnt[w])
    if bc >= 8:
        a = _rows(P[inliers(Fw[None], P, max_err2)[0]], nm)
        M = np.zeros((9, 9))
        for row in a:
            M = M + row[:, None] * row[None, :]
        Fw = solve_F(M[None], nm)[0]
    return Fw, bh, bc, inliers(Fw[None], P, max_err2)[0]
