"""Census of the stage-II Monte-Carlo shading kernels (`nero_b200/csrc/k_mcshade.cu`): every `nero_mc_*` launch of a
training step is checked against an fp64 restatement of its contract, built from the oracle's own functions, on the data
that launch saw.

Part one wraps `nero_b200.material.K` (material.py binds it with `from .ops import K`).  Per `nero_mc_*` call the wrapper
reads the `nero_mc_params` fields the launch uses (device buffers are viewed through the struct's pointers), fills every
element of the buffers the launch writes that lies outside its declared windows with a NaN sentinel, runs the kernel, checks
that every sentinel is intact (then puts the old values back) and checks each declared window:
  nero_mc_sample       DIR against OM.sample_diffuse_directions / sample_specular_directions from the same tables and
                       azimuth draws; ORG = pts + 1e-5 DIR rounded to fp32 (fused or not); column 3 of both is 0.
  nero_mc_classify     BLKC, BLKO and COUNTS exactly, recounted on the host from NRMH[:, 3] > 0.5.
  nero_mc_fill         SLOT exactly (misses 0, 1, ... and hits ~0, ~1, ... in ray order); EO = O.ide(d, 0) [| O.ide of the
                       sphere point, O.get_sphere_intersection after the |p| > 0.999 rescale]; EH = O.ipe of the
                       O.get_camera_plane_intersection mean and HHIT its hit flag; EI = O.embed(hit point, 8) | 0 | O.ide of
                       the reflection of -d about the normalised hit normal.
  nero_mc_combine_fwd  LD, LS, LSF: the estimator of OM.shade_mixed / get_lights (OM.distribution_ggx, OM.geometry_term,
                       the depth > 1e-5 mask, the human blend ol (1 - hw) + hl hw) on the MLP outputs of the step.
  nero_mc_combine_bwd  DPRE_O / DPRE_H / DPRE_I: fp64 autograd of the estimator w.r.t. the MLP outputs, times the exp
                       derivative (the output value, zero where clamped); dA: fp64 forward-mode autograd w.r.t. the
                       roughness through the weights, with the specular directions re-derived from the roughness.
  nero_mc_dir_bwd      dA2: fp64 autograd of <dE, E(d)> w.r.t. the specular directions (IDE, sphere point, human plane and
                       IPE, reflection about the normalised hit normal; the trace is not differentiated) contracted with
                       d(direction)/d(roughness); and the whole step: dA + dA2 against one fp64 autograd of the restated
                       light path with the roughness the only free input.
Directions take their VALUE from DIR (what the MLPs were fed) and, in the backward checks, their derivative from the fp64
sampler: the backward kernels recompute the specular directions, and must recompute the ones the forward pass used.
A failure names the kernel, the buffer, the point p, the sample j, the row and the column.

Part two builds `ops.McParams` directly, with hand-made hit patterns, depths, MLP outputs and geometry, and runs the same
checks at the edges a real scene rarely produces.

Bounds (U = 2^-24; every one below 1e-5 relative to the magnitudes it scales):
  * cond(x) of a per-ray weight x in {w, w (1-HoV)^5, dw/da, d(w (1-HoV)^5)/da}: |x32 - x64| + sum over NoH, HoV, NoL, NoV of
    the change of the fp64 x when that cosine moves by 4U, + the change when the specular directions take the fp64 sampler's
    values instead of DIR's (the backward kernels recompute them in fp32).  x32 is the same restatement in fp32 (torch eager: the reference's own
    arithmetic).  cond is large only where the reference's fp32 formula is ill-conditioned itself (GGX at roughness ~1e-3,
    1 + (a^2 - 1) el near el = 1), so the bound follows the conditioning instead of a blanket tolerance.
  * DIR: 2 |dir32 - dir64| + 16 U (1 + |azimuth before the mod|)  (the fp32 azimuth carries an error of its own magnitude).
  * LD, LS, LSF, dA: 4 sum_j |L_j| cond_j + (ceil(S/32) + 12) U sum_j |term_j|  (per-lane sums, the warp tree, the weight).
  * DPRE_*: (4 cond(dL) + 12 U |dL terms|) |output factor|.  Twice 2 cond: the weight of the estimator and the one of the
    backward kernel's recomputed direction each carry it.  Every bound adds 8 subnormal ulps (2^-146) for gradual underflow.
  * dA2: sum_j [2 |g.(t32 - t64)| + 2 |(g(d64) - g(DIR)).t| + 48 U sum_i |dE_i| |dE_i/dd| |t|]_j, with g = d<dE, E>/dd at DIR
    and t = dd/da: the fp32 tangent of the sampler, the kernel's recomputed direction (within DIR's own error of the exact
    one), and the 72-term fp32 sums of the encoding backward (the kernel evaluates the IDE polynomials in fp64 there).
  * IDE entries (EO, EI): 2 U (deg + 3m + 6) rho^m sum_k |mat_k| |z|^k: the condition number of the fp32 Vandermonde chain,
    which the kernel evaluates the way the reference does (DESIGN.md "IDE": near |z| = 1 that arithmetic is up to 2.4e-3 away
    from exact), plus the propagated error of a computed input: 16 U for the reflection, 8 U (1 + (dtx^2 + |x|^2 + 1) / root)
    for the sphere point.  PE8: 4 U.  IPE: 2^k delta_mean + 4 U (2 + 2^k |mean|), delta_mean from the magnitudes of the
    plane transform and of dist = -p_z / r_z.
  * Counted allowances, each reported in the table, never a fraction of rows:
      - HHIT, and the human term of dA2, where the fp64 margin of |r_z| > 1e-4, |mean| < 1.5 or dist > 0 is within its delta;
      - the |p| > 0.999 rescale of the sphere point where | |p| - 0.999 | < 4U: either branch;
      - the exp clamp: the kernel decides it from the output value, so an output equal to fp32 exp(exp_max) (a pre-activation
        at or within an ulp of exp_max, where torch still passes the gradient) may get 0 or the passed gradient.
"""
import collections
import math

import numpy as np
import pytest
import torch
import torch.autograd.forward_ad as fwAD
import torch.nn.functional as F

import nero_oracle as O
import nero_oracle_mat as OM
from helpers import load_golden, MATERIAL_FIXTURES, build_material_params, material_batch_from_golden, material_rands

pytestmark = pytest.mark.gpu
DEV = 'cuda'
U = 2.0 ** -24
F64, F32 = torch.float64, torch.float32
TINY = 2.0 ** -146         # 8 subnormal ulps: an IDE entry of 1e-41 is computed with gradual underflow
SENT = 0x7fc0dead          # a quiet NaN whose payload no kernel produces
MAX_MSGS = 12
ENTRIES = ('nero_mc_sample', 'nero_mc_classify', 'nero_mc_fill', 'nero_mc_combine_fwd', 'nero_mc_combine_bwd', 'nero_mc_dir_bwd')


# ================================================================================================ device views of the ABI
class _Dev:
    def __init__(self, ptr, shape, typestr):
        self.__cuda_array_interface__ = {'shape': tuple(shape), 'typestr': typestr, 'data': (int(ptr), False), 'version': 2}


def view(ptr, shape, typestr='<f4'):
    """The device buffer at `ptr` as a tensor of `shape` (no copy); None for a null pointer."""
    if math.prod(shape) == 0:
        return torch.zeros(shape, dtype=F32 if typestr == '<f4' else torch.int32, device=DEV)
    if not ptr:
        return None
    return torch.as_tensor(_Dev(ptr, shape, typestr), device=DEV)


def inputs(q):
    """The per-point inputs of a launch, read from its nero_mc_params."""
    P, Sd, Ss = int(q.P), int(q.Sd), int(q.Ss)
    S = Sd + Ss
    f = lambda name, *shape: view(getattr(q, name), shape)
    return dict(P=P, Sd=Sd, Ss=Ss, S=S, N=P * S, ggx=int(q.ggx_smith), sphere=int(q.sphere_dir), human=int(q.human),
                pts=f('pts', P, 3), normals=f('normals', P, 3), view=f('view', P, 3), rough=f('rough', P),
                poses=f('poses', P, 3, 4) if q.human else None, rand_d=f('rand_d', P), rand_s=f('rand_s', P),
                tab_d=f('tab_d', Sd, 2), tab_s=f('tab_s', Ss, 2))


# ================================================================================================ the fp64 restatement
def frame(I, dt):
    n, v = F.normalize(I['normals'].to(dt), dim=-1), F.normalize(I['view'].to(dt), dim=-1)
    return n, v, torch.sum(v * n, -1, keepdim=True) * n * 2 - v          # MCShadingNetwork.forward, field.py:1005-1009


def diffuse_dirs(I, dt):
    n, _, _ = frame(I, dt)
    rd = None if I['rand_d'] is None else I['rand_d'].to(dt)[:, None, None]
    return OM.sample_diffuse_directions(I['tab_d'].to(dt), n, rd)


def specular_dirs(I, dt, a):
    _, _, refl = frame(I, dt)
    rs = None if I['rand_s'] is None else I['rand_s'].to(dt)[:, None, None]
    return OM.sample_specular_directions(I['tab_s'].to(dt), refl, a[:, None], rs)


def brdf(I, d, a, off=None):
    """(w, w (1-HoV)^5) [P,S] of shade_mixed at directions d [P,S,3] and roughness a [P]; `off` moves HoV, NoH, NoL, NoV."""
    dt = d.dtype
    n, v, _ = frame(I, dt)
    Sd, Ss, S = I['Sd'], I['Ss'], I['S']
    n1, v1 = n[:, None], v[:, None]
    H = F.normalize(v1 + d, dim=-1)
    HoV, NoH, NoL = OM.saturate_dot(H, v1), OM.saturate_dot(n1, H), OM.saturate_dot(n1, d)
    if off is not None:
        HoV, NoH, NoL = HoV + off[0], NoH + off[1], NoL + off[2]
    NoV = OM.saturate_dot(n, v).unsqueeze(1)
    if off is not None:
        NoV = NoV + off[3]
    aa = a[:, None, None]
    D = OM.distribution_ggx(NoH, aa)
    prob = torch.cat([NoL[:, :Sd] / np.pi * (Sd / S), D[:, Sd:] * NoH[:, Sd:] / (4 * HoV[:, Sd:] + 1e-5) * (Ss / S)], 1)
    G = OM.geometry_term({'geometry_type': 'ggx_smith' if I['ggx'] else 'schlick'}, NoV, NoL, aa)
    w = D * G / (4 * NoV * prob + 1e-5)
    f5 = torch.clamp(1.0 - HoV, min=0.0, max=1.0) ** 5.0
    return w[..., 0], (w * f5)[..., 0]


def _primal(x):
    return fwAD.unpack_dual(x).primal


def weights(I, dt, off=None, exact=False):
    """[w, wf, dw/da, dwf/da] of every ray: directions valued at DIR (exact=True: the specular ones at the fp64 sampler's
    values), the specular ones differentiated through the sampler."""
    P, Sd = I['P'], I['Sd']
    d0 = I['DIR'].to(dt)
    with fwAD.dual_level():
        a = fwAD.make_dual(I['rough'].to(dt), torch.ones(P, dtype=dt, device=DEV))
        d = d0
        if I['Ss']:
            s = specular_dirs(I, dt, a)
            d = torch.cat([d0[:, :Sd], s if exact else d0[:, Sd:] + (s - _primal(s))], 1)
        out = [fwAD.unpack_dual(x) for x in brdf(I, d, a, off)]
    return [o.primal for o in out] + [torch.zeros_like(o.primal) if o.tangent is None else o.tangent for o in out]


def weights_cond(I):
    """fp64 weights and their cond (see the module docstring)."""
    r64 = weights(I, F64)
    c = [(x32.double() - x64).abs() for x32, x64 in zip(weights(I, F32), r64)]
    for k in range(4):
        off = [0.0, 0.0, 0.0, 0.0]
        off[k] = 4 * U
        c = [ci + (xk - x64).abs() for ci, xk, x64 in zip(c, weights(I, F64, off), r64)]
    # the backward kernel recomputes the specular directions: within DIR's own fp32 error of the exact ones
    c = [ci + (xe - x64).abs() for ci, xe, x64 in zip(c, weights(I, F64, exact=True), r64)]
    return r64, c


def lights(I, B, dt, y_o, y_h, y_i):
    """Per-ray light [P,S,3] of get_lights (field.py:858-884) from the MLP outputs y_*, and a bound of its magnitude."""
    slot = B['slot'].long()
    miss = slot >= 0
    N = slot.numel()
    L = torch.zeros(N, 3, dtype=dt, device=DEV)
    Lm = torch.zeros(N, 3, dtype=F64, device=DEV)
    mi, hi = torch.nonzero(miss)[:, 0], torch.nonzero(~miss)[:, 0]
    if mi.numel():
        ro = slot[mi]
        ol = y_o[ro, :3]
        if I['human']:
            hv = y_h[ro] * B['hhit'][ro].to(dt)[:, None]
            hl, hw = hv[:, :3], torch.clamp(hv[:, 3:], min=0.0, max=1.0)
            L = L.index_put((mi,), ol * (1 - hw) + hl * hw)
            Lm[mi] = (ol.abs() * (1 + hw.abs()) + hl.abs() * hw.abs()).detach().double()
        else:
            L = L.index_put((mi,), ol)
            Lm[mi] = ol.abs().detach().double()
    if hi.numel():
        L = L.index_put((hi,), y_i[~slot[hi], :3])
        Lm[hi] = y_i[~slot[hi], :3].abs().detach().double()
    near = B['near'].to(dt)[:, None]
    P, S = I['P'], I['S']
    return (L * near).view(P, S, 3), (Lm * B['near'].double()[:, None]).view(P, S, 3)


def estimator(L, w, wf, Sd, S):
    return L[:, :Sd].sum(1) / Sd, (L * w[..., None]).sum(1) / S, (L * wf[..., None]).sum(1) / S


def sphere_point(p, d, far):
    pp = torch.where(far[:, None], p * 0.999, p)          # outer_lights 'sphere_direction', field.py:843-853
    return pp + d * O.get_sphere_intersection(pp, d), pp


def human_geo(p, d, poses):
    """The human-light plane mean (before the hit mask), the fp64 hit flag, the flags whose margin is within its delta,
    and delta_mean (field.py:822-836)."""
    inter, dist, hits0 = O.get_camera_plane_intersection(p, d, poses)
    mean = inter[..., :2] * 0.3
    nm = torch.norm(mean, dim=-1)
    hit = hits0 & (nm < 1.5) & (dist > 0)
    R, t = poses[:, :, :3], poses[:, :, 3]
    pp = (R @ p[:, :, None])[..., 0] + t
    rr = (R @ d[:, :, None])[..., 0]
    Mpp = (R.abs() @ p.abs()[:, :, None])[..., 0] + t.abs()
    Mrr = (R.abs() @ d.abs()[:, :, None])[..., 0]
    dpz, drz = 4 * U * Mpp[:, 2], 4 * U * Mrr[:, 2]
    rel = dpz / pp[:, 2].abs() + drz / rr[:, 2].abs().clamp(min=1e-4) + 4 * U
    dmean = 0.3 * (4 * U * Mpp[:, :2].amax(-1) + dist.abs() * (4 * U * Mrr[:, :2].amax(-1) + rr[:, :2].abs().amax(-1) * rel)) + 4 * U * nm
    amb = ((rr[:, 2].abs() - 1e-4).abs() <= drz + 1e-11) | ((nm - 1.5).abs() <= 2 * dmean) | (pp[:, 2].abs() <= dpz) | (rel >= 0.5)
    return mean, hit, amb, dmean


_IDE_T = {}


def ide_bound(xyz, delta):
    """Per-entry bound [R,72] of the kernel's fp32 IDE of xyz [R,3] (module docstring)."""
    if 'mat' not in _IDE_T:
        ml, mat = O.ide_tables(5)
        _IDE_T['m'] = torch.from_numpy(ml[0]).to(DEV, F64)
        _IDE_T['deg'] = torch.from_numpy(ml[1] - ml[0]).to(DEV, F64)
        _IDE_T['mat'] = torch.from_numpy(mat).to(DEV, F64).abs()
    m, deg, mat = _IDE_T['m'], _IDE_T['deg'], _IDE_T['mat']
    k = torch.arange(17, dtype=F64, device=DEV)
    z = xyz[:, 2:3].abs()
    S = (z ** k) @ mat
    S1 = (k * z ** (k - 1).clamp(min=0)) @ mat
    rho = torch.hypot(xyz[:, 0:1], xyz[:, 1:2])
    rm = rho ** m
    rm1 = torch.where(m > 0, m * rho ** (m - 1).clamp(min=0), torch.zeros_like(rm))
    b = 2 * (U * (deg + 3 * m + 6) * rm * S + delta[:, None] * (rm * S1 + rm1 * S))
    return torch.cat([b, b], -1)


def pe_bound(x):
    return torch.full((x.shape[0], 51), 4 * U, dtype=F64, device=DEV)


def ipe_bound(mean, dmean):
    f = 2.0 ** torch.arange(6, dtype=F64, device=DEV).repeat_interleave(2)
    b = f * dmean[:, None] + 4 * U * (2 + f * mean.abs().repeat(1, 6))
    return torch.cat([b, b], -1)


# ================================================================================================ the census
def _bits(t):
    return t.view(torch.int32)


class Census:
    def __init__(self, K):
        self.orig = K
        self.sources = lambda: {}
        self.msgs = []
        self.calls = collections.Counter()
        self.table = {}
        self.allow = collections.Counter()
        self.seen = set()
        self.bwd = {}

    # ------------------------------------------------------------------------------------------ bookkeeping
    def _fail(self, msg):
        if len(self.msgs) < MAX_MSGS:
            self.msgs.append(msg)
        else:
            self.msgs[-1] = f'... and more (last: {msg})'

    def report(self, title):
        lines = [f'--- Monte-Carlo shading census: {title} ({dict(self.calls)})',
                 f'{"kernel":22s} {"buffer":8s} {"checks":>6s} {"max err/bound":>13s}']
        for k in sorted(self.table):
            n, e = self.table[k]
            lines.append(f'{k[0]:22s} {k[1]:8s} {n:6d} {e:13.3f}')
        if self.allow:
            lines.append('counted allowances: ' + ', '.join(f'{k}: {v}' for k, v in sorted(self.allow.items())))
        print('\n'.join(lines))

    def assert_clean(self):
        assert not self.msgs, 'Monte-Carlo shading census found violations:\n  ' + '\n  '.join(self.msgs)

    def check(self, kern, buf, got, ref, bound, where, alt=None, c0=0):
        """got / ref / bound: [R, C] (columns c0.. of the buffer); where(r) names row r.  alt: a second acceptable reference
        (counted allowance rows)."""
        got, ref = got.double().reshape(got.shape[0], -1), ref.double().reshape(got.shape[0], -1)
        bound = torch.as_tensor(bound, dtype=F64, device=DEV).expand_as(ref) if not torch.is_tensor(bound) else bound.double().reshape(ref.shape)
        err = (got - ref).abs()
        if alt is not None:
            err = torch.minimum(err, (got - alt.double().reshape(ref.shape)).abs())
        err = torch.where(torch.isnan(got) != torch.isnan(ref), torch.full_like(err, float('inf')), torch.nan_to_num(err, nan=0.0))
        bound = torch.where(bound > 0, bound + TINY, bound)
        ok = err <= bound
        e = self.table.setdefault((kern, buf), [0, 0.0])
        e[0] += 1
        if err.numel():
            nrm = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, float('inf')), torch.zeros_like(err)))
            e[1] = max(e[1], float(nrm.max()))
        if not bool(ok.all()):
            r, c = torch.nonzero(~ok)[0].tolist()
            self._fail(f'{kern} {buf}: {where(r)}, column {c0 + c}: got {float(got[r, c]):.7e}, want {float(ref[r, c]):.7e}, '
                       f'|err| {float(err[r, c]):.3e} > bound {float(bound[r, c]):.3e} ({int((~ok).sum())} elements)')

    def rays_where(self, S):
        return lambda r: f'point {r // S}, sample {r % S}, ray {r}'

    def rows_where(self, rays, S, what):
        return lambda r: f'point {int(rays[r]) // S}, sample {int(rays[r]) % S}, {what} row {r}'

    @staticmethod
    def point_where(r):
        return f'point {r}'

    # ------------------------------------------------------------------------------------------ written buffers
    def _guard(self, kern, name, ptr, shape, windows, typestr='<f4'):
        """Fill the elements of the written buffer outside `windows` [(rows, c0, c1)] with the sentinel.  The buffer's full
        allocation (rows beyond the declared ones) is used when the caller's sources know it."""
        full = None
        for t in self.sources().values():
            if torch.is_tensor(t) and t.data_ptr() == ptr:
                full = t
        if full is None:
            full = view(ptr, shape, typestr)
        t2 = full.view(full.shape[0], -1)
        keep = torch.ones(t2.shape, dtype=torch.bool, device=DEV)
        for rows, c0, c1 in windows:
            keep[:rows, c0:c1] = False
        snap = t2.clone()
        _bits(t2)[keep] = SENT
        return (kern, name, t2, keep, snap)

    def _unguard(self, g):
        kern, name, t2, keep, snap = g
        bad = keep & (_bits(t2) != SENT)
        if bool(bad.any()):
            r, c = torch.nonzero(bad)[0].tolist()
            self._fail(f'{kern} {name}: write outside the declared windows at row {r}, column {c} of a {tuple(t2.shape)} buffer '
                       f'({int(bad.sum())} elements)')
        t2[keep] = snap[keep]

    def _run(self, guards, run):
        run()
        torch.cuda.synchronize()
        for g in guards:
            self._unguard(g)

    # ------------------------------------------------------------------------------------------ the wrapper
    def K(self, name, *args, **kw):
        if name not in ENTRIES:
            return self.orig(name, *args, **kw)
        self.calls[name] += 1
        self.seen.add(name)
        torch.cuda.synchronize()
        with torch.enable_grad():          # the backward kernels launch from inside autograd's backward pass
            getattr(self, '_' + name[8:])(args[0], lambda: self.orig(name, *args, **kw))

    def _rays(self, q, I):
        N = I['N']
        B = dict(DIR=view(q.dir, (N, 4)), POSD=view(q.pos_depth, (N, 4)), NRMH=view(q.nrm_hit, (N, 4)))
        I['DIR'] = B['DIR'][:, :3].reshape(I['P'], I['S'], 3)
        return B

    # ---- nero_mc_sample
    def _sample(self, q, run):
        I = inputs(q)
        N, S, P, Sd = I['N'], I['S'], I['P'], I['Sd']
        k = 'nero_mc_sample'
        self._run([self._guard(k, 'DIR', q.dir, (N, 4), [(N, 0, 4)]), self._guard(k, 'ORG', q.org, (N, 4), [(N, 0, 4)])], run)
        DIR, ORG = view(q.dir, (N, 4)).double(), view(q.org, (N, 4))
        a = I['rough']
        d64 = torch.cat([diffuse_dirs(I, F64), specular_dirs(I, F64, a.double())], 1).reshape(N, 3)
        d32 = torch.cat([diffuse_dirs(I, F32), specular_dirs(I, F32, a)], 1).reshape(N, 3).double()
        az = torch.cat([I['tab_d'][:, 0], I['tab_s'][:, 0]]).double()[None, :].expand(P, S)
        rnd = torch.zeros(P, S, dtype=F64, device=DEV)
        if I['rand_d'] is not None:
            rnd[:, :Sd] = I['rand_d'].double()[:, None]
        if I['rand_s'] is not None:
            rnd[:, Sd:] = I['rand_s'].double()[:, None]
        phi = (2 * np.pi * (az + rnd)).reshape(N, 1)
        where = self.rays_where(S)
        self.check(k, 'DIR', DIR[:, :3], d64, 2 * (d32 - d64).abs() + 16 * U * (1 + phi), where)
        self.check(k, 'DIR', DIR[:, 3:], torch.zeros(N, 1, device=DEV), 0.0, where, c0=3)
        pts = I['pts'].repeat_interleave(S, 0)
        fused = (pts.double() + DIR[:, :3] * float(np.float32(1e-5))).float()
        plain = pts + DIR[:, :3].float() * np.float32(1e-5)
        self.check(k, 'ORG', ORG[:, :3], fused, 0.0, where, alt=plain)
        self.check(k, 'ORG', ORG[:, 3:], torch.zeros(N, 1, device=DEV), 0.0, where, c0=3)

    # ---- nero_mc_classify
    def _classify(self, q, run):
        I = inputs(q)
        N = I['N']
        nblk = (N + 255) // 256
        k = 'nero_mc_classify'
        gs = [self._guard(k, 'BLKC', q.blk_cnt, (nblk,), [(nblk, 0, 1)], '<i4'),
              self._guard(k, 'BLKO', q.blk_off, (nblk,), [(nblk, 0, 1)], '<i4'),
              self._guard(k, 'COUNTS', q.counts, (2,), [(2, 0, 1)], '<i4')]
        self._run(gs, run)
        hit = view(q.nrm_hit, (N, 4))[:, 3] > 0.5
        cnt = torch.zeros(nblk * 256, dtype=torch.int64, device=DEV)
        cnt[:N] = hit.long()
        cnt = cnt.view(nblk, 256).sum(1)
        off = torch.cumsum(cnt, 0) - cnt
        nh = int(hit.sum())
        where = lambda r: f'block {r}'
        self.check(k, 'BLKC', view(q.blk_cnt, (nblk,), '<i4')[:, None], cnt[:, None], 0.0, where)
        self.check(k, 'BLKO', view(q.blk_off, (nblk,), '<i4')[:, None], off[:, None], 0.0, where)
        self.check(k, 'COUNTS', view(q.counts, (2,), '<i4')[:, None], torch.tensor([[nh], [N - nh]], device=DEV), 0.0,
                   lambda r: ('n_hit', 'n_miss')[r])
        self.assert_clean()        # wrong offsets would send nero_mc_fill's rows out of bounds: stop the step here
        self.feat(I, 'scan blocks > 1024' if nblk > 1024 else None)

    def feat(self, I, extra=None):
        self.seen.add(('S', I['S'] % 32 == 0, I['Ss'] > 32))
        if extra:
            self.seen.add(extra)

    # ---- nero_mc_fill
    def _fill(self, q, run):
        I = inputs(q)
        N, S, P = I['N'], I['S'], I['P']
        B = self._rays(q, I)
        n_hit, n_miss = view(q.counts, (2,), '<i4').tolist()
        k = 'nero_mc_fill'
        ldeo, ldei, ldeh = int(q.ldeo), int(q.ldei), int(q.ldeh)
        gs = [self._guard(k, 'SLOT', q.slot, (N,), [(N, 0, 1)], '<i4'),
              self._guard(k, 'EO', q.EO, (N, ldeo), [(n_miss, 0, 144 if I['sphere'] else 72)]),
              self._guard(k, 'EI', q.EI, (N, ldei), [(n_hit, 0, 124)])]
        if I['human']:
            gs += [self._guard(k, 'EH', q.EH, (N, ldeh), [(n_miss, 0, 24)]), self._guard(k, 'HHIT', q.hhit, (N,), [(n_miss, 0, 1)])]
        self._run(gs, run)
        hit = B['NRMH'][:, 3] > 0.5
        mr, hr = torch.cumsum((~hit).long(), 0) - 1, torch.cumsum(hit.long(), 0) - 1
        want = torch.where(hit, ~hr, mr)
        slot = view(q.slot, (N,), '<i4')
        self.check(k, 'SLOT', slot[:, None], want[:, None], 0.0, self.rays_where(S))
        self.assert_clean()        # a wrong SLOT would make the estimator kernels read rows out of bounds
        miss_rays, hit_rays = torch.nonzero(~hit)[:, 0], torch.nonzero(hit)[:, 0]
        d = B['DIR'][:, :3].double()
        pts = I['pts'].double()
        if n_miss:
            wo = self.rows_where(miss_rays, S, 'outer')
            EO = view(q.EO, (n_miss, ldeo))
            dm = d[miss_rays]
            self.check(k, 'EO', EO[:, :72], O.ide(dm, 0), ide_bound(dm, torch.zeros(n_miss, dtype=F64, device=DEV)), wo)
            pm = pts[miss_rays // S]
            if I['sphere']:
                nrm = torch.norm(pm, dim=-1)
                far = nrm > 0.999
                amb = (nrm - 0.999).abs() < 4 * U
                sp, pp = sphere_point(pm, dm, far)
                sp2, _ = sphere_point(pm, dm, far ^ amb)
                dtx, xtx = (pp * dm).sum(-1), (pp * pp).sum(-1)
                root = torch.sqrt(dtx ** 2 - xtx + 1 + 1e-6)
                bnd = ide_bound(sp, 8 * U * (1 + (dtx ** 2 + xtx + 1) / root))
                self.check(k, 'EO', EO[:, 72:144], O.ide(sp, 0), bnd, wo, alt=O.ide(sp2, 0), c0=72)
                self.allow['sphere |p| = 0.999'] += int(amb.sum())
            if I['human']:
                poses = I['poses'].double()[miss_rays // S]
                mean, hh, amb, dmean = human_geo(pm, dm, poses)
                got_h = view(q.hhit, (n_miss,))
                flip = (got_h > 0.5) != hh
                self.allow['HHIT flip'] += int((flip & amb).sum())
                self.check(k, 'HHIT', got_h[:, None], torch.where(amb, got_h.double(), hh.double())[:, None], 0.0, wo)
                keep = ~flip
                mm = mean * hh[:, None]
                EH = view(q.EH, (n_miss, ldeh))[:, :24]
                ref = O.ipe(mm, torch.zeros_like(mm), 0, 6)
                bnd = ipe_bound(mm, dmean * hh)
                self.check(k, 'EH', EH[keep], ref[keep], bnd[keep], lambda r: wo(int(torch.nonzero(keep)[r, 0])))
        if n_hit:
            wi = self.rows_where(hit_rays, S, 'inner')
            EI = view(q.EI, (n_hit, ldei))
            x = B['POSD'][hit_rays, :3].double()
            self.check(k, 'EI', EI[:, :51], O.embed(x, 8), pe_bound(x), wi)
            self.check(k, 'EI', EI[:, 51:52], torch.zeros(n_hit, 1, device=DEV), 0.0, wi, c0=51)
            refl = reflect(B['NRMH'][hit_rays, :3].double(), d[hit_rays])
            self.check(k, 'EI', EI[:, 52:124], O.ide(refl, 0), ide_bound(refl, torch.full((n_hit,), 16 * U, dtype=F64, device=DEV)), wi, c0=52)
        self.feat(I, 'human' if I['human'] else None)
        if I['sphere']:
            self.seen.add('sphere')

    # ---- the estimator inputs shared by the three estimator kernels
    def _estimator_inputs(self, q, I):
        N = I['N']
        B = self._rays(q, I)
        n_hit, n_miss = view(q.counts, (2,), '<i4').tolist()
        B.update(slot=view(q.slot, (N,), '<i4'), n_hit=n_hit, n_miss=n_miss,
                 OUT_O=view(q.OUT_O, (n_miss, 4)), OUT_I=view(q.OUT_I, (n_hit, 4)),
                 OUT_H=view(q.OUT_H, (n_miss, 4)) if I['human'] else None, hhit=view(q.hhit, (n_miss,)) if I['human'] else None)
        B['near'] = (B['POSD'][:, 3] > np.float32(1e-5)).to(F32)
        if bool((B['POSD'][:, 3] <= np.float32(1e-5)).any()):
            self.seen.add('near mask')
        return B

    # ---- nero_mc_combine_fwd
    def _combine_fwd(self, q, run):
        I = inputs(q)
        P, S, Sd = I['P'], I['S'], I['Sd']
        B = self._estimator_inputs(q, I)
        k = 'nero_mc_combine_fwd'
        self._run([self._guard(k, nm, getattr(q, nm), (P, 3), [(P, 0, 3)]) for nm in ('LD', 'LS', 'LSF')], run)
        (w, wf, _, _), (cw, cwf, _, _) = weights_cond(I)
        y = [None if B[nm] is None else B[nm].double() for nm in ('OUT_O', 'OUT_H', 'OUT_I')]
        L, Lm = lights(I, B, F64, *y)
        LD, LS, LSF = estimator(L, w, wf, Sd, S)
        c = (math.ceil(S / 32) + 12) * U
        b_ld = c * Lm[:, :Sd].sum(1) / Sd
        b_ls = 4 * (Lm * cw[..., None]).sum(1) / S + c * (Lm * w.abs()[..., None]).sum(1) / S
        b_lsf = 4 * (Lm * cwf[..., None]).sum(1) / S + c * (Lm * wf.abs()[..., None]).sum(1) / S
        for nm, ref, b in (('LD', LD, b_ld), ('LS', LS, b_ls), ('LSF', LSF, b_lsf)):
            self.check(k, nm, view(getattr(q, nm), (P, 3)), ref, b, self.point_where)

    # ---- nero_mc_combine_bwd
    def _combine_bwd(self, q, run):
        I = inputs(q)
        P, S, Sd, N = I['P'], I['S'], I['Sd'], I['N']
        B = self._estimator_inputs(q, I)
        n_hit, n_miss = B['n_hit'], B['n_miss']
        k = 'nero_mc_combine_bwd'
        gs = [self._guard(k, 'DPRE_O', q.DPRE_O, (N, 4), [(n_miss, 0, 4)]), self._guard(k, 'DPRE_I', q.DPRE_I, (N, 4), [(n_hit, 0, 4)]),
              self._guard(k, 'dA', q.dA, (P,), [(P, 0, 1)])]
        if I['human']:
            gs.append(self._guard(k, 'DPRE_H', q.DPRE_H, (N, 4), [(n_miss, 0, 4)]))
        self._run(gs, run)
        dLD, dLS, dLSF = (view(getattr(q, nm), (P, 3)).double() for nm in ('dLD', 'dLS', 'dLSF'))
        (w, wf, tw, twf), (cw, cwf, ctw, ctwf) = weights_cond(I)
        y = [None if B[nm] is None else B[nm].double().requires_grad_() for nm in ('OUT_O', 'OUT_H', 'OUT_I')]
        L, Lm = lights(I, B, F64, *y)
        LD, LS, LSF = estimator(L, w, wf, Sd, S)
        loss = (dLD * LD).sum() + (dLS * LS).sum() + (dLSF * LSF).sum()
        leaves = [t for t in y if t is not None]
        grads = dict(zip([nm for nm, t in zip(('O', 'H', 'I'), y) if t is not None], torch.autograd.grad(loss, leaves, allow_unused=True)))
        # per-ray dL = (dLD/Sd [j < Sd] + dLS/S w + dLSF/S wf) near, its magnitude and its cond
        gd, gsp, gf = dLD[:, None] / Sd, dLS[:, None] / S, dLSF[:, None] / S
        isd = (torch.arange(S, device=DEV) < Sd).double()[None, :, None]
        near = B['near'].double().view(P, S, 1)
        dLm = ((gd.abs() * isd + (gsp * w[..., None]).abs() + (gf * wf[..., None]).abs()) * near).reshape(N, 3)
        dLc = (((gsp.abs() * cw[..., None]) + (gf.abs() * cwf[..., None])) * near).reshape(N, 3)
        slot = B['slot'].long()
        miss = slot >= 0
        mi, hi = torch.nonzero(miss)[:, 0], torch.nonzero(~miss)[:, 0]
        # the clamp value the light MLPs' epilogue produces: expf(exp_max) in fp32 on the device
        emax_o, emax_i = float(torch.exp(torch.tensor(q.exp_max_o, device=DEV))), float(torch.exp(torch.tensor(q.exp_max_i, device=DEV)))

        def dpre(nm, rays, yv, g, emax, factor_mag):
            """ref = g y where the output is below fp32 exp(exp_max); outputs AT it may get 0 or g y (counted)."""
            passed = g * yv
            clamped = yv >= emax
            at = yv == emax
            ref = torch.where(clamped & ~at, torch.zeros_like(passed), passed)
            alt = torch.where(at, torch.zeros_like(passed), ref)
            self.allow[f'exp clamp {nm}'] += int(at.sum())
            bound = (4 * dLc[rays] + 12 * U * dLm[rays]) * factor_mag
            return ref, alt, bound

        if n_miss:
            yo = y[0].detach()
            wo = self.rows_where(mi, S, 'outer')
            hw = torch.zeros(n_miss, 1, dtype=F64, device=DEV)
            if I['human']:
                hv = y[1].detach() * B['hhit'].double()[:, None]
                hw = torch.clamp(hv[:, 3:], 0, 1)
            ref, alt, bnd = dpre('DPRE_O', mi, yo[:, :3], grads['O'][:, :3], emax_o, (1 + hw) * yo[:, :3].abs())
            got = view(q.DPRE_O, (n_miss, 4))
            self.check(k, 'DPRE_O', got[:, :3], ref, bnd, wo, alt=alt)
            self.check(k, 'DPRE_O', got[:, 3:], torch.zeros(n_miss, 1, device=DEV), 0.0, wo, c0=3)
            if I['human']:
                yh = y[1].detach()
                hh = B['hhit'].double()[:, None]
                passed = grads['H'] * yh          # exp_max = 0 for the human light: the clamp value is 1
                at = yh == 1.0
                ref = torch.where((yh >= 1.0) & ~at, torch.zeros_like(passed), passed)
                alt = torch.where(at, torch.zeros_like(passed), ref)
                self.allow['exp clamp DPRE_H'] += int(at.sum())
                dl = 4 * dLc[mi] + 12 * U * dLm[mi]
                b3 = (dl * (hv[:, :3].abs() + yo[:, :3].abs())).sum(1, keepdim=True) * hh * yh[:, 3:].abs()
                bnd = torch.cat([dl * hw * hh * yh[:, :3].abs(), b3], 1)
                self.check(k, 'DPRE_H', view(q.DPRE_H, (n_miss, 4)), ref, bnd, wo, alt=alt)
        if n_hit:
            yi = y[2].detach()
            wi = self.rows_where(hi, S, 'inner')
            ref, alt, bnd = dpre('DPRE_I', hi, yi[:, :3], grads['I'][:, :3], emax_i, yi[:, :3].abs())
            got = view(q.DPRE_I, (n_hit, 4))
            self.check(k, 'DPRE_I', got[:, :3], ref, bnd, wi, alt=alt)
            self.check(k, 'DPRE_I', got[:, 3:], torch.zeros(n_hit, 1, device=DEV), 0.0, wi, c0=3)
        # dA: sum_j sum_c L (dLS/S dw/da + dLSF/S dwf/da)
        Ld = L.detach()
        ref = (Ld * (gsp * tw[..., None] + gf * twf[..., None])).sum((1, 2))
        c = (math.ceil(S / 32) + 12) * U
        bnd = 4 * (Lm * (gsp.abs() * ctw[..., None] + gf.abs() * ctwf[..., None])).sum((1, 2)) + \
            c * (Lm * ((gsp * tw[..., None]).abs() + (gf * twf[..., None]).abs())).sum((1, 2))
        self.check(k, 'dA', view(q.dA, (P,))[:, None], ref[:, None], bnd[:, None], self.point_where)
        self.bwd[int(q.dA)] = dict(bound=bnd, L=Ld)

    # ---- nero_mc_dir_bwd
    def _dir_bwd(self, q, run):
        I = inputs(q)
        P, S, Sd, Ss, N = I['P'], I['S'], I['Sd'], I['Ss'], I['N']
        B = self._estimator_inputs(q, I)
        n_hit, n_miss = B['n_hit'], B['n_miss']
        k = 'nero_mc_dir_bwd'
        self._run([self._guard(k, 'dA2', q.dA2, (P,), [(P, 0, 1)])], run)
        E = dict(dEO=view(q.dEO, (n_miss, int(q.ldeo))), dEI=view(q.dEI, (n_hit, int(q.ldei))),
                 dEH=view(q.dEH, (n_miss, int(q.ldeh))) if I['human'] else None)
        spec = torch.arange(Sd, S, device=DEV)
        rays = (torch.arange(P, device=DEV)[:, None] * S + spec[None, :]).reshape(-1)
        ref, bnd = self._dA2(I, B, E, rays)
        self.check(k, 'dA2', view(q.dA2, (P,))[:, None], ref[:, None], bnd[:, None], self.point_where)
        prev = self.bwd.get(int(q.dA))
        if prev is not None:            # the whole step: one autograd of the light path w.r.t. the roughness
            whole = self._whole(I, B, E, rays, prev['L'], q)
            got = view(q.dA, (P,)).double() + view(q.dA2, (P,)).double()
            self.check('dA + dA2 (step)', 'dA+dA2', got[:, None], whole[:, None], (prev['bound'] + bnd)[:, None], self.point_where)
        if Ss > 32:
            self.seen.add('Ss > 32')

    def _enc(self, I, B, E, rays, d, human_mask=None, far_flip=None):
        """Per-ray <dE, E(d)> [R] of the rows the rays landed in; human_mask / far_flip select the allowance variants."""
        S = I['S']
        dt = d.dtype
        slot = B['slot'].long()[rays]
        miss = slot >= 0
        out = torch.zeros(rays.numel(), dtype=dt, device=DEV)
        mi, hi = torch.nonzero(miss)[:, 0], torch.nonzero(~miss)[:, 0]
        if mi.numel():
            dm, ro = d[mi], slot[mi]
            dEO = E['dEO'][ro].to(dt)
            out = out.index_add(0, mi, (dEO[:, :72] * O.ide(dm, 0)).sum(-1))
            pm = I['pts'].to(dt)[rays[mi] // S]
            if I['sphere']:
                nrm = torch.norm(pm.double(), dim=-1)
                far = nrm > 0.999
                if far_flip is not None:
                    far = far ^ ((nrm - 0.999).abs() < 4 * U)
                sp, _ = sphere_point(pm, dm, far)
                out = out.index_add(0, mi, (dEO[:, 72:144] * O.ide(sp, 0)).sum(-1))
            if I['human']:
                poses = I['poses'].to(dt)[rays[mi] // S]
                mean, hh, amb, _ = human_geo(pm, dm, poses)
                hh = hh if human_mask is None else human_mask[mi]
                mm = mean * hh[:, None].to(dt)
                out = out.index_add(0, mi, (E['dEH'][ro, :24].to(dt) * O.ipe(mm, torch.zeros_like(mm), 0, 6)).sum(-1))
        if hi.numel():
            refl = reflect(B['NRMH'][rays[hi], :3].to(dt), d[hi])
            out = out.index_add(0, hi, (E['dEI'][~slot[hi], 52:124].to(dt) * O.ide(refl, 0)).sum(-1))
        return out

    def _spec_tangent(self, I, dt):
        with fwAD.dual_level():
            a = fwAD.make_dual(I['rough'].to(dt), torch.ones(I['P'], dtype=dt, device=DEV))
            t = fwAD.unpack_dual(specular_dirs(I, dt, a)).tangent
        return t.reshape(-1, 3)

    def _dA2(self, I, B, E, rays):
        P, Ss = I['P'], I['Ss']
        if Ss == 0:
            z = torch.zeros(P, dtype=F64, device=DEV)
            return z, z

        def g_at(d0, **kw):
            d = d0.clone().requires_grad_()
            g, = torch.autograd.grad(self._enc(I, B, E, rays, d, **kw).sum(), [d])
            return g
        t64, t32 = self._spec_tangent(I, F64), self._spec_tangent(I, F32).double()
        d64 = B['DIR'][rays, :3].double()
        g = g_at(d64)
        per = (g * t64).sum(-1)
        # the fp32 tangent of the sampler, and the change of g between DIR and the exact direction (the kernel recomputes it)
        ds = specular_dirs(I, F64, I['rough'].double()).reshape(-1, 3)
        cond = 2 * (g * (t32 - t64)).sum(-1).abs() + 2 * ((g_at(ds) - g) * t64).sum(-1).abs()
        # |dE_i| |dE_i/dd_c| by central differences of the encodings, one row pass per component
        mag = torch.zeros(rays.numel(), dtype=F64, device=DEV)
        h = 1e-6
        for c in range(3):
            e = torch.zeros(1, 3, dtype=F64, device=DEV)
            e[0, c] = h
            mag += self._enc_abs_jac(I, B, E, rays, d64, e) * t64[:, c].abs()
        extra = torch.zeros_like(mag)
        if I['human'] and (B['slot'].long()[rays] >= 0).any():
            d = d64.clone().requires_grad_()
            mi = B['slot'].long()[rays] >= 0
            pm = I['pts'].double()[rays // I['S']]
            _, hh, amb, _ = human_geo(pm, d64, I['poses'].double()[rays // I['S']])
            amb = amb & mi
            if bool(amb.any()):
                alt = (g_at(d64, human_mask=hh ^ amb) * t64).sum(-1)
                extra += torch.where(amb, (alt - per).abs(), torch.zeros_like(extra))
                self.allow['HHIT margin (dA2)'] += int(amb.sum())
        if I['sphere']:
            nrm = torch.norm(I['pts'].double(), dim=-1)[rays // I['S']]
            amb = ((nrm - 0.999).abs() < 4 * U) & (B['slot'].long()[rays] >= 0)
            if bool(amb.any()):
                alt = (g_at(d64, far_flip=True) * t64).sum(-1)
                extra += torch.where(amb, (alt - per).abs(), torch.zeros_like(extra))
                self.allow['sphere |p| = 0.999 (dA2)'] += int(amb.sum())
        ref = per.view(P, Ss).sum(1)
        bnd = (cond + 48 * U * mag + extra).view(P, Ss).sum(1)
        return ref, bnd

    def _enc_abs_jac(self, I, B, E, rays, d, e):
        """sum_i |dE_i| |dE_i/dd_c| per ray, with dE_i/dd_c from a central difference of step e."""
        ep, em = self._enc_vec(I, B, E, rays, d + e), self._enc_vec(I, B, E, rays, d - e)
        de = self._enc_vec(I, B, E, rays, d, grads=True)
        return (de.abs() * (ep - em).abs()).sum(-1) / (2 * float(e.abs().max()))

    def _enc_vec(self, I, B, E, rays, d, grads=False):
        """[R, 168] the encodings of each ray's row (IDE | sphere IDE | IPE, or the inner IDE in the first 72), or with
        grads=True the matching dE entries."""
        S = I['S']
        slot = B['slot'].long()[rays]
        miss = slot >= 0
        out = torch.zeros(rays.numel(), 168, dtype=F64, device=DEV)
        mi, hi = torch.nonzero(miss)[:, 0], torch.nonzero(~miss)[:, 0]
        if mi.numel():
            ro = slot[mi]
            dm = d[mi]
            pm = I['pts'].double()[rays[mi] // S]
            if grads:
                out[mi, :72] = E['dEO'][ro, :72].double()
                if I['sphere']:
                    out[mi, 72:144] = E['dEO'][ro, 72:144].double()
                if I['human']:
                    out[mi, 144:168] = E['dEH'][ro, :24].double()
            else:
                out[mi, :72] = O.ide(dm, 0)
                if I['sphere']:
                    out[mi, 72:144] = O.ide(sphere_point(pm, dm, torch.norm(pm, dim=-1) > 0.999)[0], 0)
                if I['human']:
                    mean, hh, _, _ = human_geo(pm, dm, I['poses'].double()[rays[mi] // S])
                    mm = mean * hh[:, None].double()
                    out[mi, 144:168] = O.ipe(mm, torch.zeros_like(mm), 0, 6)
        if hi.numel():
            if grads:
                out[hi, :72] = E['dEI'][~slot[hi], 52:124].double()
            else:
                out[hi, :72] = O.ide(reflect(B['NRMH'][rays[hi], :3].double(), d[hi]), 0)
        return out

    def _whole(self, I, B, E, rays, L, q):
        P, S, Sd = I['P'], I['S'], I['Sd']
        dLS, dLSF = (view(getattr(q, nm), (P, 3)).double() for nm in ('dLS', 'dLSF'))
        a = I['rough'].double().requires_grad_()
        d0 = I['DIR'].double()
        d = d0
        if I['Ss']:
            s = specular_dirs(I, F64, a)
            d = torch.cat([d0[:, :Sd], d0[:, Sd:] + (s - s.detach())], 1)
        w, wf = brdf(I, d, a)
        _, LS, LSF = estimator(L, w, wf, Sd, S)
        loss = (dLS * LS).sum() + (dLSF * LSF).sum()
        if I['Ss']:
            loss = loss + self._enc(I, B, E, rays, d[:, Sd:].reshape(-1, 3)).sum()
        g, = torch.autograd.grad(loss, [a])
        return g


def reflect(nrm, d):
    """inner_lights' reflection (field.py:814-820): view = -d, both normalised."""
    n, v = F.normalize(nrm, dim=-1), F.normalize(-d, dim=-1)
    return torch.sum(v * n, -1, keepdim=True) * n * 2 - v


@pytest.fixture
def census(monkeypatch):
    from nero_b200 import ops, material
    c = Census(ops.K)
    monkeypatch.setattr(material, 'K', c.K)
    return c


# ================================================================================================ part one: training steps
def _net(scfg, mesh, sd=None):
    from nero_b200.material import NeROMaterialRenderer
    net = NeROMaterialRenderer({'shader_cfg': scfg}, is_train=False, mesh=mesh)
    net.load_state_dict(sd if sd is not None else build_material_params(scfg))
    return net.cuda()


def _surface_batch(net, P, seed=6033):
    rays = O.synthetic_rays(4 * P, seed=seed)
    inters, normals, _, hit = net.trace(rays['rays_o'].to(DEV), rays['rays_d'].to(DEV))
    idx = torch.nonzero(hit[:, 0])[:P, 0]
    assert idx.shape[0] == P
    return {'pts': inters[idx].contiguous(), 'rays_d': rays['rays_d'].to(DEV)[idx].contiguous(), 'normals': normals[idx].contiguous(),
            'rgb': rays['rgb'].to(DEV)[idx].contiguous(), 'human_poses': rays['human_poses'].to(DEV)[idx].contiguous()}


def _volume_batch(P, seed, radius):
    """P points inside a ball of `radius` with random normals and view rays."""
    g = torch.Generator().manual_seed(seed)
    pts = F.normalize(torch.randn(P, 3, generator=g), dim=-1) * radius * torch.rand(P, 1, generator=g) ** (1 / 3)
    rays = O.synthetic_rays(P, seed=seed)
    return {'pts': pts.to(DEV), 'rays_d': F.normalize(torch.randn(P, 3, generator=g), dim=-1).to(DEV),
            'normals': F.normalize(torch.randn(P, 3, generator=g), dim=-1).to(DEV), 'rgb': rays['rgb'].to(DEV),
            'human_poses': rays['human_poses'].to(DEV)}


def _step(net, batch, step, rands):
    net.zero_grad()
    out = net.shade_batch(batch, step, rands)
    OM.material_training_loss(out).backward()
    torch.cuda.synchronize()


GGX_SPHERE = {'geometry_type': 'ggx_smith', 'outer_light_version': 'sphere_direction'}
WORKLOADS = list(MATERIAL_FIXTURES) + ['p1024_512_256', 'sd8_ss8_human', 'sd33_ss7_ggx_sphere', 'sd16_ss48_human_sphere',
                                       'eval_mode', 'all_hit', 'all_escape']


@pytest.mark.parametrize('name', WORKLOADS)
def test_training_step_mc_census(name, census):
    """Every nero_mc_* launch of one training step (or one eval-mode forward) against the fp64 restatement."""
    torch.cuda.empty_cache()
    mesh = OM.test_scene(2)
    train = True
    if name in MATERIAL_FIXTURES:                       # the golden fixtures' configurations, batches and random draws
        g = load_golden(name)
        cfg, steps = MATERIAL_FIXTURES[name]
        net = _net(cfg['shader_cfg'], mesh, build_material_params(cfg['shader_cfg'], int(g['seed']), int(g['pseed'])))
        batch = {k: v.to(DEV) for k, v in material_batch_from_golden(g).items()}
        step, rands = steps[-1], {k: v.to(DEV) for k, v in material_rands(g, steps[-1]).items()}
    else:
        scfg = {'diffuse_sample_num': 32, 'specular_sample_num': 16, 'human_lights': True}
        P = 64
        if name == 'p1024_512_256':                     # N = 786 432 rays: 3072 classify blocks, the scan's several-per-thread path
            scfg = dict(GGX_SPHERE, diffuse_sample_num=512, specular_sample_num=256, human_lights=True)
            mesh, P = OM.test_scene(5), 1024
        elif name == 'sd8_ss8_human':
            scfg.update(diffuse_sample_num=8, specular_sample_num=8)
        elif name == 'sd33_ss7_ggx_sphere':
            scfg = dict(GGX_SPHERE, diffuse_sample_num=33, specular_sample_num=7, human_lights=False)
        elif name == 'sd16_ss48_human_sphere':
            scfg = dict(GGX_SPHERE, diffuse_sample_num=16, specular_sample_num=48, human_lights=True)
        net = _net(scfg, mesh if name != 'all_escape' else (mesh[0] + 50.0, mesh[1]))
        if name in ('all_hit', 'all_escape'):
            batch = _volume_batch(P, 11, 0.25)
        else:
            batch = _surface_batch(net, P)
        step, rands = 5000, {k: v.to(DEV) for k, v in OM.draw_rands(P).items()}
        train = name != 'eval_mode'
    census.sources = lambda: net.engine.w
    if train:
        _step(net, batch, step, rands)
    else:
        with torch.no_grad():
            net.shade(batch['pts'], -batch['rays_d'], batch['normals'], batch['human_poses'], False)
    census.report(name)
    want = ENTRIES if train else ENTRIES[:4]
    assert all(census.calls[e] == 1 for e in want), f'the census did not see every kernel once: {dict(census.calls)}'
    n_hit, n_miss = net.engine.w['COUNTS'].tolist()
    if name == 'all_hit':
        assert n_miss == 0 and n_hit > 0
    if name == 'all_escape':
        assert n_hit == 0 and n_miss > 0
    if name == 'p1024_512_256':
        assert 'scan blocks > 1024' in census.seen
    census.assert_clean()


# ================================================================================================ part two: synthetic launches
class Synth:
    """Hand-made nero_mc_params: per-point inputs, hit patterns, depths, MLP outputs and incoming gradients."""

    def __init__(self, P, Sd, Ss, seed, ggx=0, sphere=0, human=0, rand=True, rough=None, norms=None, grazing=False, scale=(1.0, 1.0)):
        from nero_b200 import ops
        from nero_b200.engine import upload_ide_table
        upload_ide_table()
        self.ops = ops
        g = self.g = torch.Generator().manual_seed(seed)
        S = Sd + Ss
        N = self.N = P * S
        self.P, self.Sd, self.Ss, self.S = P, Sd, Ss, S
        n = F.normalize(torch.randn(P, 3, generator=g), dim=-1)
        v = F.normalize(torch.randn(P, 3, generator=g), dim=-1)
        v = torch.where((v * n).sum(-1, keepdim=True) < 0, -v, v)
        if grazing:                                     # NoV ~ 0: the view almost in the tangent plane
            v = F.normalize(v - (v * n).sum(-1, keepdim=True) * n + 1e-4 * n, dim=-1)
        pr = torch.rand(P, 1, generator=g) ** (1 / 3) * 0.9
        if norms is not None:
            pr = torch.tensor(norms, dtype=F32).repeat(P // len(norms) + 1)[:P, None]
        pts = F.normalize(torch.randn(P, 3, generator=g), dim=-1) * pr
        rough = torch.rand(P, generator=g) * 0.96 + 0.04 if rough is None else torch.tensor(rough, dtype=F32).repeat(P // len(rough) + 1)[:P]
        rays = O.synthetic_rays(P, seed=seed)
        z = lambda *s, dt=F32: torch.zeros(*s, dtype=dt, device=DEV)
        extra = 37                                       # rows beyond the declared ones: the sentinel covers them
        ldeo = 192 if sphere else 128
        self.b = dict(pts=pts.to(DEV), normals=(n * scale[0]).to(DEV), view=(v * scale[1]).to(DEV), rough=rough.to(DEV),
                      poses=rays['human_poses'].reshape(P, 12).to(DEV).contiguous(),
                      rand_d=torch.rand(P, generator=g).to(DEV), rand_s=torch.rand(P, generator=g).to(DEV),
                      tab_d=OM.direction_samples(Sd).to(DEV), tab_s=OM.direction_samples(Ss).to(DEV).reshape(Ss, 2),
                      ORG=z(N + extra, 4), DIR=z(N + extra, 4), POSD=z(N, 4), NRMH=z(N, 4), SLOT=z(N + extra, dt=torch.int32),
                      BLKC=z((N + 255) // 256 + 3, dt=torch.int32), BLKO=z((N + 255) // 256 + 3, dt=torch.int32),
                      COUNTS=z(4, dt=torch.int32), EO=z(N + extra, ldeo), EI=z(N + extra, 128), EH=z(N + extra, 64), HHIT=z(N + extra),
                      OUT_O=z(N, 4), OUT_I=z(N, 4), OUT_H=z(N, 4), DPRE_O=z(N + extra, 4), DPRE_I=z(N + extra, 4), DPRE_H=z(N + extra, 4),
                      LD=z(P + 3, 3), LS=z(P + 3, 3), LSF=z(P + 3, 3), dA=z(P + 3), dA2=z(P + 3),
                      dLD=(torch.randn(P, 3, generator=g)).to(DEV), dLS=torch.randn(P, 3, generator=g).to(DEV),
                      dLSF=torch.randn(P, 3, generator=g).to(DEV), dEO=z(N, ldeo), dEI=z(N, 128), dEH=z(N, 64))
        b = self.b
        q = self.q = ops.McParams()
        q.set(pts=b['pts'], normals=b['normals'], view=b['view'], rough=b['rough'], poses=b['poses'] if human else 0,
              rand_d=b['rand_d'] if rand else 0, rand_s=b['rand_s'] if rand else 0, tab_d=b['tab_d'], tab_s=b['tab_s'], P=P, Sd=Sd, Ss=Ss,
              ggx_smith=ggx, sphere_dir=sphere, human=human, org=b['ORG'], dir=b['DIR'], pos_depth=b['POSD'], nrm_hit=b['NRMH'],
              slot=b['SLOT'], blk_cnt=b['BLKC'], blk_off=b['BLKO'], counts=b['COUNTS'], EO=b['EO'], ldeo=ldeo, EI=b['EI'], ldei=128,
              OUT_O=b['OUT_O'], OUT_I=b['OUT_I'], exp_max_o=5.0, exp_max_i=5.0, LD=b['LD'], LS=b['LS'], LSF=b['LSF'],
              DPRE_O=b['DPRE_O'], DPRE_I=b['DPRE_I'], dA=b['dA'], dEO=b['dEO'], dEI=b['dEI'], dA2=b['dA2'],
              dLD=b['dLD'], dLS=b['dLS'], dLSF=b['dLSF'])
        if human:
            q.set(EH=b['EH'], ldeh=64, hhit=b['HHIT'], OUT_H=b['OUT_H'], DPRE_H=b['DPRE_H'], dEH=b['dEH'])

    def run(self, K, hit, depth=None, outputs=None, grazing_hits=False):
        """sample -> hand-made trace (hit [N] bool, depth [N] or None) -> classify -> fill -> hand-made MLP outputs ->
        combine_fwd -> combine_bwd -> hand-made input gradients -> dir_bwd."""
        b, g, N = self.b, self.g, self.N
        K('nero_mc_sample', self.q)
        hit = hit.to(DEV)
        d = b['DIR'][:N, :3]
        nrm = F.normalize(torch.randn(N, 3, generator=g), dim=-1).to(DEV) * (0.5 + 1.5 * torch.rand(N, 1, generator=g).to(DEV))
        if grazing_hits:                                 # hit normals almost perpendicular to the ray: grazing reflections
            nrm = F.normalize(torch.cross(d, nrm, dim=-1), dim=-1) + 1e-3 * d
        nrm = torch.where((nrm * d).sum(-1, keepdim=True) > 0, -nrm, nrm)
        dep = torch.rand(N, generator=g).to(DEV) * 3 + 1e-3 if depth is None else depth.to(DEV)
        b['POSD'][:] = torch.cat([b['ORG'][:N, :3] + d * dep[:, None], dep[:, None]], 1)
        b['POSD'][~hit] = torch.cat([b['ORG'][:N, :3] + d * 10.0, torch.full((N, 1), 10.0, device=DEV)], 1)[~hit]
        if depth is not None:
            b['POSD'][:, 3] = dep
        b['NRMH'][:] = torch.cat([nrm, torch.ones(N, 1, device=DEV)], 1) * hit[:, None]
        K('nero_mc_classify', self.q)
        K('nero_mc_fill', self.q)
        n_hit, n_miss = b['COUNTS'][:2].tolist()
        assert n_hit == int(hit.sum()) and n_miss == N - n_hit
        for nm, n in (('OUT_O', n_miss), ('OUT_I', n_hit), ('OUT_H', n_miss)):
            b[nm][:n] = torch.exp(torch.clamp(torch.randn(n, 4, generator=g) - (1.5 if nm == 'OUT_H' else 0), max=5.0 if nm != 'OUT_H' else 0.0)).to(DEV)
        if outputs is not None:
            outputs(b, n_hit, n_miss)
        K('nero_mc_combine_fwd', self.q)
        K('nero_mc_combine_bwd', self.q)
        for nm, n in (('dEO', n_miss), ('dEI', n_hit), ('dEH', n_miss)):
            b[nm][:n] = (torch.randn(n, b[nm].shape[1], generator=g) * 1e-2).to(DEV)
        K('nero_mc_dir_bwd', self.q)
        return n_hit, n_miss


def _patterns(N, kind, g):
    i = torch.arange(N)
    if kind == 'all_hit':
        return torch.ones(N, dtype=torch.bool)
    if kind == 'all_miss':
        return torch.zeros(N, dtype=torch.bool)
    if kind == 'alternating':
        return i % 2 == 0
    if kind == 'lane31_miss':                            # every warp's only miss is lane 31
        return i % 32 != 31
    if kind == 'last_block':                             # hits only in the last, partial 256-ray block
        return i >= (N - 1) // 256 * 256
    return torch.rand(N, generator=g) < 0.6


PATTERN_CASES = [('all_hit', 37, 16, 16), ('all_miss', 37, 16, 16), ('alternating', 37, 16, 16), ('lane31_miss', 37, 16, 16),
                 ('last_block', 41, 16, 15), ('random', 1, 1, 0), ('random', 1025, 128, 128)]


@pytest.mark.parametrize('case', PATTERN_CASES, ids=[f'{k}-P{p}-S{a}+{b}' for k, p, a, b in PATTERN_CASES])
def test_hit_patterns(case, census):
    """Compaction at every warp / block boundary: all hit, all miss, alternating, a warp whose only miss is lane 31, hits only
    in the last partial block, N = 1, and N = 1025 * 256 rays (1025 blocks: the scan sums two blocks per thread)."""
    kind, P, Sd, Ss = case
    s = Synth(P, Sd, Ss, seed=P + Sd, human=1 if kind != 'random' else 0, sphere=1 if kind in ('alternating', 'last_block') else 0)
    census.sources = lambda: s.b
    s.run(census.K, _patterns(s.N, kind, s.g))
    census.report(f'hit pattern {case}')
    census.assert_clean()


def test_depth_mask_and_exp_clamp(census):
    """POSD.w in {0, 1e-5, nextafter(1e-5, inf), 10}; light outputs at and one ulp below fp32 exp(exp_max); human hw_raw at 0
    and 1.  The exp clamp is decided from the output value: only outputs equal to exp(exp_max) may lose the gradient torch
    passes (counted), one ulp below must keep it."""
    s = Synth(48, 16, 16, seed=5, human=1)
    census.sources = lambda: s.b
    N = s.N
    d1 = float(np.float32(1e-5))
    vals = torch.tensor([0.0, d1, float(np.nextafter(np.float32(1e-5), np.float32(1))), 10.0 - 1e-3], dtype=F32)
    depth = vals.repeat(N // 4 + 1)[:N]
    hit = torch.arange(N) % 3 != 0
    emax = float(torch.exp(torch.tensor(5.0, device=DEV)))
    below = float(np.nextafter(np.float32(emax), np.float32(0)))

    def outputs(b, n_hit, n_miss):
        b['OUT_O'][0:n_miss:5, 0] = emax
        b['OUT_O'][1:n_miss:5, 1] = below
        b['OUT_I'][0:n_hit:5, 2] = emax
        b['OUT_I'][1:n_hit:5, 0] = below
        b['OUT_H'][0:n_miss:7, 3] = 0.0
        b['OUT_H'][1:n_miss:7, 3] = 1.0
        b['OUT_H'][2:n_miss:7, 1] = 1.0
    s.run(census.K, hit, depth, outputs)
    census.report('depth mask and exp clamp')
    census.assert_clean()
    b = s.b
    n_hit, n_miss = b['COUNTS'][:2].tolist()
    # the kernel's choice at the boundary: no gradient at the clamp value, the full gradient one ulp below
    assert bool((b['DPRE_O'][0:n_miss:5, 0] == 0).all()) and bool((b['DPRE_I'][0:n_hit:5, 2] == 0).all())
    slot = b['SLOT'][:N].long()
    near = b['POSD'][:N, 3] > np.float32(1e-5)
    # the census compared the rows one ulp below against the passed gradient; make sure some of them carry one
    assert bool((b['DPRE_O'][1:n_miss:5, 1] != 0).any()) and bool((b['DPRE_I'][1:n_hit:5, 0] != 0).any())
    assert census.allow['exp clamp DPRE_O'] >= len(range(0, n_miss, 5))
    # rays with depth <= 1e-5 contribute nothing: their rows get a zero gradient
    far_rows = slot[(slot >= 0) & ~near]
    assert bool((b['DPRE_O'][far_rows, :3] == 0).all())


GEOMETRY_CASES = [('schlick', {}), ('ggx_sphere', dict(ggx=1, sphere=1, norms=(0.998, 0.999, 1.0))),
                  ('grazing_view', dict(grazing=True, human=1)), ('unnormalised', dict(scale=(3.7, 0.21), ggx=1)),
                  ('eval_no_jitter', dict(rand=False, human=1, sphere=1))]


@pytest.mark.parametrize('case', GEOMETRY_CASES, ids=[c[0] for c in GEOMETRY_CASES])
def test_geometry_edges(case, census):
    """Roughness in {0.02, 0.1, 0.5, 1.0}; grazing views (NoV ~ 0); unnormalised normal and view inputs; points at
    |p| in {0.998, 0.999, 1.0} for sphere_direction; no azimuth jitter; grazing reflections on the rays that hit."""
    name, kw = case
    s = Synth(40, 24, 40, seed=len(name), rough=(0.02, 0.1, 0.5, 1.0), **kw)
    census.sources = lambda: s.b
    s.run(census.K, torch.rand(s.N, generator=s.g) < 0.5, grazing_hits=True)
    census.report(f'geometry {name}')
    assert 'Ss > 32' in census.seen
    census.assert_clean()
