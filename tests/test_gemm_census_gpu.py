"""Census of the wgmma GEMM launches: every nero_chain, nero_linear and nero_wgrad call a real training step makes is
checked against the fp64 restatement of the ABI in gemm_ref.py, on the data that launch actually sees.

Part one wraps ops.chain / ops.linear / ops.wgrad in the modules that call them (engine.py and material.py bind them with
`from .ops import ...`).  Per call the wrapper reads the device row count once (a host sync: the census is eager-only),
snapshots every buffer the launch writes, runs the kernel and then checks
  * each written window against the reference, layer-local for chains: layer l's input is the previous layer's stored
    output (the fp32 value the kernel split into the next A operand) plus the csrc columns; only when the previous
    layer stores nothing is the fp64 reference propagated through it (gemm_ref.py states how its bound carries over);
  * that every element outside the declared windows (save / out, tail, out2 on rows < M) is bit-identical to its
    snapshot;
  * for nero_wgrad, the fp64 dW / bias of every call is accumulated per gradient tensor while its inputs are live and
    compared after the step (and the engine's flush of the deferred finish jobs) on the rows the calls cover.
A failure names the caller (file:line), the tag, the layer, the epilogue kind, the column block of 8 and the row.
Tolerances are stated in gemm_ref.py.

Part two runs the same checks on synthetic layers at the row counts, device counts and layer shapes where the kernels'
tile loops, predicated pair loads and A-operand bookkeeping change paths.
"""
import collections
import gc
import os
import sys
import time

import numpy as np
import pytest
import torch

import gemm_ref as R
import nero_oracle as O
import nero_oracle_mat as OM
from helpers import build_params, build_material_params

pytestmark = pytest.mark.gpu
DEV = 'cuda'
BIG_M = 132 * 128
MAX_MSGS = 12


def _caller(depth):
    f = sys._getframe(depth + 1)
    from nero_b200 import ops
    if f.f_code is ops.mlp.__code__:      # name the line that states the pass, not the runner's launch
        f = f.f_back
    return f'{os.path.basename(f.f_code.co_filename)}:{f.f_lineno}'


def _sid(t):
    return t.untyped_storage().data_ptr()


def _overlap(a, na, b, nb, M):
    """Do columns [c0, c0 + n) of rows [0, M) of two Mats share an element?"""
    if a is None or b is None or na <= 0 or nb <= 0 or M <= 0 or _sid(a.t) != _sid(b.t):
        return False
    la, lb = a.t.stride(0), b.t.stride(0)
    oa, ob = a.t.storage_offset() + a.c0, b.t.storage_offset() + b.c0
    ra, rb = min(M, a.t.shape[0]), min(M, b.t.shape[0])
    if la != lb:
        return oa < ob + (rb - 1) * lb + nb and ob < oa + (ra - 1) * la + na
    d = ob - oa          # need k = i - j with k*ld in (d - na, d + nb), i < ra, j < rb
    kmin = max(-((-(d - na + 1)) // la), -(rb - 1))
    kmax = min((d + nb - 1) // la, ra - 1)
    return kmin <= kmax


def _bits(t):
    return t.view(torch.int32)


class Census:
    def __init__(self, ops):
        self.ops = ops
        self.orig = dict(chain=ops.chain, linear=ops.linear, wgrad=ops.wgrad)
        self.table = {}                 # configuration -> [launches, max normalised error, max rows]
        self.feat = set()
        self.msgs = []
        self.grads = {}
        self.calls = collections.Counter()

    # ------------------------------------------------------------------------------------------ bookkeeping
    def _fail(self, msg):
        if len(self.msgs) < MAX_MSGS:
            self.msgs.append(msg)
        else:
            self.msgs[-1] = f'... and more (last: {msg})'

    def _rows(self, m_ptr, cap):
        M = cap if m_ptr is None else min(int(m_ptr.reshape(-1)[0].item()), cap)
        return max(M, 0)

    def _note(self, key, norm, M):
        e = self.table.setdefault(key, [0, 0.0, 0])
        e[0] += 1
        e[1] = max(e[1], norm)
        e[2] = max(e[2], M)

    def report(self, title):
        lines = [f'--- GEMM census: {title} ({sum(self.calls.values())} launches: {dict(self.calls)})',
                 f'{"entry":7s} {"caller":22s} {"tag":20s} {"layer":>5s} {"kind":14s} {"act":>3s} {"ncol":>4s} {"main":>4s} '
                 f'{"launches":>8s} {"max rows":>9s} {"max err/bound":>13s}']
        for k in sorted(self.table, key=str):
            n, e, m = self.table[k]
            lines.append(f'{k[0]:7s} {k[1]:22s} {k[2]:20s} {k[3]:5d} {k[4]:14s} {k[5]:3d} {k[6]:4d} {k[7]:4d} {n:8d} {m:9d} {e:13.3f}')
        print('\n'.join(lines))

    def assert_clean(self):
        assert not self.msgs, 'GEMM census found violations:\n  ' + '\n  '.join(self.msgs)

    # ------------------------------------------------------------------------------------------ wrappers
    def chain(self, A0, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
        where = _caller(1)
        cap = A0.t.shape[0] if m_cap is None else m_cap
        M = self._rows(m_ptr, cap)
        descs = []
        for i, d in enumerate(layers):
            lay = d['layer']
            W, _ = R.operand(lay, d['transposed'])
            bias = lay.bias_view() if (not d['transposed'] and d['use_bias']) else None
            write_a = bool(d['write_a']) and i + 1 < len(layers)
            n_a = 0
            if write_a:
                nxt = layers[i + 1]
                nk = nxt['layer'].t_chunks if nxt['transposed'] else nxt['layer'].k_chunks
                n_a = max(64 * nk, W.shape[0])          # 'max(16 * a_blocks, n_pad)', a_blocks = 4 * next k_chunks
            addend = None if d['kind'] == R.EK_TANGENT else d['addend']
            descs.append(dict(d, W=W, bias=None if bias is None else bias.double(), write_a=write_a, n_a=n_a, addend=addend,
                              head=(not d['write_a']) and i + 1 < len(layers)))
        self.calls['chain'] += 1
        self._launch('chain', where, tag, A0, R.ceil_div(k_valid0, 4) * 4, descs, M,
                     lambda: self.orig['chain'](A0, k_valid0, layers, m_ptr=m_ptr, m_cap=m_cap, tag=tag))

    def linear(self, A, layer, out, ncol_out, *, transposed=False, mode=R.EPI_BIAS_ACT, act=R.ACT_NONE, act_param=0.0, oscale=1.0,
               H=None, hscale=1.0, dact=R.ACT_NONE, V=None, out2=None, addend=None, ncol_main=None, tail=None, m_ptr=None, m_cap=None,
               use_bias=True):
        where = _caller(1)
        cap = A.t.shape[0] if m_cap is None else m_cap
        M = self._rows(m_ptr, cap)
        kind = R.linear_kind(mode, act, H, dact)
        W, kv = R.operand(layer, transposed)
        bias = layer.bias_view() if (use_bias and not transposed) else None
        bk = kind in R.BIAS_KINDS
        d = dict(layer=layer, kind=kind, ncol_out=ncol_out, ncol_main=ncol_out if ncol_main is None else ncol_main, transposed=transposed,
                 save=out, act=act, act_param=act_param, oscale=oscale, hscale=hscale,
                 H=None if (bk or kind == R.EK_DACT_NONE) else H, V=V if kind == R.EK_TANGENT else None,
                 out2=out2 if kind == R.EK_TANGENT else None, addend=None if bk else addend, tail=None if bk else tail, csrc=None,
                 W=W, bias=None if bias is None else bias.double(), write_a=False, n_a=0, head=False)
        if mode == R.EPI_BIAS_ACT:
            self.feat.add(('linear', 'BIAS_ACT', act))
        elif mode == R.EPI_TANGENT:
            self.feat.add(('linear', 'TANGENT'))
        else:
            self.feat.add(('linear', 'MUL_DACT', 0 if H is None else dact))
            self.feat.add(('linear', 'MUL_DACT', 'tail' if (tail is not None and d['ncol_out'] > d['ncol_main']) else 'no tail'))
        self.calls['linear'] += 1
        self._launch('linear', where, '', A, kv, [d], M,
                     lambda: self.orig['linear'](A, layer, out, ncol_out, transposed=transposed, mode=mode, act=act, act_param=act_param,
                                                 oscale=oscale, H=H, hscale=hscale, dact=dact, V=V, out2=out2, addend=addend,
                                                 ncol_main=ncol_main, tail=tail, m_ptr=m_ptr, m_cap=m_cap, use_bias=use_bias))

    def wgrad(self, ws, dY, n_valid, X, k_valid, layer, grad_w, grad_g, grad_b, dY2=None, X2=None, m_ptr=None, m_cap=None, with_bias=True):
        cap = dY.t.shape[0] if m_cap is None else m_cap
        M = self._rows(m_ptr, cap)
        self.calls['wgrad'] += 1
        if M > BIG_M:
            self.feat.add('big wgrad')
        dW = dWa = db = dba = None
        for r0 in range(0, M, R.CHUNK):
            r1 = min(M, r0 + R.CHUNK)
            part = R.wgrad_layout(dY.view(r1)[r0:], n_valid, X.view(r1)[r0:], k_valid,
                                  None if dY2 is None else dY2.view(r1)[r0:], None if X2 is None else X2.view(r1)[r0:])
            dW, dWa, db, dba = part if dW is None else (dW + part[0], dWa + part[1], db + part[2], dba + part[3])
        if dW is None:
            dW = dWa = torch.zeros(n_valid, k_valid, dtype=torch.float64, device=dY.t.device)
            db = dba = torch.zeros(n_valid, dtype=torch.float64, device=dY.t.device)
        fv, fg, fb = R.wgrad_finish(layer, dW, dWa, db, dba, 2.0 ** -24 * R.ceil_div(max(M, 1), ws.P) ** 0.5)
        rows = slice(layer.row0, layer.row0 + layer.nrows)
        for t, f in ((grad_w, fv), (grad_g, fg), (grad_b if with_bias else None, fb)):
            if t is None or f is None:
                continue
            key = (t.data_ptr(), tuple(t.shape))
            e = self.grads.get(key)
            if e is None:
                z = lambda x: torch.zeros(t.shape[0], x.numel() // x.shape[0], dtype=torch.float64, device=t.device)
                e = self.grads[key] = dict(t=t, snap=t.clone(), ref=z(f[0]), scale=z(f[1]), acc=z(f[2]),
                                           rows=torch.zeros(t.shape[0], dtype=torch.bool, device=t.device))
            for nm, x in zip(('ref', 'scale', 'acc'), f):
                e[nm][rows] += x.reshape(layer.nrows, -1)
            e['rows'][rows] = True
        self.orig['wgrad'](ws, dY, n_valid, X, k_valid, layer, grad_w, grad_g, grad_b, dY2=dY2, X2=X2, m_ptr=m_ptr, m_cap=m_cap,
                           with_bias=with_bias)

    def check_wgrad(self, names):
        torch.cuda.synchronize()
        for key, e in self.grads.items():
            t, m = e['t'], e['rows']
            got = (t.double() - e['snap'].double()).reshape(t.shape[0], -1)[m]
            ok, err, ref = R.frob_ok(got, e['ref'][m], e['scale'][m], e['acc'][m])
            nm = names.get(t.data_ptr(), f'grad@{t.data_ptr():#x}{tuple(t.shape)}')
            self._note(('wgrad', '', nm[-20:], 0, 'FINISH', 0, t.shape[0], int(m.sum())), err / ref if ref > 0 else 0.0, 0)
            if not ok:
                self._fail(f'wgrad {nm}: rows {int(m.sum())} of {t.shape[0]}: ||got - ref||_F = {err:.3e} > bound {ref:.3e}')

    # ------------------------------------------------------------------------------------------ the check
    def _windows(self, descs):
        """(layer, name, Mat, ncol) of every output window the launch declares."""
        out = []
        for li, d in enumerate(descs):
            nmain = d['ncol_out'] if d['kind'] in R.BIAS_KINDS else min(d['ncol_out'], d['ncol_main'])
            d['nmain'] = nmain
            if d['save'] is not None:
                out.append((li, 'save', d['save'], nmain))
            if d['kind'] not in R.BIAS_KINDS and d['tail'] is not None and d['ncol_out'] > d['ncol_main']:
                out.append((li, 'tail', d['tail'], d['ncol_out'] - d['ncol_main']))
            if d['kind'] == R.EK_TANGENT and d['out2'] is not None:
                out.append((li, 'out2', d['out2'], nmain))
        return out

    def _reads(self, li, d):
        r = [('H', d['H'], d['nmain']), ('V', d['V'], d['nmain']), ('addend', d['addend'], d['nmain'])]
        if d['csrc'] is not None and d['write_a'] and d['n_a'] > d['nmain']:
            r.append(('csrc', self.ops.Mat(d['csrc'].t, d['csrc'].c0 + d['nmain'], d['n_a'] - d['nmain']), d['n_a'] - d['nmain']))
        return [x for x in r if x[1] is not None]

    def _launch(self, entry, where, tag, A0, kv0, descs, M, call):
        Mat = self.ops.Mat
        wins = self._windows(descs)
        # a tile runs its layers in order: a layer reading what an earlier layer of the same launch wrote would read the
        # written values.  No call site does that; assert it stays so instead of modelling it
        for i, (la, na, ma, ca) in enumerate(wins):
            for lb, nb, mb, cb in wins[i + 1:]:
                assert not _overlap(ma, ca, mb, cb, M), f'{where} {tag}: output windows of layers {la} ({na}) and {lb} ({nb}) overlap'
        for li, d in enumerate(descs):
            for nm, m, n in self._reads(li, d):
                for lw, nw, mw, cw in wins:
                    if lw < li:
                        assert not _overlap(m, n, mw, cw, M), f'{where} {tag}: layer {li} reads {nm} where layer {lw} writes {nw}'
        # inputs the launch overwrites are cloned before it runs; everything else is read afterwards
        a0 = Mat(A0.t, A0.c0, min(kv0, A0.t.shape[1] - A0.c0))
        inputs = {(-1, 'A0'): a0}
        for li, d in enumerate(descs):
            for nm, m, n in self._reads(li, d):
                inputs[(li, nm)] = Mat(m.t, m.c0, n)
        pre = {}
        for k, m in inputs.items():
            if any(_overlap(m, m.ncol, mw, cw, M) for _, _, mw, cw in wins):
                pre[k] = m.view(M).clone()
                if k[1] == 'addend':
                    self.feat.add('in-place addend')
        # snapshots of the written buffers (rows up to the end of the last row tile)
        snaps = {}
        rows_pad = R.ceil_div(M, 128) * 128
        for _, _, m, _ in wins:
            key = (_sid(m.t), m.t.storage_offset(), tuple(m.t.shape), tuple(m.t.stride()))
            if key not in snaps:
                t = m.t if m.t.numel() <= (1 << 26) else m.t[:max(rows_pad, 1)]
                snaps[key] = (t, t.clone())
        call()
        torch.cuda.synchronize()
        # --- everything outside the declared windows is unchanged
        for key, (t, snap) in snaps.items():
            changed = _bits(t) != _bits(snap)
            ld = t.stride(0)
            for _, _, m, n in wins:
                if _sid(m.t) != key[0] or m.t.stride(0) != ld or M == 0:
                    continue
                delta = m.t.storage_offset() + m.c0 - t.storage_offset()
                r_off, c_off = delta // ld, delta % ld
                changed[max(r_off, 0):max(r_off + M, 0), c_off:c_off + n] = False
            if bool(changed.any()):
                idx = torch.nonzero(changed)[0].tolist()
                self._fail(f'{where} {entry} {tag}: write outside the declared windows at row {idx[0]}, column {idx[1]} of a '
                           f'{tuple(t.shape)} buffer (M = {M})')
        # --- the declared windows against the fp64 reference
        norms = [dict() for _ in descs]
        for r0 in range(0, M, R.CHUNK):
            r1 = min(M, r0 + R.CHUNK)
            m = r1 - r0

            def inp(k):
                if k in pre:
                    return pre[k][r0:r1].double()
                mm = inputs[k]
                return mm.view(r1)[r0:].double()
            kc0 = descs[0]['W'].shape[1]
            A = torch.zeros(m, kc0, dtype=torch.float64, device=DEV)
            n0 = min(a0.ncol, kc0)
            A[:, :n0] = inp((-1, 'A0'))[:, :n0]
            Aabs = A.abs()
            for li, d in enumerate(descs):
                W = d['W']
                kc = W.shape[1]
                acc = A[:, :kc] @ W.t()
                S = Aabs[:, :kc] @ W.abs().t()
                ins = {nm: inp((li, nm)) for nm, _, _ in self._reads(li, d) if nm != 'csrc'}
                nmain, res = R.epilogue(d['kind'], acc, S, d, ins)
                got_main = None
                for name, (ref, bound) in res.items():
                    tgt = d['save'] if name == 'main' else d[name]
                    if tgt is None:
                        continue
                    got = tgt.t[r0:r1, tgt.c0:tgt.c0 + ref.shape[1]].double()
                    if name == 'main':
                        got_main = got
                    self._compare(where, entry, tag, li, d, name, got, ref, bound, r0, norms[li])
                if d['write_a']:
                    An = torch.zeros(m, d['n_a'], dtype=torch.float64, device=DEV)
                    Bn = torch.zeros_like(An)
                    ref, bound = res['main']
                    if got_main is not None:
                        An[:, :nmain], Bn[:, :nmain] = got_main, got_main.abs()
                    else:        # not stored: propagate the fp64 result, its bound enters the next layer's input scale
                        An[:, :nmain], Bn[:, :nmain] = ref, ref.abs() + bound / R.REL
                    if (li, 'csrc') in inputs:
                        c = inp((li, 'csrc'))
                        An[:, nmain:nmain + c.shape[1]], Bn[:, nmain:nmain + c.shape[1]] = c, c.abs()
                    A, Aabs = An, Bn
        # --- coverage and the configuration table
        for li, d in enumerate(descs):
            lay = d['layer']
            kname = R.KIND_NAMES[d['kind']]
            if entry == 'chain':
                self.feat.add(('chain', kname))
                if d['kind'] == R.EK_BIAS_GENERIC:
                    self.feat.add(('chain', 'BIAS_GENERIC', d['act']))
            if d['nmain'] % 2:
                self.feat.add('odd nmain')
            if d['kind'] not in R.BIAS_KINDS and d['tail'] is not None and d['ncol_out'] > d['ncol_main']:
                self.feat.add('tail')
            if d['csrc'] is not None:
                self.feat.add('csrc')
            if d['head']:
                self.feat.add('write_a = 0 head pair')
            if d['save'] is not None and d['save'].c0 > 0:
                self.feat.add('column-offset save')
            if lay.kmap_host is not None and not d['transposed']:
                self.feat.add('kmap layer')
            if M > BIG_M:
                self.feat.add(f'{entry} > 132*128 rows')
            act = d['act'] if d['kind'] == R.EK_BIAS_GENERIC or entry == 'linear' and d['kind'] in R.BIAS_KINDS else 0
            self._note((entry, where, tag[:20], li, kname, act, d['ncol_out'], d['nmain']), max(norms[li].values(), default=0.0), M)

    def _compare(self, where, entry, tag, li, d, name, got, ref, bound, r0, norms):
        err = (got - ref).abs()
        ok = err <= bound
        nrm = torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, float('inf')), torch.zeros_like(err)))
        nrm = torch.where(torch.isnan(nrm), torch.full_like(nrm, float('inf')), nrm)
        if nrm.numel():
            norms[name] = max(norms.get(name, 0.0), float(nrm.max()))
        if not bool(ok.all()):
            i, j = torch.nonzero(~ok)[0].tolist()
            self._fail(f'{where} {entry} {tag!r} layer {li} {R.KIND_NAMES[d["kind"]]} {name}: column block {j // 8} (column {j}), '
                       f'row {r0 + i}: got {float(got[i, j]):.6e}, want {float(ref[i, j]):.6e}, |err| {float(err[i, j]):.3e} > bound '
                       f'{float(bound[i, j]):.3e} ({int((~ok).sum())} elements in this chunk)')


@pytest.fixture
def census(monkeypatch):
    from nero_b200 import ops, engine, material
    c = Census(ops)
    for mod in (ops, engine, material):
        for nm in ('chain', 'linear', 'wgrad'):
            monkeypatch.setattr(mod, nm, getattr(c, nm))
    return c


# ================================================================================================ part one: training steps
SEEN = {}
WORKLOADS = ('bell_30000', 'bell_500_reg', 'bear_human', 'sphere_direction', 'bell_per_layer', 'material')


def _grad_names(params):
    return {p.grad.data_ptr(): n for n, p in params if p.grad is not None}


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, torch.cuda.max_memory_allocated()


def _shape_step(cfg, R_, step):
    from nero_b200.renderer import NeROShapeRenderer
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(cfg))
    net = net.cuda()
    rays = O.synthetic_rays(R_, seed=6033)
    r = {k: v.to(DEV) for k, v in rays.items()}
    c = O.merged_cfg(cfg)
    car = O.get_anneal_val(c, step)

    def run():
        net.zero_grad()
        z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
        out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, step, perm=torch.arange(R_ * z.shape[1], device=DEV))
        O.training_loss(out, r['rgb'], c, step).backward()
    return net, run


def _material_step(P):
    from nero_b200.material import NeROMaterialRenderer
    scfg = {'diffuse_sample_num': 512, 'specular_sample_num': 256, 'outer_light_version': 'sphere_direction', 'geometry_type': 'ggx_smith',
            'light_exp_max': 5.0, 'inner_light_exp_max': 5.0, 'human_lights': True}
    verts, tris = OM.test_scene(5)
    net = NeROMaterialRenderer({'shader_cfg': scfg}, is_train=False, mesh=(verts, tris))
    net.load_state_dict(build_material_params(scfg))
    net = net.cuda()
    rays = O.synthetic_rays(4 * P, seed=6033)
    inters, normals, _, hit = net.trace(rays['rays_o'].to(DEV), rays['rays_d'].to(DEV))
    idx = torch.nonzero(hit[:, 0])[:P, 0]
    assert idx.shape[0] == P
    batch = {'pts': inters[idx].contiguous(), 'rays_d': rays['rays_d'].to(DEV)[idx].contiguous(), 'normals': normals[idx].contiguous(),
             'rgb': rays['rgb'].to(DEV)[idx].contiguous(), 'human_poses': rays['human_poses'].to(DEV)[idx].contiguous()}
    rands = {k: v.to(DEV) for k, v in OM.draw_rands(P).items()}

    def run():
        net.zero_grad()
        out = net.shade_batch(batch, 5000, rands)
        OM.material_training_loss(out).backward()
    return net, run


@pytest.mark.parametrize('name', WORKLOADS)
def test_training_step_gemm_census(name, census, monkeypatch):
    """Every GEMM launch of one eager training step against the fp64 reference (see the module docstring)."""
    from nero_b200 import engine
    gc.collect()                                  # the previous workload's renderer and workspaces (autograd cycles)
    torch.cuda.empty_cache()
    if name == 'bell_30000':
        net, run = _shape_step({}, 1024, 30000)
    elif name == 'bell_500_reg':                  # step < 1000: value_forward / value_backward of init_sdf_reg
        net, run = _shape_step({}, 256, 500)
    elif name == 'bear_human':
        net, run = _shape_step({'shader_config': {'human_light': True}}, 2048, 30000)
    elif name == 'sphere_direction':
        net, run = _shape_step({'shader_config': {'sphere_direction': True}}, 256, 30000)
    elif name == 'bell_per_layer':                # the one-nero_linear-per-layer path kept as the fallback
        monkeypatch.setattr(engine, 'USE_CHAIN', False)
        net, run = _shape_step({}, 1024, 30000)
    else:                                         # stage II at the directions of BASELINE.json configs[3]
        net, run = _material_step(1024)
    # the same step without the census, for its cost
    from nero_b200 import ops, material
    wrapped = [(mod, nm, getattr(mod, nm)) for mod in (ops, engine, material) for nm in ('chain', 'linear', 'wgrad')]
    for mod, nm, _ in wrapped:
        setattr(mod, nm, census.orig[nm])
    t_plain, mem_plain = _peak(run)
    for mod, nm, f in wrapped:
        setattr(mod, nm, f)
    t_cen, mem_cen = _peak(run)
    census.check_wgrad(_grad_names(net.named_parameters()))
    census.report(name)
    print(f'census {name}: step {t_plain * 1e3:.0f} ms / {mem_plain / 2**20:.0f} MiB peak allocated without the census, '
          f'{t_cen:.1f} s / {mem_cen / 2**20:.0f} MiB with it (+{(mem_cen - mem_plain) / 2**20:.0f} MiB)')
    assert census.calls['chain'] + census.calls['linear'] > 0 and census.calls['wgrad'] > 0, 'the census intercepted nothing'
    SEEN[name] = set(census.feat)
    census.grads.clear()
    del net, run
    census.assert_clean()


REQUIRED = ([('chain', k) for k in R.KIND_NAMES] + [('chain', 'BIAS_GENERIC', a) for a in (0, 3, 4)] +
            [('linear', 'BIAS_ACT', a) for a in range(5)] + [('linear', 'MUL_DACT', a) for a in (0, 1, 2)] +
            [('linear', 'MUL_DACT', 'tail'), ('linear', 'MUL_DACT', 'no tail'), ('linear', 'TANGENT')] +
            ['odd nmain', 'tail', 'csrc', 'write_a = 0 head pair', 'in-place addend', 'column-offset save', 'kmap layer',
             'chain > 132*128 rows', 'big wgrad'])


def test_census_coverage():
    """The workloads above together reach every epilogue kind and operand layout the engine uses, so a refactor that stops
    the census from intercepting the launches fails here rather than passing silently."""
    missing_wl = [w for w in WORKLOADS if w not in SEEN]
    if missing_wl:
        pytest.skip(f'coverage is asserted over all training-step workloads; not run: {missing_wl}')
    seen = set().union(*SEEN.values())
    missing = [f for f in REQUIRED if f not in seen]
    assert not missing, f'the census never saw: {missing}'


# ================================================================================================ part two: synthetic edges
def _layer(ops, N, K, seed, wn=True, kmap=None, k_layout=None, t_cols=None):
    g = torch.Generator().manual_seed(seed)
    v = (torch.randn(N, K, generator=g) / np.sqrt(K)).to(DEV)
    gg = (1.0 + 0.1 * torch.randn(N, 1, generator=g)).to(DEV) if wn else None
    b = (0.1 * torch.randn(N, generator=g)).to(DEV)
    L = ops.PreparedLayer(v, gg, b, DEV, kmap=kmap, k_layout=k_layout, t_cols=t_cols)
    L.prep()
    return L


class Bufs:
    """Device buffers of `rows` rows; input rows >= M hold NaN / inf (they must never be read), outputs a sentinel."""

    def __init__(self, rows, M, seed):
        self.rows, self.M = rows, M
        self.g = torch.Generator().manual_seed(seed)

    def inp(self, ncol, scale=1.0, kind='randn', valid_cols=None):
        t = torch.randn(self.rows, ncol, generator=self.g) * scale if kind == 'randn' else torch.rand(self.rows, ncol, generator=self.g) * scale
        t[self.M:] = float('nan')
        t[self.M:, ::3] = float('inf')
        if valid_cols is not None:
            t[:, valid_cols:] = float('nan')
        return t.to(DEV)

    def out(self, ncol):
        return torch.full((self.rows, ncol), -7.0, device=DEV)


KV0 = (4, 40, 124, 144, 256)


def _even(n):
    return n + (n & 1)      # H, V and addend need even leading dimensions (nero_chain / nero_linear reject others)
CASES = [('M', 1), ('M', 127), ('M', 128), ('M', 129), ('M', BIG_M), ('M', BIG_M + 1), ('M', 45001), ('stale', 5000), ('over', 3000),
         ('zero', 2000)]


def _rows_of(case):
    kind, n = case
    if kind == 'M':
        return n, n, None                             # M, m_cap, device count
    if kind == 'stale':
        return n, n + 1000, n
    if kind == 'over':
        return n, n, n + 1000                         # the kernel clamps the device count to m_cap
    return 0, n, 0


def _fwd_chain(ops, B, kv0, long):
    Mat, CL = ops.Mat, ops.chain_layer
    A0 = B.inp(256, 0.5, valid_cols=kv0)
    if long:
        widths = [256, 64, 128, 224, 16, 256, 217, 128, 256]
        kinds = [ops.EK_BIAS_SOFTPLUS, ops.EK_BIAS_RELU, ops.EK_BIAS_GENERIC] * 3
        ls, k = [], 256
        for i, n in enumerate(widths):
            L = _layer(ops, n, k, 100 + i)
            ls.append(CL(L, kinds[i], n, save=Mat(B.out(n + 2), 2), act=(0, 4, 3)[i % 3], act_param=1.0, oscale=0.9))
            k = n
        ls.append(CL(_layer(ops, 3, k, 120), ops.EK_BIAS_GENERIC, 3, act=3, save=Mat(B.out(8), 1), write_a=False))
        return Mat(A0), kv0, ls
    L0, L1 = _layer(ops, 256, 256, 1), _layer(ops, 13, 256, 2)
    L2, L3, L4 = _layer(ops, 217, 16, 3), _layer(ops, 3, 256, 4), _layer(ops, 1, 256, 5)
    skip = B.inp(256, 0.3)
    return Mat(A0), kv0, [CL(L0, ops.EK_BIAS_SOFTPLUS, 256, save=Mat(B.out(256))),
                          CL(L1, ops.EK_BIAS_RELU, 13, save=Mat(B.out(20), 3)),                     # 16-wide, n_a = 64 > n_pad
                          CL(L2, ops.EK_BIAS_GENERIC, 217, act=4, act_param=0.5, oscale=0.70710678, save=Mat(B.out(218), 1),
                             csrc=Mat(skip)),
                          CL(L3, ops.EK_BIAS_GENERIC, 3, act=3, save=Mat(B.out(12), 5), write_a=False),
                          CL(L4, ops.EK_BIAS_GENERIC, 1, act=0, save=Mat(B.out(4), 3))]


def _dact_chain(ops, B, kv0, long):
    Mat, CL = ops.Mat, ops.chain_layer
    A0 = B.inp(256, 1.0, valid_cols=kv0)
    if long:
        widths = [256, 217, 64, 16, 128, 224, 256, 39, 256, 128, 256]
        kinds = [ops.EK_DACT_SOFTPLUS, ops.EK_DACT_RELU, ops.EK_DACT_NONE]
        ls = []
        for i in range(10):
            k_in, n = widths[i], widths[i + 1]
            L = _layer(ops, k_in, n, 200 + i, t_cols=(0, n))
            kd = kinds[i % 3]
            H = Mat(B.inp(_even(n + 2), 0.05, kind='rand'), 2) if kd != ops.EK_DACT_NONE else None
            add = Mat(B.inp(_even(n + 1), 0.5)) if i % 2 else None
            ls.append(CL(L, kd, n, transposed=True, H=H, hscale=1.41421356, oscale=0.8, addend=add, save=Mat(B.out(n + 3), 3)))
        return Mat(A0), kv0, ls
    La = _layer(ops, 256, 256, 11, t_cols=(0, 256))
    Lb = _layer(ops, 256, 16, 12, t_cols=(0, 16))
    Lc = _layer(ops, 16, 256, 13, t_cols=(0, 256))
    Ld = _layer(ops, 256, 40, 14, t_cols=(0, 40))
    io = B.inp(256, 0.5)
    dx = B.inp(64, 0.5)
    dx[:, 39:] = 0.0
    return Mat(A0), kv0, [
        CL(La, ops.EK_DACT_SOFTPLUS, 256, transposed=True, oscale=0.70710678, H=Mat(B.inp(256, 0.05, kind='rand')), hscale=1.41421356,
           ncol_main=217, tail=Mat(B.out(40)), save=Mat(B.out(256)), csrc=Mat(B.inp(256, 0.3))),
        CL(Lb, ops.EK_DACT_RELU, 13, transposed=True, H=Mat(B.inp(16, 1.0)), addend=Mat(B.inp(16, 0.5)), save=Mat(B.out(16), 2)),
        CL(Lc, ops.EK_DACT_NONE, 251, transposed=True, addend=Mat(io), save=Mat(io)),              # in place at an odd limit
        CL(Ld, ops.EK_DACT_NONE, 39, transposed=True, addend=Mat(dx), save=Mat(dx))]


def _tangent_chain(ops, B, kv0, long):
    Mat, CL = ops.Mat, ops.chain_layer
    A0 = B.inp(256, 1.0, valid_cols=kv0)
    widths = [256, 217, 64, 16, 128, 256, 224, 39, 128, 256] if long else [256, 217, 16, 256]
    ls, k = [], 256
    for i, n in enumerate(widths):
        L = _layer(ops, n, k, 300 + i)
        csrc = Mat(B.inp(256, 0.3)) if n % 2 else None
        ls.append(CL(L, ops.EK_TANGENT, n, use_bias=False, oscale=0.9 if i % 2 else 1.0, H=Mat(B.inp(_even(n + 1), 0.04, kind='rand')),
                     hscale=1.41421356 if i % 2 else 1.0, V=Mat(B.inp(_even(n + 1), 1.0)), out2=Mat(B.out(n + 4), 4),
                     save=Mat(B.out(n + 1), 1), csrc=csrc))
        k = n
    return Mat(A0), kv0, ls


def _linear_calls(ops, census, B, kv0, m_ptr, m_cap):
    Mat = ops.Mat
    kmap = list(range(51)) + [52 + i for i in range(72)] if kv0 == 124 else None
    Lf = _layer(ops, 217, 123 if kmap else kv0, 21, kmap=kmap, k_layout=124 if kmap else None)
    A = Mat(B.inp(kv0 + 8, 0.5, valid_cols=Lf.k_valid))
    for act in range(5):
        census.linear(A, Lf, Mat(B.out(220), 1), 217, act=act, act_param=0.5, oscale=0.9, m_ptr=m_ptr, m_cap=m_cap)
    L16 = _layer(ops, 13, kv0, 22)
    census.linear(Mat(B.inp(kv0, 0.5)), L16, Mat(B.out(13)), 13, act=2, m_ptr=m_ptr, m_cap=m_cap)
    Lt = _layer(ops, 256, 256, 23, t_cols=(0, 256))
    dY = Mat(B.inp(256, 1.0))
    H = Mat(B.inp(256, 0.05, kind='rand'))
    census.linear(dY, Lt, Mat(B.out(256)), 256, transposed=True, mode=ops.EPI_MUL_DACT, oscale=0.70710678, H=H, hscale=1.41421356,
                  dact=1, addend=Mat(B.inp(256, 0.5)), ncol_main=217, tail=Mat(B.out(40)), m_ptr=m_ptr, m_cap=m_cap)
    census.linear(dY, Lt, Mat(B.out(256), 2), 213, transposed=True, mode=ops.EPI_MUL_DACT, H=Mat(B.inp(256, 1.0)), dact=2,
                  addend=Mat(B.inp(214, 0.5)), m_ptr=m_ptr, m_cap=m_cap)
    io = B.inp(256, 0.5)
    census.linear(dY, Lt, Mat(io), 251, transposed=True, mode=ops.EPI_MUL_DACT, addend=Mat(io), m_ptr=m_ptr, m_cap=m_cap)
    census.linear(dY, Lt, Mat(B.out(256)), 255, transposed=True, mode=ops.EPI_TANGENT, H=H, hscale=1.0, dact=1, V=Mat(B.inp(256, 1.0)),
                  out2=Mat(B.out(256)), m_ptr=m_ptr, m_cap=m_cap)


@pytest.mark.parametrize('family', ['forward', 'dact', 'tangent', 'linear'])
@pytest.mark.parametrize('ci', range(len(CASES)), ids=[f'{k}{n}' for k, n in CASES])
def test_gemm_edges_against_fp64(family, ci, census):
    """Row counts around the 128-row tile and the 132-CTA grid, device counts below / above / at zero with NaN and inf in
    every stale input row, odd and even main widths (the two ld2 paths), 16-wide layers inside chains, in-place addends at
    odd limits and first layers reading k_valid0 in {4, 40, 124, 144, 256} columns."""
    from nero_b200 import ops
    M, cap, dev_count = _rows_of(CASES[ci])
    kv0 = KV0[ci % len(KV0)]
    B = Bufs(cap + 64, M, seed=ci)
    m_ptr = None if dev_count is None else torch.tensor([dev_count], dtype=torch.int32, device=DEV)
    if family == 'linear':
        _linear_calls(ops, census, B, kv0, m_ptr, cap)
    else:
        build = {'forward': _fwd_chain, 'dact': _dact_chain, 'tangent': _tangent_chain}[family]
        A0, k, ls = build(ops, B, kv0, False)
        census.chain(A0, k, ls, m_ptr=m_ptr, m_cap=cap, tag=f'{family} {CASES[ci]}')
    census.assert_clean()


@pytest.mark.parametrize('family', ['forward', 'dact', 'tangent'])
def test_ten_layer_chain_against_fp64(family, census):
    from nero_b200 import ops
    M, cap = 45001, 46000
    B = Bufs(cap + 64, M, seed=7)
    build = {'forward': _fwd_chain, 'dact': _dact_chain, 'tangent': _tangent_chain}[family]
    A0, k, ls = build(ops, B, 144, True)
    assert len(ls) == 10
    census.chain(A0, k, ls, m_ptr=torch.tensor([M], dtype=torch.int32, device=DEV), m_cap=cap, tag=f'{family} x10')
    census.report(f'ten-layer {family} chain')
    census.assert_clean()
