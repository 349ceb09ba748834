"""Stage II (material estimation) on the H100: `NeROMaterialRenderer` with the reference's API.

Reference being replaced (paths relative to /root/reference):
  NeROMaterialRenderer.__init__/trace/shade/train_step   network/renderer.py:666-848
  MCShadingNetwork.forward/shade_mixed/get_lights        network/field.py:858-1009
  MCShadingNetwork.predict_materials / material_regularization   field.py:896-903, 1061-1087
  MaterialFeatsNetwork                                   field.py:660-689
  raytracing.RayTracer (third party)                     renderer.py:676,720  -> k_bvh.cu

Python sequences kernels and keeps the [P,3]-sized glue (sRGB, losses) in torch autograd; the 768 rays per surface
point, their tracing, encodings, the three light MLPs and the estimator run in hand-written kernels with hand-written
backward passes (`_LightsFn`); the material MLPs are `_MaterialsFn`.  Parameter gradients are accumulated by the
kernels directly into `param.grad` (one flat buffer, `engine.Grads`), as in stage I.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
# linear is not called here (see the note on chain in engine.py): it stays bound for the GEMM census
from .ops import Mat, K, linear, wgrad, chain, mlp, chain_layer as CL, ACT_SIGMOID, ACT_EXPCLAMP
from .ops import EK_BIAS_RELU, EK_BIAS_GENERIC, EK_DACT_RELU
from .engine import Predictor, Grads, upload_ide_table, _linear_to_srgb_torch
from .params import MCShadingParams

MISS_DEPTH = 10.0       # the reference treats depth >= 10 as a miss (network/renderer.py:727)
O_MET, O_ROUGH, O_ALB, O_LD_ = 0, 4, 8, 12


def read_ply(path):
    """Minimal PLY reader (ascii / binary_little_endian; vertex x y z + triangular faces) for cfg['mesh']
    (the reference uses open3d.io.read_triangle_mesh, network/renderer.py:675)."""
    with open(path, 'rb') as f:
        header = []
        while True:
            line = f.readline().decode('ascii', 'replace').strip()
            header.append(line)
            if line == 'end_header':
                break
        fmt = [l.split()[1] for l in header if l.startswith('format')][0]
        if fmt not in ('ascii', 'binary_little_endian'):
            raise NotImplementedError(f'PLY format {fmt}')
        elems, cur = [], None
        for l in header:
            t = l.split()
            if t and t[0] == 'element':
                cur = [t[1], int(t[2]), []]
                elems.append(cur)
            elif t and t[0] == 'property' and cur is not None:
                cur[2].append(t[1:])
        npt = {'char': 'i1', 'uchar': 'u1', 'short': 'i2', 'ushort': 'u2', 'int': 'i4', 'uint': 'u4', 'float': 'f4', 'double': 'f8',
               'int8': 'i1', 'uint8': 'u1', 'int16': 'i2', 'uint16': 'u2', 'int32': 'i4', 'uint32': 'u4', 'float32': 'f4', 'float64': 'f8'}
        verts = tris = None
        for name, n, props in elems:
            if name == 'vertex':
                if fmt == 'ascii':
                    rows = np.array([f.readline().split() for _ in range(n)], dtype=np.float64)
                    names = [p[-1] for p in props]
                    verts = rows[:, [names.index(c) for c in 'xyz']]
                else:
                    dt = np.dtype([(p[-1], '<' + npt[p[0]]) for p in props])
                    raw = np.frombuffer(f.read(dt.itemsize * n), dtype=dt)
                    verts = np.stack([raw['x'], raw['y'], raw['z']], -1)
            elif name == 'face':
                if fmt == 'ascii':
                    tris = np.array([f.readline().split()[1:4] for _ in range(n)], dtype=np.int64)
                else:
                    lp = props[0]
                    assert lp[0] == 'list' and len(props) == 1, 'only a single vertex-index list per face is supported'
                    ct, it = np.dtype('<' + npt[lp[1]]), np.dtype('<' + npt[lp[2]])
                    dt = np.dtype([('n', ct), ('v', it, (3,))])
                    raw = np.frombuffer(f.read(dt.itemsize * n), dtype=dt)
                    assert (raw['n'] == 3).all(), 'non-triangular faces'
                    tris = raw['v']
            else:
                raise NotImplementedError(f'PLY element {name}')
    return np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(tris, np.int32)


class FeatsNet:
    """MaterialFeatsNetwork (field.py:660-689): PE8 -> 4 x ReLU(256) -> cat with PE8 -> 3 x ReLU(256) -> 256 (linear)."""

    def __init__(self, fp, dev):
        ls = fp.layers()
        mk = lambda l, **kw: ops.PreparedLayer(l.weight_v, l.weight_g, l.bias, dev, **kw)
        self.L0 = [mk(ls[0])] + [mk(l, t_cols=(0, 256)) for l in ls[1:4]]
        self.L1 = [mk(ls[4], t_cols=(0, 256))] + [mk(l, t_cols=(0, 256)) for l in ls[5:8]]
        self.pl = ls

    def prep(self):
        for l in self.L0 + self.L1:
            l.prep()

    def forward(self, w, M):
        A, B = w['FA'], w['FB']
        mlp(Mat(w['FX']),
            [CL(self.L0[0], EK_BIAS_RELU, 256, save=Mat(A[0])), CL(self.L0[1], EK_BIAS_RELU, 256, save=Mat(A[1])),
             CL(self.L0[2], EK_BIAS_RELU, 256, save=Mat(A[2])),
             CL(self.L0[3], EK_BIAS_RELU, 256, save=Mat(w['FCAT']), write_a=False)], None, M, tag='feats_a')
        # the second half reads cat([h, PE8]): K = 307
        mlp(Mat(w['FCAT']),
            [CL(self.L1[0], EK_BIAS_RELU, 256, save=Mat(B[0])), CL(self.L1[1], EK_BIAS_RELU, 256, save=Mat(B[1])),
             CL(self.L1[2], EK_BIAS_RELU, 256, save=Mat(B[2])),
             CL(self.L1[3], EK_BIAS_GENERIC, 256, save=Mat(w['FY']), write_a=False)], None, M, tag='feats_b')

    def backward(self, ws, w, M):
        """w['dFY'][:, :256] holds d(feats); accumulates all 8 layers' parameter gradients."""
        A, B, G = w['FA'], w['FB'], w['FG']
        chain(Mat(w['dFY']), 256,
              [CL(self.L1[3], EK_DACT_RELU, 256, transposed=True, H=Mat(B[2]), save=Mat(G[6])),
               CL(self.L1[2], EK_DACT_RELU, 256, transposed=True, H=Mat(B[1]), save=Mat(G[5])),
               CL(self.L1[1], EK_DACT_RELU, 256, transposed=True, H=Mat(B[0]), save=Mat(G[4])),
               CL(self.L1[0], EK_DACT_RELU, 256, transposed=True, H=Mat(w['FCAT']), save=Mat(G[3])),
               CL(self.L0[3], EK_DACT_RELU, 256, transposed=True, H=Mat(A[2]), save=Mat(G[2])),
               CL(self.L0[2], EK_DACT_RELU, 256, transposed=True, H=Mat(A[1]), save=Mat(G[1])),
               CL(self.L0[1], EK_DACT_RELU, 256, transposed=True, H=Mat(A[0]), save=Mat(G[0]))], None, M, tag='feats_bwd')
        g = lambda l: (l.weight_v.grad, l.weight_g.grad, l.bias.grad)
        P = self.pl
        kw = dict(m_cap=M)
        wgrad(ws, Mat(w['dFY']), 256, Mat(B[2]), 256, self.L1[3], *g(P[7]), **kw)
        wgrad(ws, Mat(G[6]), 256, Mat(B[1]), 256, self.L1[2], *g(P[6]), **kw)
        wgrad(ws, Mat(G[5]), 256, Mat(B[0]), 256, self.L1[1], *g(P[5]), **kw)
        wgrad(ws, Mat(G[4]), 256, Mat(w['FCAT']), self.L1[0].k_valid, self.L1[0], *g(P[4]), **kw)
        wgrad(ws, Mat(G[3]), 256, Mat(A[2]), 256, self.L0[3], *g(P[3]), **kw)
        wgrad(ws, Mat(G[2]), 256, Mat(A[1]), 256, self.L0[2], *g(P[2]), **kw)
        wgrad(ws, Mat(G[1]), 256, Mat(A[0]), 256, self.L0[1], *g(P[1]), **kw)
        wgrad(ws, Mat(G[0]), 256, Mat(w['FX']), self.L0[0].k_valid, self.L0[0], *g(P[0]), **kw)


class MaterialEngine:
    """Owns the BVH, the prepared tensor-core operands of every stage-II MLP and the per-step workspaces."""

    def __init__(self, shader: MCShadingParams, verts, tris, dev):
        ops.require_cuda(dev)
        self.p, self.dev = shader, dev
        c = self.cfg = shader.cfg
        if c['outer_light_version'] not in ('direction', 'sphere_direction'):
            raise NotImplementedError(c['outer_light_version'])
        if c['geometry_type'] not in ('schlick', 'ggx_smith'):
            raise NotImplementedError(c['geometry_type'])
        upload_ide_table()
        self.human = bool(c['human_lights'])
        self.sphere = c['outer_light_version'] == 'sphere_direction'
        self.Sd, self.Ss = int(c['diffuse_sample_num']), int(c['specular_sample_num'])
        self.tab_d = shader.diffuse_direction_samples.to(dev).contiguous()
        self.tab_s = shader.specular_direction_samples.to(dev).contiguous()
        # geometry
        self.verts, self.tris = np.ascontiguousarray(verts, np.float32), np.ascontiguousarray(tris, np.int32)
        nodes, tri, _ = ops.bvh_build(self.verts, self.tris)
        self.bvh_nodes = torch.from_numpy(nodes).to(dev)
        self.bvh_tris = torch.from_numpy(tri).to(dev)
        # networks
        self.feats = FeatsNet(shader.feats_network, dev)
        self.m_met = Predictor(shader.metallic_predictor, dev, 1, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        self.m_rough = Predictor(shader.roughness_predictor, dev, 1, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        self.m_alb = Predictor(shader.albedo_predictor, dev, 3, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        ko = 144 if self.sphere else 72
        self.exp_o, self.exp_i = float(c['light_exp_max']), float(c['inner_light_exp_max'])
        self.m_outer = Predictor(shader.outer_light, dev, 3, ACT_EXPCLAMP, self.exp_o, k_layout=ko, t_cols=(0, ko))
        self.m_inner = Predictor(shader.inner_light, dev, 3, ACT_EXPCLAMP, self.exp_i,
                                 kmap=list(range(51)) + [52 + i for i in range(72)], k_layout=124, t_cols=(52, 72))
        self.m_human = Predictor(shader.human_light, dev, 4, ACT_EXPCLAMP, 0.0, k_layout=24, t_cols=(0, 24)) if self.human else None
        self.grads = Grads(list(shader.parameters()))
        self.ws = None
        self.w, self.cap = {}, None
        self.mw, self.mcap = {}, None

    def predictors(self):
        return [m for m in (self.m_met, self.m_rough, self.m_alb, self.m_outer, self.m_inner, self.m_human) if m is not None]

    def prepare_weights(self):
        if getattr(self, '_all_layers', None) is None:
            ls = self.feats.L0 + self.feats.L1
            for m in self.predictors():
                ls += m.layers
            self._all_layers = ops.PrepBatch(ls)
        self._all_layers.run()

    # ------------------------------------------------------------------ tracing (renderer.py:719-729)
    def trace(self, rays_o, rays_d):
        o = rays_o.reshape(-1, 3).to(self.dev, torch.float32).contiguous()
        d = rays_d.reshape(-1, 3).to(self.dev, torch.float32).contiguous()
        n = o.shape[0]
        pos = torch.empty(n, 4, device=self.dev)
        nrm = torch.empty(n, 4, device=self.dev)
        K('nero_bvh_trace', self.bvh_nodes, self.bvh_tris, n, o, 3, d, 3, pos, nrm, MISS_DEPTH, 1)
        depth = pos[:, 3:4].clone()
        return pos[:, :3].clone(), nrm[:, :3].clone(), depth, ~(depth >= MISS_DEPTH)

    # ------------------------------------------------------------------ material MLPs
    def _alloc_materials(self, M):
        if self.mcap is not None and self.mcap >= M:      # workspaces only grow
            return
        z = lambda *s: torch.zeros(*s, device=self.dev)
        names = ['met', 'rough', 'alb']
        self.mw = dict(FX=z(M, 64), FCAT=z(M, 320), FY=z(M, 320), dFY=z(M, 320), OUT=z(M, 12), DOUT=z(M, 12),
                       FA=[z(M, 256) for _ in range(3)], FB=[z(M, 256) for _ in range(3)], FG=[z(M, 256) for _ in range(7)],
                       ACT={k: [z(M, 256) for _ in range(3)] for k in names}, dHa=z(M, 256), dHb=z(M, 256), dHc=z(M, 256))
        self.mcap = M
        if self.ws is None:
            self.ws = ops.WgradWorkspace(self.dev)
            self.ws.defer = True

    def materials_forward(self, pts):
        """predict_materials before the roughness rescale: sigmoid outputs (metallic [M,1], roughness [M,1], albedo [M,3])."""
        M = pts.shape[0]
        self._alloc_materials(M)
        w = self.mw
        K('nero_mat_prep', pts, M, w['FX'], 64, w['FCAT'], 320, w['FY'], 320)
        self.feats.forward(w, M)
        y = Mat(w['FY'])
        self.m_met.forward(y, w['ACT']['met'], Mat(w['OUT'], O_MET), None, M)
        self.m_rough.forward(y, w['ACT']['rough'], Mat(w['OUT'], O_ROUGH), None, M)
        self.m_alb.forward(y, w['ACT']['alb'], Mat(w['OUT'], O_ALB), None, M)
        o = w['OUT'][:M]
        self.m_rows = M
        return o[:, O_MET:O_MET + 1].clone(), o[:, O_ROUGH:O_ROUGH + 1].clone(), o[:, O_ALB:O_ALB + 3].clone()

    def materials_backward(self, d_met, d_rough, d_alb):
        w, M = self.mw, self.m_rows
        self.grads.ensure()
        o, d = w['OUT'][:M], w['DOUT'][:M]
        sg = lambda y, g: g * y * (1.0 - y)          # sigmoid'(x) from the post-activation value
        d[:, O_MET:O_MET + 1] = sg(o[:, O_MET:O_MET + 1], d_met)
        d[:, O_ROUGH:O_ROUGH + 1] = sg(o[:, O_ROUGH:O_ROUGH + 1], d_rough)
        d[:, O_ALB:O_ALB + 3] = sg(o[:, O_ALB:O_ALB + 3], d_alb)
        y, dy = Mat(w['FY']), Mat(w['dFY'])
        dH = (w['dHa'], w['dHb'], w['dHc'])
        dm = w['DOUT']
        self.m_rough.backward(self.ws, Mat(dm, O_ROUGH), y, w['ACT']['rough'], dH, None, M, dX=dy, dx_ncol=256)
        self.m_met.backward(self.ws, Mat(dm, O_MET), y, w['ACT']['met'], dH, None, M, dX=dy, dx_ncol=256, dx_addend=dy)
        self.m_alb.backward(self.ws, Mat(dm, O_ALB), y, w['ACT']['alb'], dH, None, M, dX=dy, dx_ncol=256, dx_addend=dy)
        self.feats.backward(self.ws, w, M)
        self.ws.flush()

    # ------------------------------------------------------------------ Monte-Carlo lights
    def _alloc_lights(self, P):
        if self.cap is not None and self.cap >= P:        # workspaces only grow
            return
        S = self.Sd + self.Ss
        N = P * S
        dev = self.dev
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        nblk = (N + 255) // 256
        ldeo = 192 if self.sphere else 128
        w = dict(ORG=z(N, 4), DIR=z(N, 4), POSD=z(N, 4), NRMH=z(N, 4), SLOT=z(N, dt=torch.int32), BLKC=z(nblk, dt=torch.int32),
                 BLKO=z(nblk, dt=torch.int32), COUNTS=z(2, dt=torch.int32), EO=z(N, ldeo), EI=z(N, 128), dEO=z(N, ldeo), dEI=z(N, 128),
                 OUT_O=z(N, 4), OUT_I=z(N, 4), DPRE_O=z(N, 4), DPRE_I=z(N, 4), LD=z(P, 3), LS=z(P, 3), LSF=z(P, 3), dA=z(P), dA2=z(P),
                 ACT=[z(N, 256) for _ in range(3)], dH=[z(N, 256) for _ in range(3)])
        if self.human:
            w.update(EH=z(N, 64), dEH=z(N, 64), HHIT=z(N), OUT_H=z(N, 4), DPRE_H=z(N, 4), ACTH=[z(N, 256) for _ in range(3)])
        self.w, self.cap, self.ldeo = w, P, ldeo
        if self.ws is None:
            self.ws = ops.WgradWorkspace(dev)
            self.ws.defer = True

    def _params(self, st):
        w = self.w
        q = ops.McParams()
        q.set(pts=st['pts'], normals=st['normals'], view=st['view'], rough=st['rough'], poses=st['poses'] if self.human else 0,
              rand_d=st['rand_d'] if st['rand_d'] is not None else 0, rand_s=st['rand_s'] if st['rand_s'] is not None else 0,
              tab_d=self.tab_d, tab_s=self.tab_s, P=st['P'], Sd=self.Sd, Ss=self.Ss, ggx_smith=1 if self.cfg['geometry_type'] == 'ggx_smith' else 0,
              sphere_dir=1 if self.sphere else 0, human=1 if self.human else 0, org=w['ORG'], dir=w['DIR'], pos_depth=w['POSD'],
              nrm_hit=w['NRMH'], slot=w['SLOT'], blk_cnt=w['BLKC'], blk_off=w['BLKO'], counts=w['COUNTS'], EO=w['EO'], ldeo=self.ldeo,
              EI=w['EI'], ldei=128, OUT_O=w['OUT_O'], OUT_I=w['OUT_I'], exp_max_o=self.exp_o, exp_max_i=self.exp_i, LD=w['LD'], LS=w['LS'],
              LSF=w['LSF'], DPRE_O=w['DPRE_O'], DPRE_I=w['DPRE_I'], dA=w['dA'], dEO=w['dEO'], dEI=w['dEI'], dA2=w['dA2'])
        if self.human:
            q.set(EH=w['EH'], ldeh=64, hhit=w['HHIT'], OUT_H=w['OUT_H'], DPRE_H=w['DPRE_H'], dEH=w['dEH'])
        return q

    def lights_forward(self, pts, normals, view, rough, poses, rand_d, rand_s):
        """Means over the sampled directions of the traced / predicted lights: LD (diffuse samples), LS (all, x specular
        weight), LSF (x weight x (1-HoV)^5) -- each [P,3] (field.py:932-984)."""
        P = pts.shape[0]
        self._alloc_lights(P)
        w = self.w
        S = self.Sd + self.Ss
        N = P * S
        st = dict(P=P, pts=pts.contiguous(), normals=normals.contiguous(), view=view.contiguous(), rough=rough.reshape(-1).contiguous(),
                  poses=poses.reshape(P, 12).contiguous() if (self.human and poses is not None) else None,
                  rand_d=None if rand_d is None else rand_d.reshape(-1).contiguous(),
                  rand_s=None if rand_s is None else rand_s.reshape(-1).contiguous())
        q = self._params(st)
        K('nero_mc_sample', q)
        K('nero_bvh_trace', self.bvh_nodes, self.bvh_tris, N, w['ORG'], 4, w['DIR'], 4, w['POSD'], w['NRMH'], MISS_DEPTH, 1)
        K('nero_mc_classify', q)
        n_hit, n_miss = w['COUNTS'].tolist()            # the one host sync of the step
        st.update(n_hit=n_hit, n_miss=n_miss)
        K('nero_mc_fill', q)
        A = w['ACT']
        if n_miss > 0:
            self.m_outer.forward(Mat(w['EO']), [a[:n_miss] for a in A], Mat(w['OUT_O']), None, n_miss)
            if self.human:
                self.m_human.forward(Mat(w['EH']), w['ACTH'], Mat(w['OUT_H']), None, n_miss)
        if n_hit > 0:
            self.m_inner.forward(Mat(w['EI']), [a[n_miss:] for a in A], Mat(w['OUT_I']), None, n_hit)
        K('nero_mc_combine_fwd', q)
        self.state = st
        return w['LD'][:P].clone(), w['LS'][:P].clone(), w['LSF'][:P].clone()

    def human_lights_output(self):
        """outputs['human_lights'] of shade_mixed (field.py:988): hl*hw of every escaping ray, or zeros [1,3]."""
        n_miss = self.state['n_miss']
        if n_miss == 0:
            return torch.zeros(1, 3, device=self.dev)
        if not self.human:
            return torch.zeros(n_miss, 3, device=self.dev)
        h = self.w['OUT_H'][:n_miss] * self.w['HHIT'][:n_miss, None]
        return h[:, :3] * torch.clamp(h[:, 3:], min=0.0, max=1.0)

    def lights_backward(self, dLD, dLS, dLSF):
        """-> d(loss)/d(roughness) [P]; accumulates the light MLPs' parameter gradients."""
        st, w = self.state, self.w
        self.grads.ensure()
        n_hit, n_miss = st['n_hit'], st['n_miss']
        q = self._params(st)
        q.set(dLD=dLD.contiguous(), dLS=dLS.contiguous(), dLSF=dLSF.contiguous())
        K('nero_mc_combine_bwd', q)
        A, D = w['ACT'], w['dH']
        if n_miss > 0:
            ko = 144 if self.sphere else 72
            self.m_outer.backward(self.ws, Mat(w['DPRE_O']), Mat(w['EO']), [a[:n_miss] for a in A], [d[:n_miss] for d in D], None, n_miss,
                                  dX=Mat(w['dEO']), dx_ncol=ko)
            if self.human:
                self.m_human.backward(self.ws, Mat(w['DPRE_H']), Mat(w['EH']), w['ACTH'], [d[:n_miss] for d in D], None, n_miss,
                                      dX=Mat(w['dEH']), dx_ncol=24)
        if n_hit > 0:
            self.m_inner.backward(self.ws, Mat(w['DPRE_I']), Mat(w['EI']), [a[n_miss:] for a in A], [d[n_miss:] for d in D], None, n_hit,
                                  dX=Mat(w['dEI'], 52), dx_ncol=72)
        self.ws.flush()
        K('nero_mc_dir_bwd', q)
        return w['dA'][:st['P']] + w['dA2'][:st['P']]


class _MaterialsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, pts, *params):
        ctx.engine = engine
        ctx.n = len(params)
        return engine.materials_forward(pts)

    @staticmethod
    def backward(ctx, d_met, d_rough, d_alb):
        ctx.engine.materials_backward(d_met, d_rough, d_alb)
        return (None, None) + (None,) * ctx.n


class _LightsFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, engine, rough, pts, normals, view, poses, rand_d, rand_s, *params):
        ctx.engine = engine
        ctx.n = len(params)
        return engine.lights_forward(pts, normals, view, rough.detach(), poses, rand_d, rand_s)

    @staticmethod
    def backward(ctx, dLD, dLS, dLSF):
        d_rough = ctx.engine.lights_backward(dLD, dLS, dLSF)
        return (None, d_rough.reshape(-1, 1)) + (None,) * (6 + ctx.n)


class NeROMaterialRenderer(nn.Module):
    default_cfg = {
        'train_ray_num': 512, 'test_ray_num': 1024, 'database_name': 'real/bear/raw_1024', 'rgb_loss': 'charbonier',
        'mesh': 'data/meshes/bear_shape-300000.ply', 'shader_cfg': {}, 'reg_mat': True, 'reg_diffuse_light': True,
        'reg_diffuse_light_lambda': 0.1, 'fixed_camera': False,
    }

    def __init__(self, cfg, is_train=True, mesh=None):
        """cfg / is_train as the reference (network/renderer.py:666-672).  `mesh=(verts, tris)` supplies the geometry directly
        instead of reading cfg['mesh']; is_train=True additionally needs the host repo's `dataset` package."""
        super().__init__()
        self.cfg = {**self.default_cfg, **cfg}
        self.warned_normal = False
        self._mesh = mesh if mesh is not None else read_ply(self.cfg['mesh'])
        self.cfg['shader_cfg'] = dict(self.cfg['shader_cfg'])
        self.cfg['shader_cfg']['is_real'] = str(self.cfg['database_name']).startswith('real')
        self.shader_network = MCShadingParams(self.cfg['shader_cfg'])
        self._engine = None
        if is_train:
            self._init_dataset(is_train)

    # ------------------------------------------------------------------ engine plumbing
    @property
    def engine(self):
        if self._engine is None:
            dev = self.shader_network.light_pts.device
            ops.require_cuda(dev, 'NeROMaterialRenderer')
            self._engine = MaterialEngine(self.shader_network, self._mesh[0], self._mesh[1], dev)
        return self._engine

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._engine = None
        return out

    # ------------------------------------------------------------------ reference API
    def trace(self, rays_o, rays_d):
        """renderer.py:719-729: (inters, normals flipped+normalised, depth [n,1], hit_mask [n,1])."""
        return self.engine.trace(rays_o, rays_d)

    def trace_in_batch(self, rays_o, rays_d, batch_size=1024 ** 2, cpu=False):
        outs = [[], [], [], []]
        for ri in range(0, rays_o.shape[0], batch_size):
            cur = self.trace(rays_o[ri:ri + batch_size], rays_d[ri:ri + batch_size])
            for o, c in zip(outs, cur):
                o.append(c.cpu() if cpu else c)
        return tuple(torch.cat(o, 0) for o in outs)

    def get_human_coordinate_poses(self, poses):
        from .renderer import NeROShapeRenderer
        return NeROShapeRenderer.get_human_coordinate_poses(self, poses)

    def compute_rgb_loss(self, rgb_pr, rgb_gt):
        if self.cfg['rgb_loss'] == 'l1':
            return torch.sum(F.l1_loss(rgb_pr, rgb_gt, reduction='none'), -1)
        if self.cfg['rgb_loss'] == 'charbonier':
            return torch.sqrt(torch.sum((rgb_gt - rgb_pr) ** 2, dim=-1) + 0.001)
        raise NotImplementedError

    def compute_diffuse_light_regularization(self, diffuse_lights):
        white = torch.sum(torch.abs(diffuse_lights - torch.mean(diffuse_lights, dim=-1, keepdim=True)), dim=-1)
        return white * self.cfg['reg_diffuse_light_lambda']

    def query_materials(self, pts):
        """MCShadingNetwork.predict_materials (field.py:896-903) on arbitrary points (no gradient bookkeeping)."""
        e = self.engine
        e.prepare_weights()
        with torch.no_grad():
            m, r, a = e.materials_forward(pts.reshape(-1, 3).float().contiguous())
        return m, r * (1.0 - 0.04 ** 2) + 0.04 ** 2, a

    def predict_materials(self, batch_size=8192):
        """Per-vertex materials of the mesh for the export scripts (renderer.py:903-915): sqrt of the predicted (squared)
        roughness, numpy arrays."""
        verts = torch.from_numpy(self._mesh[0]).to(self.shader_network.light_pts.device)
        outs = {'metallic': [], 'roughness': [], 'albedo': []}
        for vi in range(0, verts.shape[0], batch_size):
            m, r, a = self.query_materials(verts[vi:vi + batch_size])
            outs['metallic'].append(m.cpu().numpy())
            outs['roughness'].append(torch.sqrt(torch.clamp(r, min=1e-7)).cpu().numpy())
            outs['albedo'].append(a.cpu().numpy())
        return {k: np.concatenate(v, 0) for k, v in outs.items()}

    def export_lighting(self, width=1024, height=512, ssaa=4, center=(0.0, 0.0, 0.0), trans=False, max_rows=None):
        """The outer (environment) light as a CUDA float32 [height, width, 3] map in relight's convention (nero_b200/envmap.py):
        outer_light(IDE(d, 0)) (field.py:836-854), with sphere_direction seen from `center`; trans=True gives the map
        tools/relight.py --trans expects.  The inner light and the human light are not part of it."""
        from . import envmap as EM
        c = self.shader_network.cfg
        ol = EM.OuterLight(self.shader_network.outer_light, c['light_exp_max'],
                           'stage2' if c['outer_light_version'] == 'sphere_direction' else None)
        return ol.map(width, height, ssaa, 0.0, center, EM.trans_frame(trans), max_rows or EM.MAX_ROWS)

    def shade(self, pts, view_dirs, normals, human_poses, is_train, step=None, rands=None):
        """MCShadingNetwork.forward + material_regularization inputs (field.py:1005-1009, renderer.py:804-807).
        `rands` (optional dict rand_d, rand_s, rand_ang, rand_eps) replaces the in-function random draws."""
        e, c = self.engine, self.shader_network.cfg
        dev = e.dev
        e.prepare_weights()
        params = list(self.shader_network.parameters())
        P = pts.shape[0]
        pts = pts.float().contiguous()
        rands = dict(rands or {})
        jitter = is_train and c['random_azimuth']
        if jitter and 'rand_d' not in rands:        # same draw order as field.py:782, 805
            rands['rand_d'] = torch.rand(P, 1, 1, device=dev)
            rands['rand_s'] = torch.rand(P, 1, 1, device=dev)
        want_reg = is_train and self.cfg['reg_mat'] and c['reg_change']
        if want_reg:
            n = F.normalize(normals, dim=-1)
            x = _orthogonal(n)
            y = torch.cross(n, x, dim=-1)
            ang = (rands['rand_ang'] if 'rand_ang' in rands else torch.rand(P, 1, device=dev)) * np.pi * 2
            if c['change_type'] == 'constant':
                change = (torch.cos(ang) * x + torch.sin(ang) * y) * c['change_eps']
            elif c['change_type'] == 'gaussian':
                eps = rands['rand_eps'] if 'rand_eps' in rands else torch.normal(mean=0.0, std=c['change_eps'], size=[P, 1], device=dev)
                change = (torch.cos(ang) * x + torch.sin(ang) * y) * eps
            else:
                raise NotImplementedError
            query = torch.cat([pts, pts + change], 0).contiguous()
        else:
            query = pts
        met, rough_raw, alb = _MaterialsFn.apply(e, query, *params)
        rough = rough_raw * (1.0 - 0.04 ** 2) + 0.04 ** 2
        metallic, roughness, albedo = met[:P], rough[:P], alb[:P]
        LD, LS, LSF = _LightsFn.apply(e, roughness, pts, normals.float().contiguous(), view_dirs.float().contiguous(), human_poses,
                                      rands.get('rand_d') if jitter else None, rands.get('rand_s') if jitter else None, *params)
        F0 = 0.04 * (1 - metallic) + metallic * albedo
        kd = 1 - metallic
        spec_col = F0 * LS + (1.0 - F0) * LSF
        diff_col = albedo * kd * LD
        srgb = _linear_to_srgb_torch
        cl = lambda x: torch.clamp(srgb(x), min=0, max=1)
        spec_c = cl(spec_col)
        out = {'albedo': albedo, 'roughness': roughness, 'metallic': metallic, 'human_lights': e.human_lights_output(),
               'diffuse_light': cl(LD), 'specular_light': cl(LS), 'diffuse_color': cl(diff_col), 'specular_color': spec_c,
               'approximate_light': cl(kd * LD + spec_c), 'rgb_pr': srgb(diff_col + spec_col)}
        if want_reg:
            self._reg_pair = (met[P:], rough[P:], alb[P:])
        return out

    def _material_regularization(self, out, step):
        """field.py:1061-1087 given the second (perturbed) material query made in shade()."""
        c = self.shader_network.cfg
        reg = 0
        if c['reg_change']:
            m0, r0, a0 = self._reg_pair
            reg = reg + torch.mean((torch.abs(m0 - out['metallic']) + torch.abs(r0 - out['roughness']) + torch.abs(a0 - out['albedo'])) *
                                   c['reg_lambda1'], dim=1)
        if c['reg_min_max'] and step is not None and step < 2000:
            r, m = out['roughness'], out['metallic']
            reg = reg + torch.sum(torch.clamp(r - 0.98 ** 2, min=0)) + torch.sum(torch.clamp(0.02 ** 2 - r, min=0))
            reg = reg + torch.sum(torch.clamp(m - 0.98, min=0)) + torch.sum(torch.clamp(0.02 - m, min=0))
        return reg

    def shade_batch(self, batch, step, rands=None):
        """train_step (renderer.py:825-848) on an explicit batch {pts, rays_d, normals, rgb, human_poses}."""
        out = self.shade(batch['pts'], -batch['rays_d'], batch['normals'], batch['human_poses'], True, step, rands)
        out['rgb_gt'] = batch['rgb']
        out['loss_rgb'] = self.compute_rgb_loss(out['rgb_pr'], out['rgb_gt'])
        if self.cfg['reg_mat']:
            out['loss_mat_reg'] = self._material_regularization(out, step)
        if self.cfg['reg_diffuse_light']:
            out['loss_diffuse_light'] = self.compute_diffuse_light_regularization(out['diffuse_light'])
        return out

    # ------------------------------------------------------------------ dataset plumbing (host repo)
    def _init_dataset(self, is_train):
        """renderer.py:680-699 -- needs the reference's `dataset` package on sys.path (drop-in scenario)."""
        from dataset.database import parse_database_name, get_database_split     # noqa: provided by the host repo
        from network.renderer import build_imgs_info, imgs_info_to_torch
        self.database = parse_database_name(self.cfg['database_name'])
        self.train_ids, self.test_ids = get_database_split(self.database, 'validation')
        self.train_ids = np.asarray(self.train_ids)
        if is_train:
            self.train_imgs_info = imgs_info_to_torch(build_imgs_info(self.database, self.train_ids), 'cpu')
            self.test_imgs_info = imgs_info_to_torch(build_imgs_info(self.database, self.test_ids), 'cpu')
            self.train_num, self.test_num = len(self.train_ids), len(self.test_ids)
            self.train_batch = self._construct_ray_batch(self.train_imgs_info)
            self.tbn = self.train_batch['rays_o'].shape[0]
            self._shuffle_train_batch()

    def _construct_ray_batch(self, imgs_info, device='cpu', is_train=True):
        """renderer.py:756-802: camera rays of every pixel traced onto the mesh (primary hits = the training set)."""
        imn, _, h, w = imgs_info['imgs'].shape
        ys, xs = torch.meshgrid(torch.arange(h), torch.arange(w), indexing='ij')
        coords = torch.stack([xs, ys], -1).float()[None].repeat(imn, 1, 1, 1).reshape(imn, h * w, 2)
        coords = torch.cat([coords + 0.5, torch.ones(imn, h * w, 1)], 2)
        rays_d = coords @ torch.inverse(imgs_info['Ks']).permute(0, 2, 1)
        poses = imgs_info['poses']
        R, t = poses[:, :, :3], poses[:, :, 3:]
        rays_d = F.normalize(rays_d @ R, dim=-1)
        rays_o = (-R.permute(0, 2, 1) @ t).permute(0, 2, 1).repeat(1, h * w, 1)
        inters, normals, depth, hit = self.trace_in_batch(rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), cpu=True)
        inters, normals, depth, hit = inters.reshape(imn, h * w, 3), normals.reshape(imn, h * w, 3), depth.reshape(imn, h * w, 1), hit.reshape(imn, h * w)
        hp = self.get_human_coordinate_poses(poses).unsqueeze(1).repeat(1, h * w, 1, 1)
        rgb = imgs_info['imgs'].reshape(imn, 3, h * w).permute(0, 2, 1)
        pick = (lambda v: v[hit]) if is_train else (lambda v: v[0])
        batch = {'rays_o': pick(rays_o), 'rays_d': pick(rays_d), 'inters': pick(inters), 'normals': pick(normals), 'depth': pick(depth),
                 'human_poses': pick(hp), 'rgb': pick(rgb)}
        if not is_train:
            assert imn == 1
            batch['hit_mask'] = hit[0]
        return {k: v.to(device) for k, v in batch.items()}

    def _shuffle_train_batch(self):
        self.train_batch_i = 0
        idx = torch.randperm(self.tbn, device='cpu')
        for k, v in self.train_batch.items():
            self.train_batch[k] = v[idx]

    def train_step(self, step):
        rn = self.cfg['train_ray_num']
        dev = self.shader_network.light_pts.device
        i = self.train_batch_i
        tb = {k: self.train_batch[k][i:i + rn].to(dev, non_blocking=True) for k in ('inters', 'rays_d', 'normals', 'rgb', 'human_poses')}
        out = self.shade_batch({'pts': tb['inters'], 'rays_d': tb['rays_d'], 'normals': tb['normals'], 'rgb': tb['rgb'],
                                'human_poses': tb['human_poses']}, step)
        self.train_batch_i += rn
        if self.train_batch_i + rn >= self.tbn:
            self._shuffle_train_batch()
        return out

    def render_rays(self, ray_batch, h, w):
        """The chunk loop of test_step (renderer.py:854-885) over an is_train=False ray batch (with 'hit_mask')."""
        dev = self.shader_network.light_pts.device
        rb = {k: v.to(dev) for k, v in ray_batch.items()}
        trn = self.cfg['test_ray_num']
        keys = {'rgb_gt': 3, 'rgb_pr': 3, 'specular_light': 3, 'specular_color': 3, 'diffuse_light': 3, 'diffuse_color': 3, 'albedo': 3,
                'metallic': 1, 'roughness': 1}
        outs = {k: [] for k in keys}
        rn = rb['rays_o'].shape[0]
        with torch.no_grad():
            for ri in range(0, rn, trn):
                hit = rb['hit_mask'][ri:ri + trn]
                cur = {k: torch.zeros(hit.shape[0], d, device=dev) for k, d in keys.items()}
                if torch.sum(hit) > 0:
                    sl = lambda k: rb[k][ri:ri + trn][hit]
                    so = self.shade(sl('inters'), -sl('rays_d'), sl('normals'), sl('human_poses'), False)
                    cur['rgb_gt'][hit] = sl('rgb')
                    for k in ('rgb_pr', 'specular_light', 'specular_color', 'diffuse_color', 'diffuse_light', 'albedo', 'metallic'):
                        cur[k][hit] = so[k]
                    cur['roughness'][hit] = torch.sqrt(so['roughness'])      # predictions are squared roughness
                for k in keys:
                    outs[k].append(cur[k])
        return {k: torch.cat(v, 0).reshape(h, w, -1) for k, v in outs.items()}

    def test_step(self, index):
        """renderer.py:850-887 (needs the host repo's database for the test image)."""
        from network.renderer import imgs_info_slice
        info = imgs_info_slice(self.test_imgs_info, torch.from_numpy(np.asarray([index], np.int64)))
        _, _, h, w = info['imgs'].shape
        return self.render_rays(self._construct_ray_batch(info, 'cpu', False), h, w)

    def forward(self, data):
        if 'eval' in data:        # renderer.py:889-901
            return self.test_step(data['index'])
        return self.train_step(data['step'])


def _orthogonal(d):
    """get_orthogonal_directions (field.py:755-766)."""
    x, y, z = torch.split(d, 1, dim=-1)
    zero = torch.zeros_like(x)
    o0, o1 = torch.cat([y, -x, zero], -1), torch.cat([-z, zero, x], -1)
    pick0 = (torch.norm(o0, dim=-1) > torch.norm(o1, dim=-1)).unsqueeze(-1)
    return F.normalize(torch.where(pick0, o0, o1), dim=-1)
