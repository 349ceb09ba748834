"""Host-side orchestration of the stage-I hot path on one H100: sample_ray + render_core forward / backward.

Python only sequences kernels: every arithmetic step is a hand-written sm_90a kernel reached through the C ABI
(ops.K / ops.linear / ops.wgrad).  Data-dependent sizes (number of inner / outer samples) stay on the device:
workspaces are sized for the worst case and kernels read the live counts from device memory.

Reference call graph being replaced (paths relative to /root/reference):
  NeROShapeRenderer.sample_ray   network/renderer.py:403-443  -> ShapeEngine.sample_ray
  NeROShapeRenderer.render_core  network/renderer.py:550-606  -> ShapeEngine.render_core_forward / _backward
  SDFNetwork.forward/.gradient   network/field.py:130-167     -> SdfNet.forward_with_gradient (+ tangent/backward sweeps)
  AppShadingNetwork.forward      network/field.py:591-651     -> ShapeEngine._shade_forward / _shade_backward
  NeRFNetwork.forward            network/field.py:258-283     -> NerfNet.forward / backward
  compute_occ_loss/get_intersection  renderer.py:522-548, field.py:432-484 -> ShapeEngine._occ_forward
Buffer layouts are documented in DESIGN.md section 3.
"""
import math

import numpy as np
import torch

from . import ops
# chain is not called here (the passes launch through ops.mlp); it stays bound, like in material.py, because the GEMM census
# wraps chain / linear / wgrad by patching these names in ops, engine and material
from .ops import Mat, K, linear, wgrad, chain, mlp, chain_layer as CL, ACT_NONE, ACT_RELU, ACT_SIGMOID, ACT_EXPCLAMP, EPI_MUL_DACT
from .ops import EK_BIAS_SOFTPLUS, EK_BIAS_RELU, EK_BIAS_GENERIC, EK_DACT_SOFTPLUS, EK_DACT_RELU, EK_DACT_NONE, EK_TANGENT

# Every stage-I MLP pass is stated once, as the layer list of the fused chain kernel (k_gemm_chain.cu).  True: ops.mlp runs
# it as nero_chain launches; False: ops.mlp expands the same list into one nero_linear launch per layer
USE_CHAIN = True

INV_SQRT2 = 0.7071067811865476
SQRT2 = 1.4142135623730951
# E buffer columns (k_shade.cu)
E_PE6R, E_PE8X, E_IDER, E_IDEN, E_LD = 0, 40, 92, 164, 240
# OUTS buffer columns
O_MET, O_ROUGH, O_ALB, O_LD, O_LDIR, O_LI, O_IW, O_HUM, O_LDIM = 0, 4, 8, 12, 16, 20, 24, 28, 32
Y8_LD, Y8_X, Y8_SDF = 320, 256, 260


def ide_coefficient_table():
    """mat[17,36] of Ref-NeRF's integrated directional encoding (eq. 6-8 of arXiv:2112.03907), computed in float64
    and rounded to float32 exactly like utils/ref_utils.py:77-82 does before using it."""
    def gbc(a, k):
        return np.prod(a - np.arange(k)) / math.factorial(k)

    def alc(l, m, k):
        return ((-1) ** m * 2 ** l * math.factorial(l) / math.factorial(k) / math.factorial(l - k - m) *
                gbc(0.5 * (l + k + m - 1.0), l))

    def shc(l, m, k):
        return np.sqrt((2.0 * l + 1.0) * math.factorial(l - m) / (4.0 * np.pi * math.factorial(l + m))) * alc(l, m, k)

    cols = [(m, 2 ** e) for e in range(5) for m in range(2 ** e + 1)]
    mat = np.zeros((17, len(cols)))
    for i, (m, l) in enumerate(cols):
        for k in range(l - m + 1):
            mat[k, i] = shc(l, m, k)
    return np.ascontiguousarray(mat.astype(np.float32))


_ide_uploaded = False


def upload_ide_table():
    global _ide_uploaded
    if not _ide_uploaded:
        mat = ide_coefficient_table()
        ops.call('nero_set_ide_table', mat)
        _ide_uploaded = True


def _linear_to_srgb_torch(x):
    eps = torch.finfo(torch.float32).eps
    return torch.where(x <= 0.0031308, 323 / 25 * x, (211 * torch.clamp(x, min=eps) ** (5 / 12) - 11) / 200)


def _fg_lookup_torch(lut, uv):
    """bilinear clamp lookup of the [256,256,2] LUT (validation path only; the training path does this in shade_combine)."""
    H, W = lut.shape[0], lut.shape[1]
    fx, fy = uv[:, 0] * W - 0.5, uv[:, 1] * H - 0.5
    x0f, y0f = torch.floor(fx), torch.floor(fy)
    tx, ty = (fx - x0f)[:, None], (fy - y0f)[:, None]
    x0, x1 = x0f.long().clamp(0, W - 1), (x0f.long() + 1).clamp(0, W - 1)
    y0, y1 = y0f.long().clamp(0, H - 1), (y0f.long() + 1).clamp(0, H - 1)
    a = lut[y0, x0] * (1 - tx) + lut[y0, x1] * tx
    b = lut[y1, x0] * (1 - tx) + lut[y1, x1] * tx
    return a * (1 - ty) + b * ty


class Grads:
    """Maps parameters to their .grad buffers: views of ONE persistent flat buffer (the buffer a data-parallel run
    all-reduces with a single NCCL call, and whose addresses a captured CUDA graph of the backward pass can rely on).
    A parameter whose .grad is None (after zero_grad(set_to_none=True)) gets its zeroed view back; a .grad somebody else
    allocated is left alone unless `strict` (graph replay), where it is moved into the flat buffer."""

    def __init__(self, params):
        self.params = [p for p in params]
        self.total = sum(p.numel() for p in self.params)
        self.flat = None
        self.views = None

    def ensure(self, strict=False):
        if self.flat is None:
            self.flat = torch.zeros(self.total, dtype=torch.float32, device=self.params[0].device)
            off = 0
            self.views = []
            for p in self.params:
                n = p.numel()
                self.views.append(self.flat[off:off + n].view_as(p))
                off += n
        missing = [i for i, p in enumerate(self.params) if p.grad is None]
        if len(missing) == len(self.params):
            self.flat.zero_()
        else:
            for i in missing:
                self.views[i].zero_()
        for i in missing:
            self.params[i].grad = self.views[i]
        if strict:
            for p, v in zip(self.params, self.views):
                if p.grad.data_ptr() != v.data_ptr():
                    v.copy_(p.grad)
                    p.grad = v
        return self.flat


class Predictor:
    """make_predictor (network/field.py:310-346): 4 weight-normed linears, ReLU x3, final activation."""

    def __init__(self, pp, dev, n_out, act, act_param=0.0, kmap=None, k_layout=None, t_cols=None):
        ls = pp.layers()
        self.n_out, self.act, self.act_param = n_out, act, act_param
        self.layers = [ops.PreparedLayer(ls[0].weight_v, ls[0].weight_g, ls[0].bias, dev, kmap=kmap, k_layout=k_layout, t_cols=t_cols)]
        for l in ls[1:]:
            self.layers.append(ops.PreparedLayer(l.weight_v, l.weight_g, l.bias, dev, t_cols=(0, 256)))
        self.pl = ls

    def prep(self):
        for l in self.layers:
            l.prep()

    def forward(self, A, acts, out, m_ptr, m_cap):
        L = self.layers
        mlp(A, [CL(L[0], EK_BIAS_RELU, 256, save=Mat(acts[0])), CL(L[1], EK_BIAS_RELU, 256, save=Mat(acts[1])),
                CL(L[2], EK_BIAS_RELU, 256, save=Mat(acts[2])),
                CL(L[3], EK_BIAS_GENERIC, self.n_out, save=out, act=self.act, act_param=self.act_param)], m_ptr, m_cap, fused=USE_CHAIN)

    def backward(self, ws, dpre, A, acts, dH, m_ptr, m_cap, dX=None, dx_ncol=0, dx_addend=None):
        """dpre: Mat over the pre-activation gradient of the output (n_out columns); dH: three [., 256] buffers that receive
        the pre-activation gradients of the hidden layers 2, 1, 0."""
        L, P = self.layers, self.pl
        g = lambda i: (P[i].weight_v.grad, P[i].weight_g.grad, P[i].bias.grad)
        kw = dict(m_ptr=m_ptr, m_cap=m_cap)
        ls = [CL(L[3], EK_DACT_RELU, 256, transposed=True, H=Mat(acts[2]), save=Mat(dH[0])),
              CL(L[2], EK_DACT_RELU, 256, transposed=True, H=Mat(acts[1]), save=Mat(dH[1])),
              CL(L[1], EK_DACT_RELU, 256, transposed=True, H=Mat(acts[0]), save=Mat(dH[2]))]
        if dX is not None:
            ls.append(CL(L[0], EK_DACT_NONE, dx_ncol, transposed=True, addend=dx_addend, save=dX))
        mlp(dpre, ls, m_ptr, m_cap, fused=USE_CHAIN)
        wgrad(ws, dpre, self.n_out, Mat(acts[2]), 256, L[3], *g(3), **kw)
        wgrad(ws, Mat(dH[0]), 256, Mat(acts[1]), 256, L[2], *g(2), **kw)
        wgrad(ws, Mat(dH[1]), 256, Mat(acts[0]), 256, L[1], *g(1), **kw)
        wgrad(ws, Mat(dH[2]), 256, A, L[0].k_valid, L[0], *g(0), **kw)


class SdfNet:
    """SDFNetwork (network/field.py:60-181): PE6 -> 8 x softplus(beta=100) hidden layers (skip concat before layer 4) -> 257."""

    def __init__(self, sp, dev):
        self.sp = sp
        ls = sp.layers()
        assert len(ls) == 9 and sp.multires == 6 and tuple(sp.skip_in) == (4,), 'kernels are laid out for the default SDF network'
        self.L = []
        for k, l in enumerate(ls[:8]):
            tc = (0, 39) if k == 0 else (0, 256)
            self.L.append(ops.PreparedLayer(l.weight_v, l.weight_g, l.bias, dev, t_cols=tc))
        l8 = ls[8]
        self.L8f = ops.PreparedLayer(l8.weight_v, l8.weight_g, l8.bias, dev, row0=1, nrows=256, t_cols=(0, 256))   # feature rows
        self.L8s = ops.PreparedLayer(l8.weight_v, l8.weight_g, l8.bias, dev, row0=0, nrows=1, t_cols=(0, 256))     # sdf row
        self.nout = [256, 256, 256, 217, 256, 256, 256, 256]
        self.tmp_row = torch.zeros(256, device=dev)
        self.tmp_b = torch.zeros(4, device=dev)

    def prep(self):
        for l in self.L + [self.L8f, self.L8s]:
            l.prep()

    def hidden_forward(self, X0, Hs, H4buf, m_ptr, m_cap, save=True, heads=()):
        """X0 [.,64] -> Hs[k] = input of layer k+1 (k = 0..7), then the `heads` on Hs[7]; the output of lin3 goes into
        H4buf[:, :217] scaled by 1/sqrt2 next to the pre-filled PE/sqrt2 tail (skip concat, field.py:139-140).
        save=False: the fused chain stores only the heads' outputs (the per-layer path still writes Hs)."""
        ls = [CL(self.L[k], EK_BIAS_SOFTPLUS, 256, save=Mat(Hs[k]), store=save) for k in (0, 1, 2)]
        ls.append(CL(self.L[3], EK_BIAS_SOFTPLUS, 217, oscale=INV_SQRT2, save=Mat(H4buf), csrc=Mat(H4buf), store=save))
        ls += [CL(self.L[k], EK_BIAS_SOFTPLUS, 256, save=Mat(Hs[k]), store=save) for k in (4, 5, 6, 7)]
        mlp(Mat(X0), ls + list(heads), m_ptr, m_cap, tag='sdf_forward' if save else 'sdf_forward_nosave', fused=USE_CHAIN)

    def sdf_only(self, X0, SA, SB, SC, out, m_ptr, m_cap):
        """Forward-only SDF value (sampling / occlusion march): hidden stack in 3 rotating buffers, last layer row 0 only."""
        self.hidden_forward(X0, [SA, SB, SA, SC, SA, SB, SA, SB], SC, m_ptr, m_cap, save=False,
                            heads=[CL(self.L8s, EK_BIAS_GENERIC, 1, save=Mat(out), write_a=False)])

    # ---- training path on the compacted inner samples --------------------------------------------------
    def forward_with_gradient(self, w, m_ptr, m_cap):
        H, V = w['H'], w['V']   # H[1..8]; H[4] has the PE/sqrt2 tail pre-filled by ray_fill
        self.hidden_forward(w['X0'], H[1:], H[4], m_ptr, m_cap,
                            heads=[CL(self.L8f, EK_BIAS_GENERIC, 256, save=Mat(w['Y8']), write_a=False),          # feature vector
                                   CL(self.L8s, EK_BIAS_GENERIC, 1, save=Mat(w['Y8'], Y8_SDF), write_a=False)])   # sdf
        # reverse sweep for d sdf / d x  (v_k = sigma_k * u_{k+1}, u_k = W_k^T v_k);
        # u_4 = [217 -> v_3 (through 1/sqrt2) | 39 -> skip branch to the PE input]
        K('nero_dact_times_row', H[8], 256, self.L8s.w_eff, V[7], 256, 256, m_ptr, m_cap)
        ls = []
        for k in range(7, 0, -1):
            if k == 4:
                ls.append(CL(self.L[4], EK_DACT_SOFTPLUS, 256, transposed=True, oscale=INV_SQRT2, H=Mat(H[4]), hscale=SQRT2,
                             ncol_main=217, tail=Mat(w['USKIP']), save=Mat(V[3])))
            else:
                ls.append(CL(self.L[k], EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[k]), save=Mat(V[k - 1])))
        ls.append(CL(self.L[0], EK_DACT_NONE, 39, transposed=True, save=Mat(w['U0'])))
        mlp(Mat(V[7]), ls, m_ptr, m_cap, tag='sdf_reverse_sweep', fused=USE_CHAIN)
        K('nero_pe_grad', w['X0'], 64, w['U0'], 64, w['USKIP'], 64, w['G'], m_ptr, m_cap)

    def backward(self, ws, w, m_ptr, m_cap, grads_of):
        """Given dY8 (feature cols 0..255, sdf col 260) and DG (d loss / d gradient), accumulate all SDF parameter grads."""
        H, V, UB, AB = w['H'], w['V'], w['UB'], w['ABAR']
        kw = dict(m_ptr=m_ptr, m_cap=m_cap)
        dY8 = w['dY8']
        # tangent sweep (adjoint of the reverse sweep): ubar_0 = J_PE dg ; vbar_k = W_k ubar_k ; ubar_{k+1} = sigma_k vbar_k,
        # which also leaves the softplus'' term q_k = 100 (1 - sigma_k) v_k vbar_k in ABAR[k]
        K('nero_pe_tangent', w['X0'], 64, w['DG'], UB[0], 64, UB[4], 256, m_ptr, m_cap)
        ls = []
        for k in range(8):
            if k == 3:
                ls.append(CL(self.L[3], EK_TANGENT, 217, use_bias=False, oscale=INV_SQRT2, H=Mat(H[4]), hscale=SQRT2, V=Mat(V[3]),
                             out2=Mat(AB[3]), save=Mat(UB[4]), csrc=Mat(UB[4])))
            else:
                ls.append(CL(self.L[k], EK_TANGENT, 256, use_bias=False, H=Mat(H[k + 1]), V=Mat(V[k]), out2=Mat(AB[k]), save=Mat(UB[k + 1])))
        mlp(Mat(UB[0]), ls, m_ptr, m_cap, tag='sdf_tangent_sweep', fused=USE_CHAIN)
        # value backward: abar_7 = sigma_7*(W8f^T dfeat) + q_7 + dsdf*v_7 (v_7 = sigma_7*W8[0,:] from the reverse sweep);
        # abar_{k-1} = sigma_{k-1} * (W_k^T abar_k) + q_{k-1}
        K('nero_row_axpy', Mat(dY8, Y8_SDF), Y8_LD, V[7], 256, AB[7], 256, 256, m_ptr, m_cap)
        ls = [CL(self.L8f, EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[8]), addend=Mat(AB[7]), save=Mat(AB[7]))]
        for k in range(7, 0, -1):
            if k == 4:
                ls.append(CL(self.L[4], EK_DACT_SOFTPLUS, 217, transposed=True, oscale=INV_SQRT2, H=Mat(H[4]), hscale=SQRT2,
                             addend=Mat(AB[3]), save=Mat(AB[3])))
            else:
                ls.append(CL(self.L[k], EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[k]), addend=Mat(AB[k - 1]), save=Mat(AB[k - 1])))
        mlp(Mat(dY8), ls, m_ptr, m_cap, tag='sdf_value_backward', fused=USE_CHAIN)
        # weight gradients: dW_k = abar_k^T h_k + v_k^T ubar_k
        ls = self.sp.layers()
        for k in range(8):
            Hin = Mat(w['X0']) if k == 0 else Mat(H[k])
            wgrad(ws, Mat(AB[k]), self.nout[k], Hin, self.L[k].k_valid, self.L[k], ls[k].weight_v.grad, ls[k].weight_g.grad,
                  ls[k].bias.grad, dY2=Mat(V[k]), X2=Mat(UB[k]), **kw)
        l8 = ls[8]
        wgrad(ws, Mat(dY8), 256, Mat(H[8]), 256, self.L8f, l8.weight_v.grad, l8.weight_g.grad, l8.bias.grad, **kw)
        # sdf row: dW8[0,:] = sum_m dsdf[m] h8[m,:] + sum_m ubar_8[m,:] ; db8[0] = sum dsdf
        self.tmp_row.zero_()
        self.tmp_b.zero_()
        ops.colsum(Mat(H[8]), 256, self.tmp_row, w=Mat(dY8, Y8_SDF), m_ptr=m_ptr, m_cap=m_cap)
        ops.colsum(Mat(UB[8]), 256, self.tmp_row, m_ptr=m_ptr, m_cap=m_cap)
        ops.colsum(Mat(dY8, Y8_SDF), 1, self.tmp_b, m_ptr=m_ptr, m_cap=m_cap)
        K('nero_wgrad_finish', self.tmp_row, 1, 1, 256, self.tmp_b, 256, 0, 1, None, 1.0, l8.weight_v.detach(), l8.weight_g.detach(),
          l8.weight_v.grad, l8.weight_g.grad, l8.bias.grad, None, 0.0)

    def value_forward(self, X0, H, out, m_ptr, m_cap):
        """SDF value with saved activations H[1..8] (step<1000 regulariser points, renderer.py:591-594)."""
        self.hidden_forward(X0, H[1:], H[4], m_ptr, m_cap, heads=[CL(self.L8s, EK_BIAS_GENERIC, 1, save=Mat(out), write_a=False)])

    def value_backward(self, ws, X0, H, dsdf, AB, scratch, m_ptr, m_cap):
        """Backward of value_forward: dsdf [.,1] -> parameter grads.  abar_7 = dsdf * sigma_7 * W8[0,:], then the
        plain reverse chain abar_{k-1} = sigma_{k-1} * (W_k^T abar_k), then dW_k = abar_k^T h_k."""
        kw = dict(m_ptr=m_ptr, m_cap=m_cap)
        K('nero_dact_times_row', H[8], 256, self.L8s.w_eff, scratch, 256, 256, m_ptr, m_cap)
        AB[7].zero_()
        K('nero_row_axpy', dsdf, dsdf.stride(0), scratch, 256, AB[7], 256, 256, m_ptr, m_cap)
        ls = []
        for k in range(7, 0, -1):
            if k == 4:
                ls.append(CL(self.L[4], EK_DACT_SOFTPLUS, 217, transposed=True, oscale=INV_SQRT2, H=Mat(H[4]), hscale=SQRT2, save=Mat(AB[3])))
            else:
                ls.append(CL(self.L[k], EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[k]), save=Mat(AB[k - 1])))
        mlp(Mat(AB[7]), ls, m_ptr, m_cap, fused=USE_CHAIN)
        ls_ = self.sp.layers()
        for k in range(8):
            Hin = Mat(X0) if k == 0 else Mat(H[k])
            wgrad(ws, Mat(AB[k]), self.nout[k], Hin, self.L[k].k_valid, self.L[k], ls_[k].weight_v.grad, ls_[k].weight_g.grad,
                  ls_[k].bias.grad, **kw)
        l8 = ls_[8]
        self.tmp_row.zero_()
        self.tmp_b.zero_()
        ops.colsum(Mat(H[8]), 256, self.tmp_row, w=Mat(dsdf), m_ptr=m_ptr, m_cap=m_cap)
        ops.colsum(Mat(dsdf), 1, self.tmp_b, m_ptr=m_ptr, m_cap=m_cap)
        K('nero_wgrad_finish', self.tmp_row, 1, 1, 256, self.tmp_b, 256, 0, 1, None, 1.0, l8.weight_v.detach(), l8.weight_g.detach(),
          l8.weight_v.grad, l8.weight_g.grad, l8.bias.grad, None, 0.0)


class NerfNet:
    """Outer NeRF++ (NeRFNetwork, network/field.py:205-297): PE10(4-d) -> 8 x ReLU(256) with skip, density head,
    feature + PE4(view) -> 128 -> rgb."""

    def __init__(self, npar, dev):
        self.np = npar
        pl = npar.pts_linears
        mk = lambda l, **kw: ops.PreparedLayer(l.weight, None, l.bias, dev, **kw)
        self.P = [mk(pl[0])] + [mk(pl[i], t_cols=(0, 256)) for i in range(1, 5)] + [mk(pl[5], t_cols=(84, 256))] + \
                 [mk(pl[i], t_cols=(0, 256)) for i in (6, 7)]
        self.alpha = mk(npar.alpha_linear, t_cols=(0, 256))
        self.feature = mk(npar.feature_linear, t_cols=(0, 256))
        self.views = mk(npar.views_linears[0], t_cols=(0, 256))
        self.rgb = mk(npar.rgb_linear, t_cols=(0, 128))

    def all_layers(self):
        return self.P + [self.alpha, self.feature, self.views, self.rgb]

    def prep(self):
        for l in self.all_layers():
            l.prep()

    def forward(self, w, m_ptr, m_cap):
        kw = dict(m_ptr=m_ptr, m_cap=m_cap)
        N = w['NH']
        mlp(Mat(w['XN']),
            [CL(self.P[0], EK_BIAS_RELU, 256, save=Mat(N[1])), CL(self.P[1], EK_BIAS_RELU, 256, save=Mat(N[2])),
             CL(self.P[2], EK_BIAS_RELU, 256, save=Mat(N[3])), CL(self.P[3], EK_BIAS_RELU, 256, save=Mat(N[4])),
             CL(self.P[4], EK_BIAS_RELU, 256, save=Mat(w['H5'], 84), write_a=False)], m_ptr, m_cap, tag='nerf_fwd_a', fused=USE_CHAIN)
        # layer 5 reads cat([input_pts, h]) (field.py:268-269): K = 340
        mlp(Mat(w['H5']),
            [CL(self.P[5], EK_BIAS_RELU, 256, save=Mat(N[6])), CL(self.P[6], EK_BIAS_RELU, 256, save=Mat(N[7])),
             CL(self.P[7], EK_BIAS_RELU, 256, save=Mat(N[8])),
             CL(self.alpha, EK_BIAS_GENERIC, 1, save=Mat(w['DENS']), write_a=False),
             CL(self.feature, EK_BIAS_GENERIC, 256, save=Mat(w['FV']), write_a=False)], m_ptr, m_cap, tag='nerf_fwd_b', fused=USE_CHAIN)
        linear(Mat(w['FV']), self.views, Mat(w['HV']), 128, act=ACT_RELU, **kw)
        linear(Mat(w['HV']), self.rgb, Mat(w['RGBRAW']), 3, **kw)

    def backward(self, ws, w, m_ptr, m_cap):
        kw = dict(m_ptr=m_ptr, m_cap=m_cap)
        N, dA, G = w['NH'], w['dNa'], w['dNG']   # G: pre-activation gradients of layers 6..0 (dA holds layer 7's)
        n = self.np
        gp = lambda l: (l.weight.grad, None, l.bias.grad)
        R = dict(transposed=True, mode=EPI_MUL_DACT, dact=ACT_RELU)
        linear(Mat(w['dRGBRAW']), self.rgb, Mat(w['dHV']), 128, H=Mat(w['HV']), **R, **kw)
        wgrad(ws, Mat(w['dRGBRAW']), 3, Mat(w['HV']), 128, self.rgb, *gp(n.rgb_linear), **kw)
        linear(Mat(w['dHV']), self.views, Mat(w['dFV']), 256, transposed=True, mode=EPI_MUL_DACT, **kw)
        wgrad(ws, Mat(w['dHV']), 128, Mat(w['FV']), self.views.k_valid, self.views, *gp(n.views_linears[0]), **kw)
        linear(Mat(w['dFV']), self.feature, Mat(dA), 256, H=Mat(N[8]), **R, **kw)
        linear(Mat(w['dDENS']), self.alpha, Mat(dA), 256, H=Mat(N[8]), addend=Mat(dA), **R, **kw)
        wgrad(ws, Mat(w['dFV']), 256, Mat(N[8]), 256, self.feature, *gp(n.feature_linear), **kw)
        wgrad(ws, Mat(w['dDENS']), 1, Mat(N[8]), 256, self.alpha, *gp(n.alpha_linear), **kw)
        pl = n.pts_linears
        mlp(Mat(dA),
            [CL(self.P[7], EK_DACT_RELU, 256, transposed=True, H=Mat(N[7]), save=Mat(G[6])),
             CL(self.P[6], EK_DACT_RELU, 256, transposed=True, H=Mat(N[6]), save=Mat(G[5])),
             CL(self.P[5], EK_DACT_RELU, 256, transposed=True, H=Mat(w['H5'], 84), save=Mat(G[4])),
             CL(self.P[4], EK_DACT_RELU, 256, transposed=True, H=Mat(N[4]), save=Mat(G[3])),
             CL(self.P[3], EK_DACT_RELU, 256, transposed=True, H=Mat(N[3]), save=Mat(G[2])),
             CL(self.P[2], EK_DACT_RELU, 256, transposed=True, H=Mat(N[2]), save=Mat(G[1])),
             CL(self.P[1], EK_DACT_RELU, 256, transposed=True, H=Mat(N[1]), save=Mat(G[0]))], m_ptr, m_cap, tag='nerf_bwd', fused=USE_CHAIN)
        wgrad(ws, Mat(dA), 256, Mat(N[7]), 256, self.P[7], *gp(pl[7]), **kw)
        wgrad(ws, Mat(G[6]), 256, Mat(N[6]), 256, self.P[6], *gp(pl[6]), **kw)
        wgrad(ws, Mat(G[5]), 256, Mat(w['H5']), self.P[5].k_valid, self.P[5], *gp(pl[5]), **kw)
        wgrad(ws, Mat(G[4]), 256, Mat(N[4]), 256, self.P[4], *gp(pl[4]), **kw)
        wgrad(ws, Mat(G[3]), 256, Mat(N[3]), 256, self.P[3], *gp(pl[3]), **kw)
        wgrad(ws, Mat(G[2]), 256, Mat(N[2]), 256, self.P[2], *gp(pl[2]), **kw)
        wgrad(ws, Mat(G[1]), 256, Mat(N[1]), 256, self.P[1], *gp(pl[1]), **kw)
        wgrad(ws, Mat(G[0]), 256, Mat(w['XN']), self.P[0].k_valid, self.P[0], *gp(pl[0]), **kw)


class ShapeEngine:
    def __init__(self, params, cfg):
        """params: nero_b200.params.ShapeParams on a CUDA device; cfg: merged renderer cfg."""
        self.p = params
        self.cfg = cfg
        self.scfg = params.color_network.cfg
        dev = params.deviation_network.variance.device
        ops.require_cuda(dev)
        self.dev = dev
        if self.scfg['light_pos_freq'] != 8:
            raise NotImplementedError('light_pos_freq != 8')
        upload_ide_table()
        self.human = bool(self.scfg['human_light'])
        self.exp_max = float(self.scfg['light_exp_max'])
        c = params.color_network
        self.sdf = SdfNet(params.sdf_network, dev)
        self.nerf = NerfNet(params.outer_nerf, dev)
        self.m_met = Predictor(c.metallic_predictor, dev, 1, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        self.m_rough = Predictor(c.roughness_predictor, dev, 1, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        self.m_alb = Predictor(c.albedo_predictor, dev, 3, ACT_SIGMOID, k_layout=259, t_cols=(0, 256))
        # sphere_direction (field.py:560-563, 583-586): outer_light reads [IDE(d, k) | IDE(s_d, k)], s_d = direction of the
        # unit-sphere exit point of the ray (x, d); the E buffer then holds the two 144-wide windows (k_shade.cu)
        self.sphere = bool(self.scfg['sphere_direction'])
        self.e_iden, self.e_ld = (236, 384) if self.sphere else (E_IDEN, E_LD)
        ko = 144 if self.sphere else 72
        self.m_outer = Predictor(c.outer_light, dev, 3, ACT_EXPCLAMP, self.exp_max, k_layout=ko, t_cols=(0, ko))
        self.m_inner = Predictor(c.inner_light, dev, 3, ACT_EXPCLAMP, self.exp_max,
                                 kmap=list(range(51)) + [52 + i for i in range(72)], k_layout=124, t_cols=(52, 72))
        self.m_iw = Predictor(c.inner_weight, dev, 1, ACT_NONE, kmap=[40 + i for i in range(51)] + list(range(39)), k_layout=91)
        self.m_human = Predictor(c.human_light_predictor, dev, 4, ACT_EXPCLAMP, 0.0, k_layout=24, t_cols=(0, 24)) if self.human else None
        self.lut = c.FG_LUT
        self.grads = Grads(list(params.parameters()))
        self.ws = ops.WgradWorkspace(dev)
        self.ws.defer = True      # weight-gradient reductions are queued and run as one batched launch per backward pass
        self.w = None
        self.cap = (0, 0)
        n, nb = cfg['n_samples'], cfg['n_bg_samples']
        # constant tables evaluated by torch on the CPU exactly like renderer.py:411-421
        zo = torch.linspace(1e-3, 1.0 - 1.0 / (nb + 1.0), nb)
        mids = .5 * (zo[1:] + zo[:-1])
        self.t_lin = torch.linspace(0.0, 1.0, n).to(dev)
        self.t_bg = zo.to(dev)
        self.t_bg_lo = torch.cat([zo[:1], mids]).to(dev)
        self.t_bg_hi = torch.cat([mids, zo[-1:]]).to(dev)
        self.t_lin64 = torch.linspace(0, 1, 64).to(dev)
        self.prepared_version = None
        self.car_dev = torch.zeros(1, device=dev)      # cos_anneal_ratio: read by the kernels through a pointer, so a
                                                       # captured graph of the step sees each step's value

    # ------------------------------------------------------------------ weights
    def predictors(self):
        ps = [self.m_met, self.m_rough, self.m_alb, self.m_outer, self.m_inner, self.m_iw]
        return ps + ([self.m_human] if self.human else [])

    def prepare_weights(self):
        """Fold weight-norm and rebuild the tensor-core operand images of every layer (one batched launch)."""
        if getattr(self, '_all_layers', None) is None:
            ls = self.sdf.L + [self.sdf.L8f, self.sdf.L8s] + self.nerf.all_layers()
            for m in self.predictors():
                ls += m.layers
            self._all_layers = ops.PrepBatch(ls)
        self._all_layers.run()

    # ------------------------------------------------------------------ workspaces
    def _alloc(self, R, S):
        """Workspaces only grow: every kernel takes explicit R / S / leading dimensions / row caps, so a smaller batch (the
        ragged last chunk of an image, a train -> validation switch) runs in the buffers of a larger one."""
        if R <= self.cap[0] and S <= self.cap[1]:
            return
        R, S = max(R, self.cap[0]), max(S, self.cap[1])
        self.w = None                       # release the old workspaces before allocating the larger ones
        dev = self.dev
        cap = R * S
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev)
        w = {}
        ns = self.cfg['n_samples']
        caps = max(R * ns, self.cfg['occ_loss_max_pn'] * 64)
        w.update(SX0=z(caps, 64), SA=z(caps, 256), SB=z(caps, 256), SC=z(caps, 256), SSDF=z(caps, 1), SSDF0=z(R * ns, 1),
                 ZA=z(R, 128), ZB=z(R, 128), SDFA=z(R, 128), SDFB=z(R, 128), NEWZ=z(R, 32))
        w.update(cnt_in=z(R, dt=torch.int32), cnt_out=z(R, dt=torch.int32), off_in=z(R, dt=torch.int32), off_out=z(R, dt=torch.int32),
                 n_in=z(1, dt=torch.int32), n_out=z(1, dt=torch.int32), slot=z(R, S, dt=torch.int32))
        # inner
        w.update(X0=z(cap, 64), PTS=z(cap, 4), RAY_IN=z(cap, dt=torch.int32), Y8=z(cap, Y8_LD), U0=z(cap, 64), USKIP=z(cap, 64),
                 G=z(cap, 4), OUTS=z(cap, O_LDIM), E=z(cap, self.e_ld), GEO=z(cap, 8), EH=z(cap, 64), COLOR_IN=z(cap, 4), OCCP=z(cap),
                 REFL=z(cap, 4), ALPHA_IN=z(cap), GERR=z(cap))
        w['H'] = [None] + [z(cap, 256) for _ in range(8)]
        w['V'] = [z(cap, 256) for _ in range(8)]
        names = ['met', 'rough', 'alb', 'odir', 'odif', 'inner', 'iw'] + (['human'] if self.human else [])
        w['ACT'] = {k: [z(cap, 256) for _ in range(3)] for k in names}
        # outer
        w.update(XN=z(cap, 128), H5=z(cap, 384), DENS=z(cap, 4), FV=z(cap, 320), HV=z(cap, 128), RGBRAW=z(cap, 4), DIST_OUT=z(cap),
                 RAY_OUT=z(cap, dt=torch.int32), ALPHA_OUT=z(cap), COLOR_OUT=z(cap, 4))
        w['NH'] = [None] + [z(cap, 256) for _ in range(4)] + [None] + [z(cap, 256) for _ in range(3)]
        # occlusion march
        P = self.cfg['occ_loss_max_pn']
        w.update(SEL=z(cap, dt=torch.int32), OCC_COUNT=z(1, dt=torch.int32), OCC_O=z(P, 3), OCC_D=z(P, 3), OCC_Z=z(P, 64),
                 OCC_NEWZ=z(P, 16), OCC_GT=z(P), OCC_LOSS=z(1), DOCC=z(cap))
        self.w = w
        self.cap = (R, S)
        self.bw_ready = False

    def _alloc_reg(self):
        if 'REG_H' in self.w:
            return
        R, S = self.cap
        cap = R * S
        z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=self.dev)
        self.w.update(REG_CNT=z(R, dt=torch.int32), REG_OFF=z(R, dt=torch.int32), REG_N=z(1, dt=torch.int32), REG_DUMMY=z(R, dt=torch.int32),
                      REG_DUMMY1=z(1, dt=torch.int32), REG_PTS=z(cap, 4), REG_X0=z(cap, 64), REG_SDF=z(cap, 1), REG_DSDF=z(cap, 1))
        self.w['REG_H'] = [None] + [z(cap, 256) for _ in range(8)]

    def reg_forward(self, rays_o, rays_d, z_vals):
        """sdf_pts / sdf_vals of renderer.py:591-594 (value-only SDF pass on every mid-point with |p| < 1.2)."""
        R, S = z_vals.shape
        self._alloc_reg()
        w = self.w
        K('nero_reg_prepare', rays_o, rays_d, z_vals, R, S, 1.2, w['REG_CNT'], w['REG_DUMMY'], w['REG_OFF'], w['REG_DUMMY'], w['REG_N'],
          w['REG_DUMMY1'])
        K('nero_reg_fill', rays_o, rays_d, z_vals, R, S, 1.2, w['REG_OFF'], w['REG_PTS'], w['REG_X0'], 64, w['REG_H'][4], 256)
        self.sdf.value_forward(w['REG_X0'], w['REG_H'], w['REG_SDF'], w['REG_N'], R * S)

    def reg_backward(self, d_sdf_vals):
        self._alloc_backward()
        self.grads.ensure()
        w = self.w
        k = d_sdf_vals.shape[0]
        w['REG_DSDF'][:k, 0].copy_(d_sdf_vals)
        cap = self.cap[0] * self.cap[1]
        self.sdf.value_backward(self.ws, w['REG_X0'], w['REG_H'], w['REG_DSDF'], w['ABAR'], w['dHa'], w['REG_N'], cap)
        self.ws.flush()

    def _alloc_backward(self):
        if self.bw_ready:
            return
        R, S = self.cap
        cap = R * S
        z = lambda *s: torch.zeros(*s, dtype=torch.float32, device=self.dev)
        w = self.w
        w.update(dALPHA_IN=z(cap), dCOLOR_IN=z(cap, 4), DOUTS=z(cap, O_LDIM), DNOV=z(cap), dE_dir=z(cap, 160), dE_inn=z(cap, 128),
                 dE_dif=z(cap, 160), dEH=z(cap, 64), DG=z(cap, 4), dY8=z(cap, Y8_LD), dHa=z(cap, 256), dHb=z(cap, 256), dHc=z(cap, 256),
                 D_INV_S=z(1))
        w['UB'] = [z(cap, 64)] + [z(cap, 256) for _ in range(8)]
        w['ABAR'] = [z(cap, 256) for _ in range(8)]
        w.update(dALPHA_OUT=z(cap), dCOLOR_OUT=z(cap, 4), dDENS=z(cap, 4), dRGBRAW=z(cap, 4), dHV=z(cap, 128), dFV=z(cap, 256),
                 dNa=z(cap, 256))
        w['dNG'] = [z(cap, 256) for _ in range(7)]
        self.bw_ready = True

    # ------------------------------------------------------------------ sampling (renderer.py:403-443)
    def sample_ray(self, rays_o, rays_d, near, far, rand_inner=None, rand_bg=None):
        cfg = self.cfg
        R = rays_o.shape[0]
        n, nb, nimp, steps = cfg['n_samples'], cfg['n_bg_samples'], cfg['n_importance'], cfg['up_sample_steps']
        S = n + nimp + nb
        nn_ = nimp // steps
        assert nimp % steps == 0 and nn_ <= 32 and n + nimp <= 128 and nb <= n, 'sampling kernels: <=32 new samples / step, <=128 inner samples'
        self._alloc(R, S)
        w = self.w
        z_vals = torch.empty(R, S, device=self.dev)
        var = self.p.deviation_network.variance.detach()
        K('nero_sample_init', rays_o, rays_d, near, far, R, n, nb, self.t_lin, self.t_bg, self.t_bg_lo, self.t_bg_hi,
          rand_inner, rand_bg, w['ZA'], 128, Mat(z_vals, n + nimp), S, w['SX0'], 64, w['SC'], 256)
        self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF0'], None, R * n)   # coarse sdf kept apart:
        cur_z, cur_sdf, lds = w['ZA'], w['SSDF0'], n                                        # SSDF is reused per iteration
        nxt_z, nxt_sdf = w['ZB'], w['SDFB']
        cur_n = n
        for i in range(steps):
            last = i + 1 == steps
            K('nero_upsample', rays_o, rays_d, R, cur_z, 128, cur_sdf, lds, cur_n, nn_, var, float(64 * 2 ** i),
              1 if cfg['clip_sample_variance'] else 0, 0, w['NEWZ'], 32, None if last else w['SX0'], 64,
              None if last else w['SC'], 256, None)
            if last:
                K('nero_merge_samples', cur_z, 128, None, 0, cur_n, w['NEWZ'], 32, None, 0, nn_, z_vals, S, None, 0, R)
            else:
                self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, R * nn_)
                K('nero_merge_samples', cur_z, 128, cur_sdf, lds, cur_n, w['NEWZ'], 32, w['SSDF'], nn_, nn_, nxt_z, 128, nxt_sdf, 128, R)
                cur_z, nxt_z = nxt_z, (w['ZA'] if nxt_z is w['ZB'] else w['ZB'])
                cur_sdf, nxt_sdf = nxt_sdf, (w['SDFA'] if nxt_sdf is w['SDFB'] else w['SDFB'])
                lds = 128
            cur_n += nn_
        return z_vals

    # ------------------------------------------------------------------ render_core forward (renderer.py:550-606)
    def render_core_forward(self, rays_o, rays_d, z_vals, human_poses, cos_anneal_ratio, step, perm=None, static=None):
        """`static` (graph.TrainStepGraphs) selects the sync-free form used under CUDA-graph capture: no count is read back
        to the host -- every kernel takes the device-side row count, the occlusion subset is drawn on the device, and
        `cos_anneal_ratio` is whatever the caller put into `car_dev` -- and only `rgb` is returned."""
        cfg = self.cfg
        R, S = z_vals.shape
        self._alloc(R, S)
        w = self.w
        cap = R * S
        if static is None:
            self.car_dev.fill_(float(cos_anneal_ratio))
        var = self.p.deviation_network.variance.detach()
        K('nero_ray_prepare', rays_o, rays_d, z_vals, R, S, w['cnt_in'], w['cnt_out'], w['off_in'], w['off_out'], w['n_in'], w['n_out'])
        K('nero_ray_fill', rays_o, rays_d, z_vals, R, S, w['off_in'], w['off_out'], w['slot'], w['PTS'], w['RAY_IN'],
          w['X0'], 64, w['Y8'], Y8_LD, w['H'][4], 256, w['XN'], 128, w['H5'], 384, w['FV'], 320, w['DIST_OUT'], w['RAY_OUT'])
        n_in, n_out = w['n_in'], w['n_out']
        # ---- inner samples: SDF value + analytic gradient
        self.sdf.forward_with_gradient(w, n_in, cap)
        self._shade_forward(rays_d, human_poses, n_in, cap)
        K('nero_sdf_alpha_fwd', w['Y8'], Y8_LD, Y8_SDF, w['G'], w['PTS'], w['RAY_IN'], rays_d, var, self.car_dev, w['ALPHA_IN'],
          w['GERR'], n_in, cap)
        # ---- outer samples: NeRF++
        self.nerf.forward(w, n_out, cap)
        K('nero_nerf_post_fwd', w['DENS'], 4, w['RGBRAW'], 4, w['DIST_OUT'], w['ALPHA_OUT'], w['COLOR_OUT'], n_out, cap)
        # ---- compositing
        rgb = torch.empty(R, 3, device=self.dev)
        K('nero_composite_fwd', w['slot'], R, S, w['ALPHA_IN'], w['COLOR_IN'], w['ALPHA_OUT'], w['COLOR_OUT'], rgb, None)
        # ---- occlusion loss
        occ_on = cfg['apply_occ_loss'] and step >= cfg['occ_loss_step']
        P = 0
        if occ_on:
            K('nero_occ_select', w['PTS'], w['Y8'], Y8_LD, Y8_SDF, w['G'], w['RAY_IN'], rays_d, float(cfg['occ_sdf_thresh']), n_in, cap,
              w['SEL'], w['OCC_COUNT'])
        with_reg = step < 1000
        if static is not None:
            assert not with_reg, 'the SDF-initialisation phase (step < 1000) runs eagerly'
            P = self._occ_forward_static(static) if occ_on else 0
            self.n_reg = 0
            self.state = dict(R=R, S=S, N_in=None, P=P, rays_d=rays_d, hp=self._hp, step=step)
            return rgb
        if with_reg:
            self.reg_forward(rays_o, rays_d, z_vals)
            w = self.w
        counts = torch.cat([w['n_in'], w['OCC_COUNT'], w['REG_N'] if with_reg else w['n_out']]).tolist()   # the one host sync
        N_in = counts[0]
        self.n_reg = counts[2] if with_reg else 0
        if occ_on:
            P = self._occ_forward(counts[1], perm)
        self.state = dict(R=R, S=S, N_in=N_in, P=P, rays_d=rays_d, hp=self._hp, step=step)
        return rgb, N_in, P

    def _occ_forward(self, cnt, perm):
        cfg, w = self.cfg, self.w
        maxp = cfg['occ_loss_max_pn']
        if cnt == 0:
            return 0
        sel = w['SEL']
        if cnt > maxp:   # renderer.py:535-541 random subset
            idx = perm if perm is not None else torch.randperm(cnt, device=self.dev)
            # the compaction kernel orders candidates only within a block (and the blocks by atomic arrival); the reference
            # indexes them in sample order (boolean-mask gather): restore that order before the permutation picks its subset,
            # which also makes the subset a function of the RNG state alone (run-to-run determinism under a fixed seed)
            sel = torch.sort(sel[:cnt])[0][idx[:maxp].to(self.dev)].contiguous()
            cnt = maxp
            w['SEL_SUB'] = sel
        return self._occ_march(sel, None, cnt)

    def _occ_forward_static(self, static):
        """The same uniform subset without a host-side count: every candidate draws a key, the `occ_loss_max_pn` smallest keys
        win (a uniformly random subset, like randperm(cnt)[:max_pn]); the number of winners stays on the device and bounds
        the occlusion kernels through their row-count pointer."""
        w = self.w
        maxp = self.cfg['occ_loss_max_pn']
        cnt = w['OCC_COUNT']
        keys = torch.where(static.ar < cnt, static.occ_keys, 2.0)
        maxp = min(maxp, keys.shape[0])
        vals, idx = torch.topk(keys, maxp, largest=False)
        static.P_dev = (vals < 1.5).sum(dtype=torch.int32).reshape(1)
        sel = w['SEL'][idx].contiguous()
        return self._occ_march(sel, static.P_dev, maxp)

    def _occ_march(self, sel, p_ptr, P):
        """get_intersection / occlusion ground truth of the selected samples (renderer.py:514-548) and the L1 occlusion loss.
        p_ptr: optional device count (<= P) bounding the rows that are initialised and that enter the loss."""
        w = self.w
        var = self.p.deviation_network.variance.detach()
        K('nero_occ_init', w['PTS'], w['REFL'], sel, p_ptr, P, 64, self.t_lin64, w['OCC_O'], w['OCC_D'], w['OCC_Z'], 64, w['SX0'], 64,
          w['SC'], 256)
        self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, P * 64)
        K('nero_upsample', w['OCC_O'], w['OCC_D'], P, w['OCC_Z'], 64, w['SSDF'], 64, 64, 16, var, 3.0e38, 1, 1, w['OCC_NEWZ'], 16,
          w['SX0'], 64, w['SC'], 256, None)
        self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, P * 16)
        K('nero_upsample', w['OCC_O'], w['OCC_D'], P, w['OCC_NEWZ'], 16, w['SSDF'], 16, 16, 16, var, 3.0e38, 1, 1, None, 0, None, 0, None, 0,
          w['OCC_GT'])
        w['OCC_LOSS'].zero_()
        w['DOCC'].zero_()
        K('nero_occ_loss', w['OCCP'], w['OCC_GT'], sel, p_ptr, P, w['OCC_LOSS'], w['DOCC'])
        self.occ_sel = sel
        return P

    def _shade_forward(self, rays_d, human_poses, n_in, cap):
        """AppShadingNetwork.forward on the compacted inner samples (network/field.py:591-651)."""
        w = self.w
        # ---- materials
        A = w['ACT']
        matin = Mat(w['Y8'])
        self.m_met.forward(matin, A['met'], Mat(w['OUTS'], O_MET), n_in, cap)
        self.m_rough.forward(matin, A['rough'], Mat(w['OUTS'], O_ROUGH), n_in, cap)
        self.m_alb.forward(matin, A['alb'], Mat(w['OUTS'], O_ALB), n_in, cap)
        hp = human_poses.contiguous() if self.human else None
        self._hp = hp
        K('nero_shade_prep_fwd', w['G'], w['PTS'], w['RAY_IN'], rays_d, w['OUTS'], w['E'], self.e_ld, w['GEO'], hp, w['EH'] if self.human else None,
          64, 8, n_in, cap, 1 if self.sphere else 0)
        self.m_outer.forward(Mat(w['E'], E_IDER), A['odir'], Mat(w['OUTS'], O_LDIR), n_in, cap)
        self.m_outer.forward(Mat(w['E'], self.e_iden), A['odif'], Mat(w['OUTS'], O_LD), n_in, cap)
        self.m_inner.forward(Mat(w['E'], E_PE8X), A['inner'], Mat(w['OUTS'], O_LI), n_in, cap)
        self.m_iw.forward(Mat(w['E'], 0), A['iw'], Mat(w['OUTS'], O_IW), n_in, cap)
        if self.human:
            self.m_human.forward(Mat(w['EH']), A['human'], Mat(w['OUTS'], O_HUM), n_in, cap)
        K('nero_shade_combine_fwd', w['OUTS'], w['GEO'], self.lut, self.exp_max, 1 if self.human else 0, w['COLOR_IN'], w['OCCP'], w['REFL'],
          n_in, cap)

    # ------------------------------------------------------------------ SDF grid query (field.py:150-153 via extract_mesh.py:27)
    QUERY_CHUNK = 131072

    def sdf_query(self, x):
        """sdf_network.sdf(x): value-only SDF of arbitrary points, forward only, chunked through a private workspace."""
        shape = x.shape[:-1]
        x = x.reshape(-1, 3).to(self.dev, torch.float32).contiguous()
        M = x.shape[0]
        out = torch.empty(M, 1, device=self.dev)
        if M == 0:
            return out.reshape(*shape, 1)
        q = getattr(self, '_qws', None)
        if q is None:
            c = self.QUERY_CHUNK
            z = lambda *s: torch.zeros(*s, device=self.dev)
            q = self._qws = dict(X0=z(c, 64), SA=z(c, 256), SB=z(c, 256), SC=z(c, 256), OUT=z(c, 1))
        self.sdf.prep()
        for c0 in range(0, M, self.QUERY_CHUNK):
            n = min(self.QUERY_CHUNK, M - c0)
            K('nero_points_fill', x[c0:c0 + n], n, None, None, q['X0'], 64, None, 0, q['SC'], 256)
            self.sdf.sdf_only(q['X0'], q['SA'], q['SB'], q['SC'], q['OUT'], None, n)
            out[c0:c0 + n] = q['OUT'][:n]
        return out.reshape(*shape, 1)

    # ------------------------------------------------------------------ per-point materials (renderer.py:629-647 -> field.py:653-657)
    def materials_query(self, x):
        """(metallic [M,1], roughness [M,1], albedo [M,3]) of arbitrary points: the SDF feature vector (sdf_network(x)[:, 1:])
        through the three material predictors -- forward only, chunked through the training workspaces."""
        x = x.reshape(-1, 3).to(self.dev, torch.float32).contiguous()
        M = x.shape[0]
        if self.w is None:
            self._alloc(self.cfg['test_ray_num'], self.cfg['n_samples'] + self.cfg['n_importance'] + self.cfg['n_bg_samples'])
        w = self.w
        chunk = w['X0'].shape[0]
        out = torch.empty(M, 5, device=self.dev)
        A = w['ACT']
        for c0 in range(0, M, chunk):
            n = min(chunk, M - c0)
            K('nero_points_fill', x[c0:c0 + n], n, w['PTS'], w['RAY_IN'], w['X0'], 64, w['Y8'], Y8_LD, w['H'][4], 256)
            H = w['H']
            self.sdf.hidden_forward(w['X0'], [H[1], H[2], H[3], H[4], H[5], H[6], H[7], H[8]], H[4], None, n, save=False,
                                    heads=[CL(self.sdf.L8f, EK_BIAS_GENERIC, 256, save=Mat(w['Y8']), write_a=False)])
            matin = Mat(w['Y8'])
            self.m_met.forward(matin, A['met'], Mat(w['OUTS'], O_MET), None, n)
            self.m_rough.forward(matin, A['rough'], Mat(w['OUTS'], O_ROUGH), None, n)
            self.m_alb.forward(matin, A['alb'], Mat(w['OUTS'], O_ALB), None, n)
            o = w['OUTS'][:n]
            out[c0:c0 + n, 0] = o[:, O_MET]
            out[c0:c0 + n, 1] = o[:, O_ROUGH]
            out[c0:c0 + n, 2:5] = o[:, O_ALB:O_ALB + 3]
        return out[:, 0:1], out[:, 1:2], out[:, 2:5]

    # ------------------------------------------------------------------ validation extras (renderer.py:465-482)
    def validation_info(self, rays_o, rays_d, z_vals, human_poses):
        """depth, normal, shading intermediates and occ_prob_gt on the expected surface point of every ray.
        Forward only (called under no_grad); re-uses the training workspaces."""
        R, S = z_vals.shape
        w, dev = self.w, self.dev
        weights = torch.empty(R, S, device=dev)
        rgb = torch.empty(R, 3, device=dev)
        K('nero_composite_fwd', w['slot'], R, S, w['ALPHA_IN'], w['COLOR_IN'], w['ALPHA_OUT'], w['COLOR_OUT'], rgb, weights)
        depth = torch.sum(weights * z_vals, -1, keepdim=True)
        points = (depth * rays_d + rays_o).contiguous()
        K('nero_points_fill', points, R, w['PTS'], w['RAY_IN'], w['X0'], 64, w['Y8'], Y8_LD, w['H'][4], 256)
        self.sdf.forward_with_gradient(w, None, R)
        self._shade_forward(rays_d, human_poses, None, R)
        O = w['OUTS'][:R]
        geo = w['GEO'][:R]
        grads = w['G'][:R, :3]
        inner = (torch.norm(points, dim=-1, keepdim=True) <= 1.0).float()
        met, rough, alb = O[:, O_MET:O_MET + 1], O[:, O_ROUGH:O_ROUGH + 1], O[:, O_ALB:O_ALB + 3]
        Ld, Ldir, Li, iw = O[:, O_LD:O_LD + 3], O[:, O_LDIR:O_LDIR + 3], O[:, O_LI:O_LI + 3], O[:, O_IW:O_IW + 1]
        occ = iw * 0.5 + 0.5
        occ_ = occ.clamp(0, 1)
        if self.human:
            hit = geo[:, 7:8]
            hl = O[:, O_HUM:O_HUM + 4] * hit
            Lh, wh = hl[:, :3], hl[:, 3:].clamp(0, 1)
        else:
            Lh, wh = 0.0, 0.0
        spec_light = Li * occ_ + (Lh * wh + Ldir * (1 - wh)) * (1 - occ_)
        uv = torch.cat([geo[:, 3:4].clamp(0, 1), rough.clamp(0, 1)], -1)
        fg = _fg_lookup_torch(self.lut[0], uv)
        diff_alb = (1 - met) * alb
        spec_alb = 0.04 * (1 - met) + met * alb
        spec_ref = spec_alb * fg[:, 0:1] + fg[:, 1:2]
        srgb = _linear_to_srgb_torch
        out = {'depth': depth, 'normal': ((torch.nn.functional.normalize(grads, dim=-1) + 1.0) * 0.5) * inner}
        inter = {'specular_albedo': spec_alb, 'specular_ref': spec_ref.clamp(0, 1), 'specular_light': srgb(spec_light).clamp(0, 1),
                 'specular_color': srgb(spec_ref * spec_light).clamp(0, 1), 'diffuse_albedo': diff_alb,
                 'diffuse_light': srgb(Ld).clamp(0, 1), 'diffuse_color': srgb(diff_alb * Ld).clamp(0, 1), 'metallic': met.clone(),
                 'roughness': rough.clone(), 'occ_prob': occ.clamp(0, 1), 'indirect_light': Li * occ_}
        if self.human:
            inter['human_light'] = srgb(Lh * wh)
        # occlusion ground truth: get_intersection(points, reflective, sn0=128, sn1=9) (field.py:454-484)
        sel = torch.nonzero(torch.norm(points, dim=-1) < 0.999)[:, 0].to(torch.int32).contiguous()
        P = int(sel.shape[0])
        gt = torch.zeros(R, 1, device=dev)
        if P > 0:
            var = self.p.deviation_network.variance.detach()
            if not hasattr(self, 't_lin128'):
                self.t_lin128 = torch.linspace(0, 1, 128).to(dev)
            chunk = w['SX0'].shape[0] // 128          # points per pass through the sampling workspace
            oo, dd = torch.empty(chunk, 3, device=dev), torch.empty(chunk, 3, device=dev)
            zz, nz, g_ = torch.empty(chunk, 128, device=dev), torch.empty(chunk, 16, device=dev), torch.empty(chunk, device=dev)
            for c0 in range(0, P, chunk):
                sl = sel[c0:c0 + chunk]
                pc = int(sl.shape[0])
                K('nero_occ_init', w['PTS'], w['REFL'], sl, None, pc, 128, self.t_lin128, oo, dd, zz, 128, w['SX0'], 64, w['SC'], 256)
                self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, pc * 128)
                K('nero_upsample', oo, dd, pc, zz, 128, w['SSDF'], 128, 128, 9, var, 3.0e38, 1, 1, nz, 16, w['SX0'], 64, w['SC'], 256, None)
                self.sdf.sdf_only(w['SX0'], w['SA'], w['SB'], w['SC'], w['SSDF'], None, pc * 9)
                K('nero_upsample', oo, dd, pc, nz, 16, w['SSDF'], 9, 9, 9, var, 3.0e38, 1, 1, None, 0, None, 0, None, 0, g_)
                gt[sl.long(), 0] = g_[:pc]
        out['occ_prob_gt'] = gt
        out.update({k: v * inner for k, v in inter.items()})
        return out

    # ------------------------------------------------------------------ render_core backward
    def render_core_backward(self, d_rgb, d_gerr, d_occ_scale, static=None):
        """d_rgb [R,3]; d_gerr [N_in] or None; d_occ_scale: float tensor [] = dL/d(loss_occ) / P or None.
        Accumulates into the .grad of every parameter.  Under graph capture (`static`) the caller has already made the .grad
        buffers the views of the persistent flat buffer."""
        self._alloc_backward()
        if static is None:
            self.grads.ensure()
        st, w, cfg = self.state, self.w, self.cfg
        R, S, cap = st['R'], st['S'], st['R'] * st['S']
        rays_d = st['rays_d']
        n_in, n_out = w['n_in'], w['n_out']
        var_p = self.p.deviation_network.variance
        var = var_p.detach()
        ws = self.ws
        K('nero_composite_bwd', w['slot'], R, S, w['ALPHA_IN'], w['COLOR_IN'], w['ALPHA_OUT'], w['COLOR_OUT'], d_rgb.contiguous(),
          w['dALPHA_IN'], w['dCOLOR_IN'], w['dALPHA_OUT'], w['dCOLOR_OUT'])
        # ---- outer NeRF
        K('nero_nerf_post_bwd', w['DENS'], 4, w['RGBRAW'], 4, w['DIST_OUT'], w['dALPHA_OUT'], w['dCOLOR_OUT'], w['dDENS'], 4, w['dRGBRAW'], 4,
          n_out, cap)
        self.nerf.backward(ws, w, n_out, cap)
        # ---- shading
        docc = None
        if d_occ_scale is not None and st['P'] > 0:
            docc = w['DOCC'] * d_occ_scale          # sign * dL/dloss_occ / P   (tiny elementwise op on [cap])
        K('nero_shade_combine_bwd', w['OUTS'], w['GEO'], self.lut, self.exp_max, 1 if self.human else 0, w['dCOLOR_IN'], docc, w['DOUTS'],
          w['DNOV'], n_in, cap)
        A = w['ACT']
        dH = (w['dHa'], w['dHb'], w['dHc'])
        ko = 144 if self.sphere else 72
        self.m_outer.backward(ws, Mat(w['DOUTS'], O_LDIR), Mat(w['E'], E_IDER), A['odir'], dH, n_in, cap, dX=Mat(w['dE_dir']), dx_ncol=ko)
        self.m_outer.backward(ws, Mat(w['DOUTS'], O_LD), Mat(w['E'], self.e_iden), A['odif'], dH, n_in, cap, dX=Mat(w['dE_dif']), dx_ncol=ko)
        self.m_inner.backward(ws, Mat(w['DOUTS'], O_LI), Mat(w['E'], E_PE8X), A['inner'], dH, n_in, cap, dX=Mat(w['dE_inn']), dx_ncol=72)
        self.m_iw.backward(ws, Mat(w['DOUTS'], O_IW), Mat(w['E'], 0), A['iw'], dH, n_in, cap)
        if self.human:
            self.m_human.backward(ws, Mat(w['DOUTS'], O_HUM), Mat(w['EH']), A['human'], dH, n_in, cap, dX=Mat(w['dEH']), dx_ncol=24)
        K('nero_shade_prep_bwd', w['G'], w['PTS'], w['RAY_IN'], rays_d, w['OUTS'], w['GEO'], w['dE_dir'], 160, w['dE_inn'], 128, w['dE_dif'], 160,
          w['dEH'] if self.human else None, 64, st['hp'], w['DNOV'], w['DOUTS'], w['DG'], n_in, cap, 1 if self.sphere else 0)
        matin = Mat(w['Y8'])
        self.m_rough.backward(ws, Mat(w['DOUTS'], O_ROUGH), matin, A['rough'], dH, n_in, cap, dX=Mat(w['dY8']), dx_ncol=256)
        self.m_met.backward(ws, Mat(w['DOUTS'], O_MET), matin, A['met'], dH, n_in, cap, dX=Mat(w['dY8']), dx_ncol=256, dx_addend=Mat(w['dY8']))
        self.m_alb.backward(ws, Mat(w['DOUTS'], O_ALB), matin, A['alb'], dH, n_in, cap, dX=Mat(w['dY8']), dx_ncol=256, dx_addend=Mat(w['dY8']))
        # ---- SDF -> alpha
        w['D_INV_S'].zero_()
        dg = None if d_gerr is None else d_gerr.contiguous()
        K('nero_sdf_alpha_bwd', w['Y8'], Y8_LD, Y8_SDF, w['G'], w['PTS'], w['RAY_IN'], rays_d, var, self.car_dev, w['dALPHA_IN'], dg,
          w['dY8'], Y8_LD, w['DG'], w['D_INV_S'], n_in, cap)
        frozen = cfg['freeze_inv_s_step'] is not None and st['step'] < cfg['freeze_inv_s_step']
        if not frozen:
            inv_s = torch.exp(var * 10.0)
            inr = ((inv_s >= 1e-6) & (inv_s <= 1e6)).float()
            var_p.grad.add_((w['D_INV_S'][0] * 10.0 * inv_s * inr).reshape(var_p.shape))
        # ---- SDF network (value + gradient paths)
        self.sdf.backward(ws, w, n_in, cap, None)
        ws.flush()
