"""TEST INFRASTRUCTURE: walk the host-side logic of nero_b200 on CPU tensors without launching a kernel.

The product package has no alternate backend; this harness substitutes things from OUTSIDE:
  * `ops.lib` is wrapped: every device entry point becomes a no-op returning 0 (host-only entry points -- the BVH builder,
    the ABI self-checks -- still run for real) once its arguments pass the prototype the bindings read from the header
    (count, then each argtype's from_param), so the walk checks the signature of every call site it reaches; the few entry
    points whose device-side counts drive host control flow write plausible counts through the (CPU) pointers they were given;
  * `ops._stream` returns a null stream, `ops.require_cuda` accepts any device;
  * `ops.linear / chain / wgrad` are wrapped with the argument / buffer-shape assertions a wrong call sequence would trip,
    and every GEMM layer they launch is appended to GEMMS.
Numerical results are meaningless in this mode.
"""
import ctypes

from nero_b200 import ops

GEMMS = []    # (PreparedLayer, transposed, ncol_out) of every nero_linear launch and every nero_chain layer, in launch order


class FakeLib:
    HOST_ONLY = {'nero_bvh_build_host', 'nero_abi_sizeof', 'nero_version'}

    def __init__(self, real):
        self._real = real
        self.calls = 0

    def __getattr__(self, name):
        real = getattr(self._real, name)         # a symbol the library does not export is still an error
        if name in self.HOST_ONLY:
            return real

        def fake(*args):
            assert len(args) == len(real.argtypes), f'{name}: {len(args)} arguments for {len(real.argtypes)} parameters'
            for i, (t, a) in enumerate(zip(real.argtypes, args)):
                try:
                    t.from_param(a)
                except (TypeError, ValueError) as e:
                    raise AssertionError(f'{name}: argument {i} ({a!r}) does not convert to {t.__name__}: {e}') from None
            self.calls += 1
            hook = getattr(self, '_hook_' + name, None)
            if hook is not None:
                hook(*args)
            return 0
        return fake

    @staticmethod
    def _poke(ptr, value, ctype=ctypes.c_int):
        addr = ops._addr(ptr)
        if addr:
            ctype.from_address(addr).value = int(value)

    # (rays_o, rays_d, z_vals, R, S, cnt_in, cnt_out, off_in, off_out, n_in, n_out, stream)
    def _hook_nero_ray_prepare(self, *a):
        R, S = a[3], a[4]
        self._poke(a[9], min(100, R * S))
        self._poke(a[10], max(R * S - 100, 0))

    # (..., n_in, cap, SEL, OCC_COUNT, stream): more candidates than occ_loss_max_pn so the random-subset branch is walked
    def _hook_nero_occ_select(self, *a):
        self._poke(a[-2], min(3000, int(a[-4])))

    # (rays_o, rays_d, z_vals, R, S, radius, cnt, dummy, off, dummy, n, dummy1, stream)
    def _hook_nero_reg_prepare(self, *a):
        self._poke(a[10], min(50, a[3] * a[4]))

    # (u, nx, ny, nz, iso, blk_cnt, blk_off, totals, stream): totals = (V, T) as long long
    def _hook_nero_mcubes_count(self, *a):
        self._poke(a[7], 6, ctypes.c_longlong)
        self._poke(ops._addr(a[7]) + 8, 2, ctypes.c_longlong)

    # (depth, n_views, height, width, lo, hi, blk_cnt, blk_off, total, stream)
    def _hook_nero_depth_points_count(self, *a):
        self._poke(a[8], min(5, a[1] * a[2] * a[3]), ctypes.c_longlong)

    def _hook_nero_mc_classify(self, p, stream):
        n = p.P * (p.Sd + p.Ss)
        if p.counts:
            ctypes.c_int.from_address(p.counts).value = n // 4
            ctypes.c_int.from_address(p.counts + 4).value = n - n // 4


def install():
    if isinstance(ops.lib, FakeLib):
        return ops.lib
    ops.lib = FakeLib(ops.lib)
    ops._stream = lambda: ctypes.c_void_p(0)
    ops.require_cuda = lambda dev, what='nero_b200': None

    real_linear, real_chain, real_wgrad = ops.linear, ops.chain, ops.wgrad

    def linear(A, layer, out, ncol_out, *, transposed=False, mode=ops.EPI_BIAS_ACT, H=None, V=None, out2=None, **kw):
        img, n_pad, _, k_valid, _ = layer.operand(transposed, False)
        GEMMS.append((layer, transposed, ncol_out))
        assert A.ld % 4 == 0 and A.c0 % 4 == 0 and ncol_out <= n_pad and img is not None
        assert A.c0 + k_valid <= A.t.shape[1] and out.c0 + ncol_out <= out.t.shape[1], (A.c0, k_valid, A.t.shape, out.c0, ncol_out, out.t.shape)
        assert mode != ops.EPI_TANGENT or (H is not None and V is not None and out2 is not None)
        return real_linear(A, layer, out, ncol_out, transposed=transposed, mode=mode, H=H, V=V, out2=out2, **kw)

    def chain(A0, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
        assert A0.c0 % 4 == 0 and A0.ld % 4 == 0 and A0.c0 + ops.ceil_div(k_valid0, 4) * 4 <= A0.t.shape[1]
        for d in layers:
            lay = d['layer']
            GEMMS.append((lay, d['transposed'], d['ncol_out']))
            assert lay.operand(d['transposed'], False)[0] is not None
            if d['kind'] in (ops.EK_DACT_SOFTPLUS, ops.EK_DACT_RELU, ops.EK_TANGENT):
                assert d['H'] is not None
            if d['kind'] == ops.EK_TANGENT:
                assert d['V'] is not None and d['out2'] is not None
            if d['save'] is not None:
                assert d['save'].c0 + min(d['ncol_out'], d['ncol_main']) <= d['save'].t.shape[1]
        return real_chain(A0, k_valid0, layers, m_ptr, m_cap, tag)

    def wgrad(ws, dY, n_valid, X, k_valid, layer, grad_w, grad_g, grad_b, dY2=None, X2=None, m_ptr=None, m_cap=None, with_bias=True):
        assert grad_w is not None and (grad_b is not None or not with_bias) and (layer.g is None or grad_g is not None)
        assert dY.c0 + n_valid <= dY.t.shape[1] and X.c0 + k_valid <= X.t.shape[1], (dY.c0, n_valid, dY.t.shape, X.c0, k_valid, X.t.shape)
        return real_wgrad(ws, dY, n_valid, X, k_valid, layer, grad_w, grad_g, grad_b, dY2, X2, m_ptr, m_cap, with_bias)

    ops.linear, ops.chain, ops.wgrad = linear, chain, wgrad
    # modules that imported the names directly
    import nero_b200.engine as E
    import nero_b200.material as M
    for mod in (E, M):
        for name, fn in (('linear', linear), ('chain', chain), ('wgrad', wgrad)):
            if hasattr(mod, name):
                setattr(mod, name, fn)
    return ops.lib
