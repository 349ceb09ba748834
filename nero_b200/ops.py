"""ctypes bindings of libnero_b200.so + thin tensor-level wrappers.

The product path has NO fallback and no alternate backend: importing this module without the built library raises, and
every wrapper launches a hand-written sm_90a kernel through the C ABI declared in include/nero_b200.h.  (The CPU walk of
the host logic used by the test-suite lives in tests/dry_run_harness.py and works by substituting `lib` from outside.)
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get('NERO_LIB') or os.path.join(_HERE, 'libnero_b200.so')   # NERO_LIB: A/B builds (profiling only)

ACT_NONE, ACT_SOFTPLUS100, ACT_RELU, ACT_SIGMOID, ACT_EXPCLAMP = 0, 1, 2, 3, 4
EPI_BIAS_ACT, EPI_MUL_DACT, EPI_TANGENT = 0, 1, 2
_NPADS = (16, 64, 128, 224, 256)

if not os.path.exists(_LIB_PATH):
    raise ImportError(f'{_LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                      '(nero_b200 has no CPU or PyTorch fallback)')
lib = ctypes.CDLL(_LIB_PATH)

launch_count = 0  # kernels launched through the C ABI (bench.py reports it)


def require_cuda(dev, what='nero_b200'):
    """The kernels run on a CUDA device only: there is no CPU path to fall back to."""
    if torch.device(dev).type != 'cuda':
        raise RuntimeError(f'{what} runs on a CUDA device only (move the module with .cuda(); there is no CPU fallback)')


def _ptr(t):
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, name):
    if rc != 0:
        raise RuntimeError(f'{name} failed with code {rc}')


def npad_for(n):
    for c in _NPADS:
        if n <= c:
            return c
    raise ValueError(f'width {n} > 256 not supported by one MMA tile')


def ceil_div(a, b):
    return (a + b - 1) // b


class PreparedLayer:
    """Tensor-core operand images of rows [row0,row0+nrows) of one linear layer, rebuilt by prep() whenever the
    parameters change (once per optimizer step).

    k_layout : width of the activation layout the layer reads (A operand columns actually touched)
    kmap     : reference input column -> layout column (None = identity)
    t_cols   : (c0, ncols) layout columns for which input gradients are needed (None = no dX image)
    """

    def __init__(self, weight, g, bias, device, row0=0, nrows=None, kmap=None, k_layout=None, t_cols=None):
        self.weight, self.g, self.bias = weight, g, bias
        N, K = weight.shape
        self.K = K
        self.row0 = row0
        self.nrows = N - row0 if nrows is None else nrows
        self.k_layout = k_layout if k_layout is not None else K
        self.kmap_host = kmap
        self.kmap = None if kmap is None else torch.tensor(kmap, dtype=torch.int32, device=device)
        self.n_pad = npad_for(self.nrows)
        self.k_chunks = ceil_div(self.k_layout, 64)
        self.k_valid = ceil_div(self.k_layout, 4) * 4
        self.img_f = torch.zeros(self.k_chunks * 2 * self.n_pad * 128, dtype=torch.uint8, device=device)
        self.t_cols = t_cols
        if t_cols is not None:
            self.t_npad = npad_for(t_cols[1])
            self.t_chunks = ceil_div(self.nrows, 64)
            self.img_t = torch.zeros(self.t_chunks * 2 * self.t_npad * 128, dtype=torch.uint8, device=device)
        else:
            self.img_t = None
        self.w_eff = torch.zeros(N, K, dtype=torch.float32, device=device)

    def prep(self):
        global launch_count
        w = self.weight.detach()
        g = None if self.g is None else self.g.detach()
        rc = lib.nero_prep_weight(_ptr(w), _ptr(g), self.K, self.row0, self.nrows, _ptr(self.kmap), ctypes.c_float(1.0),
                                  _ptr(self.img_f), self.n_pad, _ptr(self.img_t), self.t_npad if self.img_t is not None else 0,
                                  self.t_cols[0] if self.t_cols else 0, self.t_cols[1] if self.t_cols else 0,
                                  _ptr(self.w_eff), self.K, _stream())
        _check(rc, 'nero_prep_weight')
        launch_count += 1

    def bias_view(self):
        return None if self.bias is None else self.bias.detach()[self.row0:self.row0 + self.nrows]


_PREP_JOB = None


class PrepBatch:
    """PreparedLayer.prep() of many layers as ONE nero_prep_weight_batch launch.  The job table only holds device pointers;
    it is owned by the object that owns the layers (an engine) and is rebuilt whenever ANY pointer it holds changes
    (parameter storages after .to()/load_state_dict, operand images, kmaps), so a table can never outlive its buffers."""

    def __init__(self, layers):
        self.layers = list(layers)
        self.key, self.tab, self.max_rows = None, None, 0

    @staticmethod
    def _ptrs(l):
        p = lambda t: 0 if t is None else t.data_ptr()
        return (p(l.weight), p(l.g), p(l.kmap), p(l.img_f), p(l.img_t), p(l.w_eff))

    def run(self):
        global _PREP_JOB, launch_count
        if not self.layers:
            return
        import numpy as np
        if _PREP_JOB is None:
            _PREP_JOB = np.dtype([('v', 'u8'), ('g', 'u8'), ('kmap', 'u8'), ('img_f', 'u8'), ('img_t', 'u8'), ('w_eff', 'u8'), ('K', 'i4'),
                                  ('row0', 'i4'), ('nrows', 'i4'), ('rows_pad_f', 'i4'), ('rows_pad_t', 'i4'), ('t_c0', 'i4'),
                                  ('t_ncols', 'i4'), ('ld_weff', 'i4'), ('in_scale', 'f4'), ('pad', 'i4')])
            assert _PREP_JOB.itemsize == 88
        key = tuple(self._ptrs(l) for l in self.layers)
        if key != self.key:
            arr = np.zeros(len(self.layers), dtype=_PREP_JOB)
            for i, (l, pt) in enumerate(zip(self.layers, key)):
                arr[i] = pt + (l.K, l.row0, l.nrows, l.n_pad, l.t_npad if l.img_t is not None else 0, l.t_cols[0] if l.t_cols else 0,
                               l.t_cols[1] if l.t_cols else 0, l.K, 1.0, 0)
            self.tab = torch.from_numpy(arr.view(np.uint8).copy()).to(self.layers[0].img_f.device)
            self.key, self.max_rows = key, int(arr['nrows'].max())
        rc = lib.nero_prep_weight_batch(_ptr(self.tab), len(self.layers), self.max_rows, _stream())
        _check(rc, 'nero_prep_weight_batch')
        launch_count += 1


class Mat:
    """A column window [c0, c0+ncol) of a 2-D fp32 row-major device buffer."""
    __slots__ = ('t', 'c0', 'ncol')

    def __init__(self, t, c0=0, ncol=None):
        self.t, self.c0 = t, c0
        self.ncol = t.shape[1] - c0 if ncol is None else ncol

    @property
    def ld(self):
        return self.t.stride(0)

    def ptr(self):
        return ctypes.c_void_p(self.t.data_ptr() + 4 * self.c0)

    def view(self, m=None):
        v = self.t[:, self.c0:self.c0 + self.ncol]
        return v if m is None else v[:m]


def linear(A: Mat, layer: PreparedLayer, out: Mat, ncol_out, *, transposed=False, mode=EPI_BIAS_ACT, act=ACT_NONE,
           act_param=0.0, oscale=1.0, H: Mat = None, hscale=1.0, dact=ACT_NONE, V: Mat = None, out2: Mat = None,
           addend: Mat = None, ncol_main=None, tail: Mat = None, m_ptr=None, m_cap=None, use_bias=True):
    """out = epilogue(A @ W^T) (transposed=False) or epilogue(A @ W) restricted to t_cols (transposed=True)."""
    global launch_count
    if ncol_main is None:
        ncol_main = ncol_out
    if transposed:
        img, n_pad, k_chunks, k_valid = layer.img_t, layer.t_npad, layer.t_chunks, ceil_div(layer.nrows, 4) * 4
        bias = None
    else:
        img, n_pad, k_chunks, k_valid = layer.img_f, layer.n_pad, layer.k_chunks, layer.k_valid
        bias = layer.bias_view() if use_bias else None
    if m_cap is None:
        m_cap = A.t.shape[0]
    rc = lib.nero_linear(A.ptr(), A.ld, k_valid, _ptr(img), n_pad, k_chunks, _ptr(bias), 0 if bias is None else bias.numel(), out.ptr(), out.ld, ncol_out,
                         ctypes.c_float(oscale), mode, act, ctypes.c_float(act_param),
                         H.ptr() if H else None, H.ld if H else 0, ctypes.c_float(hscale), dact,
                         V.ptr() if V else None, V.ld if V else 0, out2.ptr() if out2 else None, out2.ld if out2 else 0,
                         addend.ptr() if addend else None, addend.ld if addend else 0, ncol_main,
                         tail.ptr() if tail else None, tail.ld if tail else 0, _ptr(m_ptr), m_cap, _stream())
    _check(rc, 'nero_linear')
    launch_count += 1


_FINISH_JOB = None


def _finish_job_dtype():
    global _FINISH_JOB
    if _FINISH_JOB is None:
        import numpy as np
        _FINISH_JOB = np.dtype([('partial', 'u8'), ('bias_partial', 'u8'), ('kmap', 'u8'), ('v', 'u8'), ('g', 'u8'), ('grad_w', 'u8'),
                                ('grad_g', 'u8'), ('grad_b', 'u8'), ('extra_row', 'u8'), ('P', 'i4'), ('rows_partial', 'i4'),
                                ('ld_partial', 'i4'), ('K', 'i4'), ('row0', 'i4'), ('nrows', 'i4'), ('in_scale', 'f4'),
                                ('extra_scale', 'f4')])
        assert _FINISH_JOB.itemsize == 104
    return _FINISH_JOB


class WgradWorkspace:
    """Accumulators of the weight-gradient GEMMs.  nero_wgrad splits the sample rows over `P` CTAs per output tile; CTA p adds
    its tile into slice p of a [P, rows, ld] fp32 accumulator, and the finish kernel sums the slices in a fixed order, so the
    gradients are the same every run (no floating-point atomics).
    With `defer` set (the engines do), every nero_wgrad launch gets its own accumulator slot and its weight-norm chain rule is
    queued; `flush()` runs all queued jobs in ONE nero_wgrad_finish_batch launch and re-zeroes the used slots (one memset).
    Jobs that would accumulate into the same gradient rows are never queued together (the queue is flushed first), so the
    batched kernel has no write conflicts."""

    def __init__(self, device, P=66, rows=256, ld=384, max_slots=48):
        self.P, self.rows, self.ld = P, rows, ld
        self.device, self.max_slots = device, max_slots
        # slot i = acc[i] [P, rows, ld] followed by its bias sums [P, rows]; zero = ready to accumulate into.  Slots are made
        # on first use and kept, so their addresses stay valid for graph replay
        self.slots = []
        self.jobs, self.dest, self.keep = [], set(), []
        self.defer = False
        self._tabs = {}      # device copies of the finish-job tables, keyed by their content: a training step queues the same
                             # jobs every iteration, so the steady state uploads nothing (and can be graph-captured)

    def _slot(self):
        i = len(self.jobs)
        while len(self.slots) <= i:
            self.slots.append(torch.zeros(self.P * (self.rows * self.ld + self.rows), dtype=torch.float32, device=self.device))
        row = self.slots[i]
        n = self.P * self.rows * self.ld
        return row[:n].view(self.P, self.rows, self.ld), row[n:].view(self.P, self.rows)

    @property
    def partial(self):
        return self._slot()[0]

    @property
    def bias_partial(self):
        return self._slot()[1]

    def enqueue(self, job, dest_key, keep):
        self.jobs.append(job)
        self.dest.add(dest_key)
        self.keep.append(keep)
        if len(self.jobs) >= self.max_slots:
            self.flush()

    def flush(self):
        global launch_count
        if not self.jobs:
            return
        key = tuple(self.jobs)
        hit = self._tabs.get(key)
        if hit is None:
            import numpy as np
            arr = np.zeros(len(self.jobs), dtype=_finish_job_dtype())
            for i, j in enumerate(self.jobs):
                arr[i] = j
            if len(self._tabs) >= 64:
                self._tabs.clear()
            hit = self._tabs[key] = (torch.from_numpy(arr.view(np.uint8).copy()).to(self.device), int(arr['nrows'].max()),
                                     int(arr['K'].max()))
        tab, max_rows, max_k = hit
        rc = lib.nero_wgrad_finish_batch(_ptr(tab), len(self.jobs), max_rows, max_k, _stream())
        _check(rc, 'nero_wgrad_finish_batch')
        launch_count += 1
        torch._foreach_zero_(self.slots[:len(self.jobs)])     # the used accumulators are ready for the next pass
        self.jobs, self.dest, self.keep = [], set(), []


def wgrad(ws: WgradWorkspace, dY: Mat, n_valid, X: Mat, k_valid, layer: PreparedLayer, grad_w, grad_g, grad_b,
          dY2: Mat = None, X2: Mat = None, m_ptr=None, m_cap=None, with_bias=True):
    """Accumulate d(weight_g, weight_v, bias) (or d(weight, bias)) of rows [row0,row0+nrows) of `layer` from
    dW_layout = dY^T X (+ dY2^T X2)."""
    global launch_count
    if m_cap is None:
        m_cap = dY.t.shape[0]
    n_rows_pad = ceil_div(n_valid, 16) * 16
    k_pad = ceil_div(layer.k_layout, 64) * 64
    assert k_pad <= ws.ld and n_rows_pad <= ws.rows
    if ws.defer and grad_w is not None and (grad_w.data_ptr(), layer.row0) in ws.dest:
        ws.flush()                      # a queued job already accumulates into these rows
    partial_t, bias_t = ws.partial, ws.bias_partial
    P = ws.P          # row slices per 128-row output tile, one accumulator slice each
    if not ws.defer:          # stand-alone use: the accumulator slot is zeroed per call
        partial_t.zero_()
        bias_t.zero_()
    rc = lib.nero_wgrad(dY.ptr(), dY.ld, n_valid, X.ptr(), X.ld, k_valid,
                        dY2.ptr() if dY2 else None, dY2.ld if dY2 else 0, X2.ptr() if X2 else None, X2.ld if X2 else 0,
                        _ptr(partial_t), ws.ld, ws.rows, _ptr(bias_t), n_rows_pad, k_pad, P, _ptr(m_ptr),
                        m_cap, _stream())
    _check(rc, 'nero_wgrad')
    launch_count += ceil_div(n_rows_pad, 128) * max(1, ceil_div(k_pad, 256))
    g = None if layer.g is None else layer.g.detach()
    w_ = layer.weight.detach()
    if ws.defer:
        ptr = lambda t: 0 if t is None else t.data_ptr()
        job = (ptr(partial_t), ptr(bias_t) if with_bias else 0, ptr(layer.kmap), ptr(w_), ptr(g), ptr(grad_w), ptr(grad_g),
               ptr(grad_b) if with_bias else 0, 0, P, ws.rows, ws.ld, layer.K, layer.row0, layer.nrows, 1.0, 0.0)
        ws.enqueue(job, (grad_w.data_ptr(), layer.row0), (w_, g))
        return
    rc = lib.nero_wgrad_finish(_ptr(partial_t), P, ws.rows, ws.ld, _ptr(bias_t) if with_bias else None,
                               layer.K, layer.row0, layer.nrows, _ptr(layer.kmap), ctypes.c_float(1.0),
                               _ptr(w_), _ptr(g), _ptr(grad_w), _ptr(grad_g),
                               _ptr(grad_b) if with_bias else None, None, ctypes.c_float(0.0), _stream())
    _check(rc, 'nero_wgrad_finish')
    launch_count += 1


def colsum(X: Mat, ncol, out, w: Mat = None, m_ptr=None, m_cap=None):
    global launch_count
    if m_cap is None:
        m_cap = X.t.shape[0]
    rc = lib.nero_colsum(X.ptr(), X.ld, ncol, w.ptr() if w else None, w.ld if w else 0, _ptr(m_ptr), m_cap, _ptr(out),
                         _stream())
    _check(rc, 'nero_colsum')
    launch_count += 1


def K(name, *args):
    """Generic launcher: tensors / Mat -> device pointers, float -> c_float, int stays int, None -> NULL; the
    current CUDA stream is appended as the last argument."""
    global launch_count
    conv = []
    for a in args:
        if a is None:
            conv.append(ctypes.c_void_p(0))
        elif isinstance(a, torch.Tensor):
            conv.append(ctypes.c_void_p(a.data_ptr()))
        elif isinstance(a, Mat):
            conv.append(a.ptr())
        elif isinstance(a, float):
            conv.append(ctypes.c_float(a))
        elif isinstance(a, ctypes._SimpleCData):
            conv.append(a)
        else:
            conv.append(int(a))
    rc = getattr(lib, name)(*conv, _stream())
    _check(rc, name)
    launch_count += 1


# ------------------------------------------------------------------------------------------------ stand-alone encodings
def positional_encoding(x, L, scale=1.0):
    """get_embedder(L, d)[0](x) (network/field.py:14-58) for d = 3 or 4 on the CUDA path: [M, d] -> [M, d(1+2L)]."""
    global launch_count
    x = x.contiguous().float()
    M, d = x.shape
    out = torch.empty(M, d * (1 + 2 * L), device=x.device)
    rc = lib.nero_pe(_ptr(x), d, d, M, L, ctypes.c_float(scale), _ptr(out), out.shape[1], _stream())
    _check(rc, 'nero_pe')
    launch_count += 1
    return out


def integrated_dir_enc(dirs, kappa_inv):
    """generate_ide_fn(5)(dirs, kappa_inv) (utils/ref_utils.py:53-117) on the CUDA path: [M,3], [M,1] or float -> [M,72]."""
    global launch_count
    from .engine import upload_ide_table
    upload_ide_table()
    dirs = dirs.contiguous().float()
    M = dirs.shape[0]
    out = torch.empty(M, 72, device=dirs.device)
    if torch.is_tensor(kappa_inv):
        k = kappa_inv.reshape(-1).contiguous().float()
        rc = lib.nero_ide(_ptr(dirs), 3, _ptr(k), 1, ctypes.c_float(0.0), M, _ptr(out), 72, _stream())
    else:
        rc = lib.nero_ide(_ptr(dirs), 3, None, 0, ctypes.c_float(float(kappa_inv)), M, _ptr(out), 72, _stream())
    _check(rc, 'nero_ide')
    launch_count += 1
    return out


# ------------------------------------------------------------------------------------------------ fused MLP chain
EK_BIAS_SOFTPLUS, EK_BIAS_RELU, EK_BIAS_GENERIC, EK_DACT_SOFTPLUS, EK_DACT_RELU, EK_DACT_NONE, EK_TANGENT = range(7)


class _ChainLayer(ctypes.Structure):
    _fields_ = [('wimg', ctypes.c_void_p), ('bias', ctypes.c_void_p),
                ('save', ctypes.c_void_p), ('H', ctypes.c_void_p), ('addend', ctypes.c_void_p), ('V', ctypes.c_void_p),
                ('out2', ctypes.c_void_p), ('tail', ctypes.c_void_p),
                ('n_pad', ctypes.c_int), ('k_chunks', ctypes.c_int), ('n_bias', ctypes.c_int), ('ncol_out', ctypes.c_int),
                ('ncol_main', ctypes.c_int), ('kind', ctypes.c_int), ('act', ctypes.c_int),
                ('ld_save', ctypes.c_int), ('ldh', ctypes.c_int), ('ldadd', ctypes.c_int), ('ldv', ctypes.c_int),
                ('ldo2', ctypes.c_int), ('ldt', ctypes.c_int),
                ('oscale', ctypes.c_float), ('hscale', ctypes.c_float), ('act_param', ctypes.c_float),
                ('write_a', ctypes.c_int), ('a_blocks', ctypes.c_int),
                ('csrc', ctypes.c_void_p), ('ld_csrc', ctypes.c_int), ('pad_', ctypes.c_int)]


class _ChainParams(ctypes.Structure):
    _fields_ = [('A0', ctypes.c_void_p), ('lda0', ctypes.c_int), ('k_valid0', ctypes.c_int),
                ('n_layers', ctypes.c_int), ('m_ptr', ctypes.c_void_p), ('m_cap', ctypes.c_int),
                ('L', _ChainLayer * 10)]


def _p(m):
    if m is None:
        return None
    if isinstance(m, Mat):
        return m.t.data_ptr() + 4 * m.c0
    return m.data_ptr()


def chain_layer(layer: PreparedLayer, kind, ncol_out, *, transposed=False, save: Mat = None, act=ACT_NONE, act_param=0.0, oscale=1.0,
                H: Mat = None, hscale=1.0, V: Mat = None, out2: Mat = None, addend: Mat = None, ncol_main=None, tail: Mat = None,
                write_a=True, csrc: Mat = None, use_bias=True):
    """Describe one layer of a fused chain (same semantics as ops.linear for the matching kind)."""
    return dict(layer=layer, kind=kind, ncol_out=ncol_out, transposed=transposed, save=save, act=act, act_param=act_param, oscale=oscale,
                H=H, hscale=hscale, V=V, out2=out2, addend=addend, ncol_main=ncol_out if ncol_main is None else ncol_main, tail=tail,
                write_a=write_a, csrc=csrc, use_bias=use_bias)


PROFILE = None   # bench.py: list collecting (tag, event0, event1, flops_per_row, m_ptr_addr, m_cap) per chain launch


def chain(A0: Mat, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
    """Run consecutive layers on each 128-row tile with the A operand kept in shared memory (k_gemm_chain.cu)."""
    global launch_count
    assert 1 <= len(layers) <= 10
    if m_cap is None:
        m_cap = A0.t.shape[0]
    P = _ChainParams()
    P.A0, P.lda0, P.k_valid0 = _p(A0), A0.ld, ceil_div(k_valid0, 4) * 4
    P.n_layers, P.m_ptr, P.m_cap = len(layers), _p(m_ptr), m_cap
    keep = []
    for i, d in enumerate(layers):
        lay, L = d['layer'], P.L[i]
        if d['transposed']:
            img, n_pad, k_chunks, bias = lay.img_t, lay.t_npad, lay.t_chunks, None
        else:
            img, n_pad, k_chunks = lay.img_f, lay.n_pad, lay.k_chunks
            bias = lay.bias_view() if d['use_bias'] else None
        assert k_chunks <= 4 and d['ncol_out'] <= n_pad
        keep.append(bias)
        L.wimg, L.bias, L.n_bias = _p(img), _p(bias), 0 if bias is None else bias.numel()
        L.n_pad, L.k_chunks, L.ncol_out, L.ncol_main, L.kind, L.act = n_pad, k_chunks, d['ncol_out'], d['ncol_main'], d['kind'], d['act']
        for name, key, ldname in (('save', 'save', 'ld_save'), ('H', 'H', 'ldh'), ('addend', 'addend', 'ldadd'), ('V', 'V', 'ldv'),
                                  ('out2', 'out2', 'ldo2'), ('tail', 'tail', 'ldt'), ('csrc', 'csrc', 'ld_csrc')):
            m = d[key]
            setattr(L, name, _p(m))
            setattr(L, ldname, m.ld if m is not None else 0)
        L.oscale, L.hscale, L.act_param = d['oscale'], d['hscale'], d['act_param']
        L.write_a = 1 if (d['write_a'] and i + 1 < len(layers)) else 0
        nxt = layers[i + 1]['layer'] if i + 1 < len(layers) else None
        if nxt is not None:
            nk = nxt.t_chunks if layers[i + 1]['transposed'] else nxt.k_chunks
            L.a_blocks = 4 * nk
    if PROFILE is not None:
        fl = 0.0
        for d in layers:
            lay = d['layer']
            kdim = lay.nrows if d['transposed'] else lay.K
            fl += 2.0 * kdim * d['ncol_out']
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    rc = lib.nero_chain(ctypes.byref(P), _stream())
    _check(rc, 'nero_chain')
    launch_count += 1
    if PROFILE is not None:
        e1.record()
        PROFILE.append((tag, e0, e1, fl, None if m_ptr is None else m_ptr.data_ptr(), m_cap))


# ------------------------------------------------------------------------------------------------ stage II (k_mcshade.cu, k_bvh.cu)
_vp, _ci, _cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


class McParams(ctypes.Structure):
    """Mirror of nero_mc_params (include/nero_b200.h)."""
    _fields_ = [('pts', _vp), ('normals', _vp), ('view', _vp), ('rough', _vp), ('poses', _vp), ('rand_d', _vp), ('rand_s', _vp),
                ('tab_d', _vp), ('tab_s', _vp), ('P', _ci), ('Sd', _ci), ('Ss', _ci), ('ggx_smith', _ci), ('sphere_dir', _ci),
                ('human', _ci), ('org', _vp), ('dir', _vp), ('pos_depth', _vp), ('nrm_hit', _vp), ('slot', _vp), ('blk_cnt', _vp),
                ('blk_off', _vp), ('counts', _vp), ('EO', _vp), ('ldeo', _ci), ('EH', _vp), ('ldeh', _ci), ('hhit', _vp), ('EI', _vp),
                ('ldei', _ci), ('OUT_O', _vp), ('OUT_H', _vp), ('OUT_I', _vp), ('exp_max_o', _cf), ('exp_max_i', _cf), ('LD', _vp),
                ('LS', _vp), ('LSF', _vp), ('dLD', _vp), ('dLS', _vp), ('dLSF', _vp), ('DPRE_O', _vp), ('DPRE_H', _vp), ('DPRE_I', _vp),
                ('dA', _vp), ('dEO', _vp), ('dEH', _vp), ('dEI', _vp), ('dA2', _vp)]

    def set(self, **kw):
        for k, v in kw.items():
            if isinstance(v, torch.Tensor):
                v = v.data_ptr()
            elif isinstance(v, Mat):
                v = v.t.data_ptr() + 4 * v.c0
            setattr(self, k, v)
        return self


def mc(name, params: McParams):
    """Launch one of the nero_mc_* kernels on the current stream."""
    global launch_count
    rc = getattr(lib, name)(ctypes.byref(params), _stream())
    _check(rc, name)
    launch_count += 1


def bvh_build(verts, tris):
    """Host BVH build through the C ABI: numpy verts [V,3] f32, tris [T,3] i32 -> (nodes uint8 [n,32], tri float32 [T,12],
    tri_ids int32 [T]) as numpy arrays ready to upload."""
    import numpy as np
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    T = tris.shape[0]
    nodes = np.zeros((2 * T, 32), np.uint8)
    tri = np.zeros((T, 12), np.float32)
    ids = np.zeros(T, np.int32)
    n = ctypes.c_int(0)
    rc = lib.nero_bvh_build_host(verts.ctypes.data_as(_vp), verts.shape[0], tris.ctypes.data_as(_vp), T, nodes.ctypes.data_as(_vp),
                                 tri.ctypes.data_as(_vp), ids.ctypes.data_as(_vp), ctypes.byref(n))
    _check(rc, 'nero_bvh_build_host')
    return nodes[:n.value].copy(), tri, ids
