"""ctypes bindings of libnero_b200.so + thin tensor-level wrappers.

The product path has NO fallback and no alternate backend: importing this module without the built library raises, and
every wrapper launches a hand-written sm_90a kernel through the C ABI declared in include/nero_b200.h.  The bindings are
read from that header at import: every entry point gets its prototype (argtypes), every struct a ctypes.Structure with
the header's fields.  (The CPU walk of the host logic used by the test-suite lives in tests/dry_run_harness.py and works
by substituting `lib` from outside.)
"""
import ctypes
import os
import re

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.environ.get('NERO_LIB') or os.path.join(_HERE, 'libnero_b200.so')   # NERO_LIB: A/B builds (profiling only)
_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_b200.h')
_TEXMAP_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_texmap.h')   # same library, plain-argument entry points
_ENVMAP_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_envmap.h')   # same library, plain-argument entry points
_METRICS_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_metrics.h')  # same library, plain-argument entry points
_RELIGHT_TEX_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_relight_tex.h')   # same library, plain arguments
_MESHPTS_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_meshpts.h')  # same library, plain-argument entry points
_OBJPREP_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_objprep.h')  # same library, plain-argument entry points
_MCSPARSE_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_mcsparse.h')  # same library, plain-argument entry points
_MVS_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_mvs.h')  # same library, plain-argument entry points
_FEATURES_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_features.h')  # same library, plain-argument entry points
_SFM_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_sfm.h')  # same library, plain-argument entry points
_SIMPLIFY_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_simplify.h')  # same library, plain-argument entry points
_DENOISE_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_denoise.h')  # same library, plain-argument entry points
_NORMALMAP_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_normalmap.h')  # same library, plain-argument entry points
_GLTF_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_gltf.h')  # same library, plain-argument entry points
_OCCLUSION_HEADER = os.path.join(os.path.dirname(_HERE), 'include', 'nero_occlusion.h')  # same library, plain-argument entry points

ACT_NONE, ACT_SOFTPLUS100, ACT_RELU, ACT_SIGMOID, ACT_EXPCLAMP = 0, 1, 2, 3, 4
EPI_BIAS_ACT, EPI_MUL_DACT, EPI_TANGENT = 0, 1, 2
_NPADS = (16, 64, 128, 224, 256)

if not os.path.exists(_LIB_PATH):
    raise ImportError(f'{_LIB_PATH} is missing: run `python -c "import __graft_entry__ as g; g.build()"` '
                      '(nero_b200 has no CPU or PyTorch fallback)')
lib = ctypes.CDLL(_LIB_PATH)

launch_count = 0  # kernels launched through the C ABI (bench.py reports it)


def _addr(a):
    """Address of a tensor, a Mat (its column c0), a numpy array or a ctypes struct; anything else is returned as is."""
    if a is None:
        return None
    if a.__class__ is Mat:
        return a.t.data_ptr() + 4 * a.c0
    if isinstance(a, torch.Tensor):
        return a.data_ptr()
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if isinstance(a, ctypes.Structure):
        return ctypes.addressof(a)
    return a


_CArgObject = type(ctypes.byref(ctypes.c_int()))


class Ptr(ctypes.c_void_p):
    """The parameter type of every pointer of the C ABI: accepts None, an int address, a tensor, a Mat, a numpy array, a
    ctypes struct or byref(...)."""

    @staticmethod
    def from_param(a, _vp=ctypes.c_void_p, _tensor=torch.Tensor, _pass=(_CArgObject, ctypes.c_void_p)):
        # runs for every pointer argument of every launch: the common cases first, without a further call
        if a.__class__ is Mat:
            return _vp(a.t.data_ptr() + 4 * a.c0)
        if isinstance(a, _tensor):
            return _vp(a.data_ptr())
        if a is None or isinstance(a, _pass):
            return a
        return _vp(_addr(a))


class Struct(ctypes.Structure):
    """Base of the structs read from the header."""

    def set(self, **kw):
        for k, v in kw.items():
            setattr(self, k, _addr(v))
        return self


_CTYPES = {'int': ctypes.c_int, 'unsigned int': ctypes.c_uint, 'float': ctypes.c_float, 'double': ctypes.c_double,
           'long long': ctypes.c_longlong}


def _parse_header(path):
    """-> ({struct name: Struct subclass}, {entry point: argtypes}) from the typedefs and prototypes of the C header."""
    txt = re.sub(r'/\*.*?\*/', ' ', open(path).read(), flags=re.S)
    txt = re.sub(r'^\s*#.*$', ' ', txt, flags=re.M)
    structs = {}
    for body, name in re.findall(r'typedef\s+struct\s+\w*\s*\{(.*?)\}\s*(\w+)\s*;', txt, re.S):
        fields = []
        for decl in filter(None, (d.strip() for d in body.split(';'))):
            first, *rest = decl.split(',')
            base, var = re.match(r'(.*?)(\**\s*\w+\s*(?:\[\d+\])?)$', first.strip()).groups()
            base = base.replace('const', '').strip()
            for v in [var] + rest:
                ptr, fname, n = re.match(r'\s*(\**)\s*(\w+)\s*(?:\[(\d+)\])?\s*$', v).groups()
                t = ctypes.c_void_p if ptr or '*' in base else (structs.get(base) or _CTYPES[base])
                fields.append((fname, t * int(n) if n else t))
        structs[name] = type(name, (Struct,), {'_fields_': fields})
    protos = {}
    for name, params in re.findall(r'\bint\s+(nero_\w+)\s*\(([^)]*)\)\s*;', txt):
        decls = [p.strip() for p in params.split(',') if p.strip() not in ('', 'void')]
        protos[name] = [Ptr if '*' in p else _CTYPES[re.sub(r'\s+\w+$', '', p).replace('const', '').strip()] for p in decls]
    return structs, protos


STRUCTS, _PROTOS = _parse_header(_HEADER)
TEXMAP_PROTOS = _parse_header(_TEXMAP_HEADER)[1]
ENVMAP_PROTOS = _parse_header(_ENVMAP_HEADER)[1]
METRICS_PROTOS = _parse_header(_METRICS_HEADER)[1]
RELIGHT_TEX_PROTOS = _parse_header(_RELIGHT_TEX_HEADER)[1]
MESHPTS_PROTOS = _parse_header(_MESHPTS_HEADER)[1]
OBJPREP_PROTOS = _parse_header(_OBJPREP_HEADER)[1]
MCSPARSE_PROTOS = _parse_header(_MCSPARSE_HEADER)[1]
MVS_PROTOS = _parse_header(_MVS_HEADER)[1]
FEATURES_PROTOS = _parse_header(_FEATURES_HEADER)[1]
SFM_PROTOS = _parse_header(_SFM_HEADER)[1]
SIMPLIFY_PROTOS = _parse_header(_SIMPLIFY_HEADER)[1]
DENOISE_PROTOS = _parse_header(_DENOISE_HEADER)[1]
NORMALMAP_PROTOS = _parse_header(_NORMALMAP_HEADER)[1]
GLTF_PROTOS = _parse_header(_GLTF_HEADER)[1]
OCCLUSION_PROTOS = _parse_header(_OCCLUSION_HEADER)[1]
for _name, _argtypes in (list(_PROTOS.items()) + list(TEXMAP_PROTOS.items()) + list(ENVMAP_PROTOS.items()) +
                         list(METRICS_PROTOS.items()) + list(RELIGHT_TEX_PROTOS.items()) + list(MESHPTS_PROTOS.items()) +
                         list(OBJPREP_PROTOS.items()) + list(MCSPARSE_PROTOS.items()) + list(MVS_PROTOS.items()) +
                         list(FEATURES_PROTOS.items()) + list(SFM_PROTOS.items()) + list(SIMPLIFY_PROTOS.items()) +
                         list(DENOISE_PROTOS.items()) + list(NORMALMAP_PROTOS.items()) + list(GLTF_PROTOS.items()) +
                         list(OCCLUSION_PROTOS.items())):
    _fn = getattr(lib, _name)
    _fn.argtypes, _fn.restype = _argtypes, ctypes.c_int
# nero_abi_sizeof(i) is the size of ABI_RECORDS[i]; a library built from another version of the header would read the
# structs of every launch wrongly
ABI_RECORDS = ('nero_chain_layer', 'nero_chain_params', 'nero_mc_params', 'nero_finish_job', 'nero_prep_job', 'nero_relight_params',
               'nero_depth_params')
for _i, _name in enumerate(ABI_RECORDS):
    if lib.nero_abi_sizeof(_i) != ctypes.sizeof(STRUCTS[_name]):
        raise ImportError(f'{_LIB_PATH}: {_name} is {lib.nero_abi_sizeof(_i)} bytes in the library but '
                          f'{ctypes.sizeof(STRUCTS[_name])} in {_HEADER}: rebuild the library')
ChainParams, McParams, RelightParams, DepthParams = (STRUCTS[f'nero_{n}_params'] for n in ('chain', 'mc', 'relight', 'depth'))
_PREP_JOB, _FINISH_JOB = np.dtype(STRUCTS['nero_prep_job']), np.dtype(STRUCTS['nero_finish_job'])


def require_cuda(dev, what='nero_b200'):
    """The kernels run on a CUDA device only: there is no CPU path to fall back to."""
    if torch.device(dev).type != 'cuda':
        raise RuntimeError(f'{what} runs on a CUDA device only (move the module with .cuda(); there is no CPU fallback)')


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def call(name, *args):
    """Call entry point `name` of the library; a non-zero return code raises."""
    rc = getattr(lib, name)(*args)
    if rc != 0:
        raise RuntimeError(f'{name} failed with code {rc}')


def K(name, *args, launches=1):
    """Launch entry point `name` on the current CUDA stream (appended as its last argument) and count its kernels."""
    global launch_count
    rc = getattr(lib, name)(*args, _stream())
    if rc != 0:
        raise RuntimeError(f'{name} failed with code {rc}')
    launch_count += launches


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
        K('nero_prep_weight', self.weight, self.g, self.K, self.row0, self.nrows, self.kmap, 1.0, self.img_f, self.n_pad, self.img_t,
          self.t_npad if self.img_t is not None else 0, self.t_cols[0] if self.t_cols else 0, self.t_cols[1] if self.t_cols else 0,
          self.w_eff, self.K)

    def bias_view(self):
        return None if self.bias is None else self.bias.detach()[self.row0:self.row0 + self.nrows]

    def operand(self, transposed, use_bias=True):
        """(image, n_pad, k_chunks, k_valid, bias) of a GEMM through this layer: forward (out = A W^T + b over the layout
        columns) or transposed (out = A W restricted to t_cols, contracting over the nrows outputs, no bias)."""
        if transposed:
            return self.img_t, self.t_npad, self.t_chunks, ceil_div(self.nrows, 4) * 4, None
        return self.img_f, self.n_pad, self.k_chunks, self.k_valid, self.bias_view() if use_bias else None


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
        if not self.layers:
            return
        key = tuple(self._ptrs(l) for l in self.layers)
        if key != self.key:
            arr = np.zeros(len(self.layers), dtype=_PREP_JOB)
            for i, (l, pt) in enumerate(zip(self.layers, key)):
                arr[i] = pt + (l.K, l.row0, l.nrows, l.n_pad, l.t_npad if l.img_t is not None else 0, l.t_cols[0] if l.t_cols else 0,
                               l.t_cols[1] if l.t_cols else 0, l.K, 1.0, 0)
            self.tab = torch.from_numpy(arr.view(np.uint8).copy()).to(self.layers[0].img_f.device)
            self.key, self.max_rows = key, int(arr['nrows'].max())
        K('nero_prep_weight_batch', self.tab, len(self.layers), self.max_rows)


class Mat:
    """A column window [c0, c0+ncol) of a 2-D fp32 row-major device buffer."""
    __slots__ = ('t', 'c0', 'ncol')

    def __init__(self, t, c0=0, ncol=None):
        self.t, self.c0 = t, c0
        self.ncol = t.shape[1] - c0 if ncol is None else ncol

    @property
    def ld(self):
        return self.t.stride(0)

    def view(self, m=None):
        v = self.t[:, self.c0:self.c0 + self.ncol]
        return v if m is None else v[:m]


def linear(A: Mat, layer: PreparedLayer, out: Mat, ncol_out, *, transposed=False, mode=EPI_BIAS_ACT, act=ACT_NONE,
           act_param=0.0, oscale=1.0, H: Mat = None, hscale=1.0, dact=ACT_NONE, V: Mat = None, out2: Mat = None,
           addend: Mat = None, ncol_main=None, tail: Mat = None, m_ptr=None, m_cap=None, use_bias=True):
    """out = epilogue(A @ W^T) (transposed=False) or epilogue(A @ W) restricted to t_cols (transposed=True)."""
    if ncol_main is None:
        ncol_main = ncol_out
    img, n_pad, k_chunks, k_valid, bias = layer.operand(transposed, use_bias)
    if m_cap is None:
        m_cap = A.t.shape[0]
    K('nero_linear', A, A.ld, k_valid, img, n_pad, k_chunks, bias, 0 if bias is None else bias.numel(), out, out.ld, ncol_out,
      oscale, mode, act, act_param, H, H.ld if H else 0, hscale, dact, V, V.ld if V else 0, out2, out2.ld if out2 else 0,
      addend, addend.ld if addend else 0, ncol_main, tail, tail.ld if tail else 0, m_ptr, m_cap)


class WgradWorkspace:
    """Split-K slices of the weight-gradient GEMMs.  nero_wgrad splits the sample rows over `P` CTAs per output tile; CTA p
    stores its tile into slice p of a [P, rows, ld] fp32 slot, and the finish kernel sums the slices in a fixed order, so the
    gradients are the same every run (no floating-point atomics).  Every launch stores its whole window of every slice
    (zeros where a CTA has no samples) and the finish reads only that window, so slots are never zeroed.
    With `defer` set (the engines do), every nero_wgrad launch gets its own slot and its weight-norm chain rule is queued;
    `flush()` runs all queued jobs in ONE nero_wgrad_finish_batch launch.
    Jobs that would accumulate into the same gradient rows are never queued together (the queue is flushed first), so the
    batched kernel has no write conflicts."""

    def __init__(self, device, P=66, rows=256, ld=384, max_slots=48):
        self.P, self.rows, self.ld = P, rows, ld
        self.device, self.max_slots = device, max_slots
        # slot i = slices[i] [P, rows, ld] followed by its bias sums [P, rows].  Slots are made on first use and kept, so their
        # addresses stay valid for graph replay
        self.slots = []
        self.jobs, self.dest, self.keep = [], set(), []
        self.defer = False
        self._tabs = {}      # device copies of the finish-job tables, keyed by their content: a training step queues the same
                             # jobs every iteration, so the steady state uploads nothing (and can be graph-captured)

    def _slot(self):
        i = len(self.jobs)
        while len(self.slots) <= i:
            self.slots.append(torch.empty(self.P * (self.rows * self.ld + self.rows), dtype=torch.float32, device=self.device))
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
        if not self.jobs:
            return
        key = tuple(self.jobs)
        hit = self._tabs.get(key)
        if hit is None:
            arr = np.zeros(len(self.jobs), dtype=_FINISH_JOB)
            for i, j in enumerate(self.jobs):
                arr[i] = j
            if len(self._tabs) >= 64:
                self._tabs.clear()
            hit = self._tabs[key] = (torch.from_numpy(arr.view(np.uint8).copy()).to(self.device), int(arr['nrows'].max()),
                                     int(arr['K'].max()))
        tab, max_rows, max_k = hit
        K('nero_wgrad_finish_batch', tab, len(self.jobs), max_rows, max_k)
        self.jobs, self.dest, self.keep = [], set(), []


def wgrad(ws: WgradWorkspace, dY: Mat, n_valid, X: Mat, k_valid, layer: PreparedLayer, grad_w, grad_g, grad_b,
          dY2: Mat = None, X2: Mat = None, m_ptr=None, m_cap=None, with_bias=True):
    """Accumulate d(weight_g, weight_v, bias) (or d(weight, bias)) of rows [row0,row0+nrows) of `layer` from
    dW_layout = dY^T X (+ dY2^T X2)."""
    if m_cap is None:
        m_cap = dY.t.shape[0]
    n_rows_pad = ceil_div(n_valid, 16) * 16
    k_pad = ceil_div(layer.k_layout, 64) * 64
    # the finish reads slice rows [0, nrows) and columns kmap[k] < k_layout: all inside the window the launches store
    assert k_pad <= ws.ld and n_rows_pad <= ws.rows and layer.nrows <= n_rows_pad
    if ws.defer and grad_w is not None and (grad_w.data_ptr(), layer.row0) in ws.dest:
        ws.flush()                      # a queued job already accumulates into these rows
    partial_t, bias_t = ws.partial, ws.bias_partial
    P = ws.P          # row slices per 128-row output tile, one slice each
    K('nero_wgrad', dY, dY.ld, n_valid, X, X.ld, k_valid, dY2, dY2.ld if dY2 else 0, X2, X2.ld if X2 else 0,
      partial_t, ws.ld, ws.rows, bias_t, n_rows_pad, k_pad, P, m_ptr, m_cap,
      launches=ceil_div(n_rows_pad, 128) * max(1, ceil_div(k_pad, 256)))
    g = None if layer.g is None else layer.g.detach()
    w_ = layer.weight.detach()
    if ws.defer:
        ptr = lambda t: 0 if t is None else t.data_ptr()
        job = (ptr(partial_t), ptr(bias_t) if with_bias else 0, ptr(layer.kmap), ptr(w_), ptr(g), ptr(grad_w), ptr(grad_g),
               ptr(grad_b) if with_bias else 0, 0, P, ws.rows, ws.ld, layer.K, layer.row0, layer.nrows, 1.0, 0.0)
        ws.enqueue(job, (grad_w.data_ptr(), layer.row0), (w_, g))
        return
    K('nero_wgrad_finish', partial_t, P, ws.rows, ws.ld, bias_t if with_bias else None, layer.K, layer.row0, layer.nrows, layer.kmap,
      1.0, w_, g, grad_w, grad_g, grad_b if with_bias else None, None, 0.0)


def colsum(X: Mat, ncol, out, w: Mat = None, m_ptr=None, m_cap=None):
    if m_cap is None:
        m_cap = X.t.shape[0]
    K('nero_colsum', X, X.ld, ncol, w, w.ld if w else 0, m_ptr, m_cap, out)


# ------------------------------------------------------------------------------------------------ stand-alone encodings
def positional_encoding(x, L, scale=1.0):
    """get_embedder(L, d)[0](x) (network/field.py:14-58) for d = 3 or 4 on the CUDA path: [M, d] -> [M, d(1+2L)]."""
    x = x.contiguous().float()
    M, d = x.shape
    out = torch.empty(M, d * (1 + 2 * L), device=x.device)
    K('nero_pe', x, d, d, M, L, scale, out, out.shape[1])
    return out


def integrated_dir_enc(dirs, kappa_inv):
    """generate_ide_fn(5)(dirs, kappa_inv) (utils/ref_utils.py:53-117) on the CUDA path: [M,3], [M,1] or float -> [M,72]."""
    from .engine import upload_ide_table
    upload_ide_table()
    dirs = dirs.contiguous().float()
    M = dirs.shape[0]
    out = torch.empty(M, 72, device=dirs.device)
    if torch.is_tensor(kappa_inv):
        K('nero_ide', dirs, 3, kappa_inv.reshape(-1).contiguous().float(), 1, 0.0, M, out, 72)
    else:
        K('nero_ide', dirs, 3, None, 0, float(kappa_inv), M, out, 72)
    return out


# ------------------------------------------------------------------------------------------------ fused MLP chain
EK_BIAS_SOFTPLUS, EK_BIAS_RELU, EK_BIAS_GENERIC, EK_DACT_SOFTPLUS, EK_DACT_RELU, EK_DACT_NONE, EK_TANGENT = range(7)


def chain_layer(layer: PreparedLayer, kind, ncol_out, *, transposed=False, save: Mat = None, act=ACT_NONE, act_param=0.0, oscale=1.0,
                H: Mat = None, hscale=1.0, V: Mat = None, out2: Mat = None, addend: Mat = None, ncol_main=None, tail: Mat = None,
                write_a=True, csrc: Mat = None, use_bias=True, store=True):
    """Describe one layer of a fused chain (same semantics as ops.linear for the matching kind).  store=False (read by
    mlp()): the fused chain gets no `save` and keeps the output in shared memory only; the per-layer expansion still writes
    `save`, because its next launch reads the output from there."""
    return dict(layer=layer, kind=kind, ncol_out=ncol_out, transposed=transposed, save=save, act=act, act_param=act_param, oscale=oscale,
                H=H, hscale=hscale, V=V, out2=out2, addend=addend, ncol_main=ncol_out if ncol_main is None else ncol_main, tail=tail,
                write_a=write_a, csrc=csrc, use_bias=use_bias, store=store)


PROFILE = None   # bench.py: list collecting (tag, event0, event1, flops_per_row, m_ptr_addr, m_cap) per chain launch
CHAIN_PHASES = None   # tools/chain_phases.py: int64 device counters the NERO_CHAIN_PHASES build adds each launch's phases to


def chain(A0: Mat, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
    """Run consecutive layers on each 128-row tile with the A operand kept in shared memory (k_gemm_chain.cu)."""
    if m_cap is None:
        m_cap = A0.t.shape[0]
    P = ChainParams()
    assert 1 <= len(layers) <= len(P.L)
    P.A0, P.lda0, P.k_valid0 = _addr(A0), A0.ld, ceil_div(k_valid0, 4) * 4
    P.n_layers, P.m_ptr, P.m_cap = len(layers), _addr(m_ptr), m_cap
    P.phase_clk = _addr(CHAIN_PHASES)
    opnd = [d['layer'].operand(d['transposed'], d['use_bias']) for d in layers]
    for i, d in enumerate(layers):
        L = P.L[i]
        img, n_pad, k_chunks, _, bias = opnd[i]
        assert k_chunks <= 4 and d['ncol_out'] <= n_pad
        L.wimg, L.bias, L.n_bias = _addr(img), _addr(bias), 0 if bias is None else bias.numel()
        L.n_pad, L.k_chunks, L.ncol_out, L.ncol_main, L.kind, L.act = n_pad, k_chunks, d['ncol_out'], d['ncol_main'], d['kind'], d['act']
        for name, ldname in (('save', 'ld_save'), ('H', 'ldh'), ('addend', 'ldadd'), ('V', 'ldv'), ('out2', 'ldo2'), ('tail', 'ldt'),
                             ('csrc', 'ld_csrc')):
            m = d[name]
            setattr(L, name, _addr(m))
            setattr(L, ldname, m.ld if m is not None else 0)
        L.oscale, L.hscale, L.act_param = d['oscale'], d['hscale'], d['act_param']
        L.write_a = 1 if (d['write_a'] and i + 1 < len(layers)) else 0
        if i + 1 < len(layers):
            L.a_blocks = 4 * opnd[i + 1][2]
    if PROFILE is not None:
        fl = 0.0
        for d in layers:
            lay = d['layer']
            kdim = lay.nrows if d['transposed'] else lay.K
            fl += 2.0 * kdim * d['ncol_out']
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
    K('nero_chain', ctypes.byref(P))
    if PROFILE is not None:
        e1.record()
        PROFILE.append((tag, e0, e1, fl, None if m_ptr is None else m_ptr.data_ptr(), m_cap))


# chain kind -> the nero_linear (mode, act, dact) with the same epilogue; act None: the descriptor's own act
_LINEAR_EPILOGUE = {EK_BIAS_SOFTPLUS: (EPI_BIAS_ACT, ACT_SOFTPLUS100, ACT_NONE), EK_BIAS_RELU: (EPI_BIAS_ACT, ACT_RELU, ACT_NONE),
                    EK_BIAS_GENERIC: (EPI_BIAS_ACT, None, ACT_NONE), EK_DACT_SOFTPLUS: (EPI_MUL_DACT, ACT_NONE, ACT_SOFTPLUS100),
                    EK_DACT_RELU: (EPI_MUL_DACT, ACT_NONE, ACT_RELU), EK_DACT_NONE: (EPI_MUL_DACT, ACT_NONE, ACT_NONE),
                    EK_TANGENT: (EPI_TANGENT, ACT_NONE, ACT_SOFTPLUS100)}


def mlp(A0: Mat, layers, m_ptr=None, m_cap=None, tag='', fused=True):
    """Run a pass stated as chain_layer descriptors; A0 holds the first layer's input.

    fused: the leading layers whose operand has more than 4 K chunks (K > 256 does not fit the chain's shared-memory A
    operand) run as nero_linear, the rest as one nero_chain.  Otherwise every layer is one nero_linear launch with the same
    epilogue, so the per-layer path runs exactly the layers of the fused one.  The next layer reads the output a layer
    saves when it has write_a, else the same A (the heads)."""
    A = A0
    for i, d in enumerate(layers):
        _, _, k_chunks, k_valid, _ = d['layer'].operand(d['transposed'], False)
        if fused and k_chunks <= 4:
            chain(A, k_valid, [d if d['store'] else dict(d, save=None) for d in layers[i:]], m_ptr, m_cap, tag)
            return
        mode, act, dact = _LINEAR_EPILOGUE[d['kind']]
        save = d['save']
        linear(A, d['layer'], save, d['ncol_out'], transposed=d['transposed'], mode=mode, act=d['act'] if act is None else act,
               act_param=d['act_param'], oscale=d['oscale'], H=d['H'], hscale=d['hscale'], dact=dact, V=d['V'], out2=d['out2'],
               addend=d['addend'], ncol_main=d['ncol_main'], tail=d['tail'], m_ptr=m_ptr, m_cap=m_cap, use_bias=d['use_bias'])
        # a skip-concat's extra columns are already in the saved output's buffer: the next layer reads them from there
        assert d['csrc'] is None or (d['csrc'].t is save.t and d['csrc'].c0 == save.c0)
        if d['write_a']:
            A = Mat(save.t, save.c0)


# ------------------------------------------------------------------------------------------------ stage II (k_bvh.cu)
def bvh_build(verts, tris):
    """Host BVH build through the C ABI: numpy verts [V,3] f32, tris [T,3] i32 -> (nodes uint8 [n,32], tri float32 [T,12],
    tri_ids int32 [T]) as numpy arrays ready to upload."""
    verts = np.ascontiguousarray(verts, np.float32)
    tris = np.ascontiguousarray(tris, np.int32)
    T = tris.shape[0]
    nodes = np.zeros((2 * T, 32), np.uint8)
    tri = np.zeros((T, 12), np.float32)
    ids = np.zeros(T, np.int32)
    n = ctypes.c_int(0)
    call('nero_bvh_build_host', verts, verts.shape[0], tris, T, nodes, tri, ids, ctypes.byref(n))
    return nodes[:n.value].copy(), tri, ids
