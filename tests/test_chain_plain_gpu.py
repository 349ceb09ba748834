"""The fused chain's two epilogues: plain layers (all 256 columns main, 8-byte pair stores; k_gemm_chain.cu chain_layer)
and general ones (skip-concat layer, heads, narrow outputs, misaligned outputs) mixed in one chain.

Every chain runs twice: once with each output window (`save`, `out2`, `tail`) at column 0 of its buffer, which keeps the
256-wide layers plain, and once at column 1, one float off 8-byte alignment, which makes every layer with an output
general.  Both runs must store bit-identical values, leave every element outside the written windows as it was (rows
past the device-side row count included, whose inputs are NaN), and match the fp64 restatement of tests/gemm_ref.py
layer by layer, each layer fed with the fp32 output the chain stored for the layer before it."""
import pytest
import torch

import gemm_ref as R
from test_gemm_gpu import _mk_layer

pytestmark = pytest.mark.gpu

SENT = -7.0
W_BUF = 258          # output buffers: a 256-wide window at column 0 or 1, row stride even either way


def _buf(cap, dev):
    return torch.full((cap, W_BUF), SENT, device=dev)


def _check_layer(d, A, m, got, got2=None, got_tail=None, ins=None):
    """gemm_ref bound check of one layer on rows [0, m): A is the fp64 input [m, >= 64 k_chunks]."""
    layer, kind = d['layer'], d['kind']
    W, kv = R.operand(layer, d['transposed'])
    A = A[:m, :W.shape[1]].clone()
    A[:, kv:] = 0
    acc, S = A @ W.t(), A.abs() @ W.abs().t()
    bias = layer.operand(d['transposed'], d['use_bias'])[4]
    dd = dict(d, bias=None if bias is None else bias.double())
    nmain, res = R.epilogue(kind, acc, S, dd, ins or {})
    for name, g in (('main', got), ('out2', got2), ('tail', got_tail)):
        if name in res:
            ref, bound = res[name]
            g = g[:m, :ref.shape[1]].double()
            assert bool(((g - ref).abs() <= bound).all()), f'{name}: max err {float((g - ref).abs().max()):.3e}'
    return nmain


def _next_a(saved, nmain, m, csrc=None, width=256):
    A = torch.zeros(m, width, dtype=torch.float64, device=saved.device)
    A[:, :nmain] = saved[:m, :nmain].double()
    if csrc is not None:
        A[:, nmain:] = csrc[:m, nmain:width].double()
    return A


def _bits(t):
    return t.contiguous().view(torch.int32)


def _run_twice(make, bufs, win):
    """make(off) runs the chain with its outputs at column `off`; returns {name: window} of the aligned run after
    checking the two runs against each other."""
    out = {}
    for off in (0, 1):
        for b in bufs.values():
            b.fill_(SENT)
        make(off)
        torch.cuda.synchronize()
        out[off] = {k: b.clone() for k, b in bufs.items()}
    for k in bufs:
        a, b = out[0][k], out[1][k]
        w = win[k]
        assert torch.equal(_bits(a[:, :w]), _bits(b[:, 1:1 + w])), f'{k}: aligned and offset outputs differ'
        assert bool((a[:, w:] == SENT).all()) and bool((b[:, 0] == SENT).all()) and bool((b[:, 1 + w:] == SENT).all()), \
            f'{k}: written outside its columns'
    return out[0]


CASES = [(127, 127), (128, 128), (129, 200), (16895, 16895), (16897, 16897), (16896, 20000), (40007, 45000)]


def _inputs(m, cap, width, dev, seed, scale=0.5):
    g = torch.Generator().manual_seed(seed)
    X = (torch.randn(cap, width, generator=g) * scale).to(dev)
    X[m:] = float('nan')                     # stale rows past the device-side count
    return X


def _mcount(m, cap, dev):
    return (torch.tensor([m], dtype=torch.int32, device=dev), cap) if cap > m else (None, None)


@pytest.mark.parametrize('M,cap', CASES)
def test_forward_chain_plain_and_general(M, cap):
    """39 -> 256 (plain) -> 217 + skip-concat (general) -> 256 (plain, softplus) -> 256 (plain, ReLU) -> 1 (head)."""
    from nero_b200 import ops
    from nero_b200.ops import Mat, chain, chain_layer as CL
    dev = torch.device('cuda')
    L0, _, _ = _mk_layer(ops, 256, 39, dev, seed=21)
    L1, _, _ = _mk_layer(ops, 217, 256, dev, seed=22)
    L2, _, _ = _mk_layer(ops, 256, 256, dev, seed=23)
    L3, _, _ = _mk_layer(ops, 256, 256, dev, seed=24)
    L4, _, _ = _mk_layer(ops, 1, 256, dev, seed=25)
    X = torch.zeros(cap, 64, device=dev)
    X[:, :39] = _inputs(M, cap, 39, dev, M)
    skip = X[:, :39] * 0.5
    B = {k: _buf(cap, dev) for k in ('h1', 'h2', 'h3', 'h4', 'o')}
    m_ptr, m_cap = _mcount(M, cap, dev)
    descs = {}

    def make(off):
        B['h2'][:M, off + 217:off + 256] = skip[:M]          # concat source, pre-stored in the save buffer
        w = lambda k, n=256: Mat(B[k], off, n)
        ls = [CL(L0, ops.EK_BIAS_SOFTPLUS, 256, save=w('h1')),
              CL(L1, ops.EK_BIAS_SOFTPLUS, 217, oscale=0.70710678, save=w('h2'), csrc=w('h2')),
              CL(L2, ops.EK_BIAS_SOFTPLUS, 256, save=w('h3')),
              CL(L3, ops.EK_BIAS_RELU, 256, save=w('h4')),
              CL(L4, ops.EK_BIAS_GENERIC, 1, act=3, save=w('o', 1), write_a=False)]
        descs.update(zip(('h1', 'h2', 'h3', 'h4', 'o'), ls))
        chain(Mat(X), 39, ls, m_ptr=m_ptr, m_cap=m_cap)

    got = _run_twice(make, B, {'h1': 256, 'h2': 256, 'h3': 256, 'h4': 256, 'o': 1})
    for k in got:
        assert bool((got[k][M:] == SENT).all()), f'{k}: rows past the row count written'
    A = X[:M].double()
    for k in ('h1', 'h2', 'h3', 'h4', 'o'):
        d = descs[k]
        nmain = _check_layer(d, A, M, got[k])
        A = _next_a(got[k], nmain, M, csrc=got[k] if d['csrc'] is not None else None)


@pytest.mark.parametrize('M,cap', CASES)
def test_gradient_chain_plain_and_general(M, cap):
    """Reverse sweep: 256 (plain, dsoftplus) -> 256 (plain, dReLU + addend) -> 217 + tail (general) -> 39 (U0, general)."""
    from nero_b200 import ops
    from nero_b200.ops import Mat, chain, chain_layer as CL
    dev = torch.device('cuda')
    L0, _, _ = _mk_layer(ops, 256, 39, dev, seed=31, t_cols=(0, 39))
    L1, _, _ = _mk_layer(ops, 217, 256, dev, seed=32, t_cols=(0, 256))
    L2, _, _ = _mk_layer(ops, 256, 256, dev, seed=33, t_cols=(0, 256))
    L3, _, _ = _mk_layer(ops, 256, 256, dev, seed=34, t_cols=(0, 256))
    G = _inputs(M, cap, 256, dev, M + 1, 1.0)
    H3 = _inputs(M, cap, 256, dev, M + 2, 0.05).abs()
    H2 = _inputs(M, cap, 256, dev, M + 3, 1.0)
    H1 = _inputs(M, cap, 256, dev, M + 4, 0.05).abs()
    add = _inputs(M, cap, 256, dev, M + 5, 1.0)
    B = {k: _buf(cap, dev) for k in ('g3', 'g2', 'g1', 'tl', 'g0')}
    m_ptr, m_cap = _mcount(M, cap, dev)
    descs = {}

    def make(off):
        w = lambda k, n=256: Mat(B[k], off, n)
        ls = [CL(L3, ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H3), save=w('g3')),
              CL(L2, ops.EK_DACT_RELU, 256, transposed=True, H=Mat(H2), addend=Mat(add), save=w('g2')),
              CL(L1, ops.EK_DACT_SOFTPLUS, 256, transposed=True, oscale=0.70710678, H=Mat(H1), hscale=1.41421356,
                 ncol_main=217, tail=w('tl', 39), save=w('g1')),
              CL(L0, ops.EK_DACT_NONE, 39, transposed=True, save=w('g0', 39))]
        descs.update(zip(('g3', 'g2', 'g1', 'g0'), ls))
        chain(Mat(G), 256, ls, m_ptr=m_ptr, m_cap=m_cap)

    got = _run_twice(make, B, {'g3': 256, 'g2': 256, 'g1': 217, 'tl': 39, 'g0': 39})
    for k in got:
        assert bool((got[k][M:] == SENT).all()), f'{k}: rows past the row count written'
    A = G[:M].double()
    ins = {'g3': {'H': H3}, 'g2': {'H': H2, 'addend': add}, 'g1': {'H': H1}, 'g0': {}}
    for k in ('g3', 'g2', 'g1', 'g0'):
        d = descs[k]
        nm = min(d['ncol_out'], d['ncol_main'])
        i = {n: t[:M, :nm].double() for n, t in ins[k].items()}
        nmain = _check_layer(d, A, M, got[k], got_tail=got['tl'] if k == 'g1' else None, ins=i)
        A = _next_a(got[k], nmain, M)


@pytest.mark.parametrize('M,cap', CASES)
def test_tangent_chain_plain_and_general(M, cap):
    """Tangent sweep: 39 -> 256 (plain) -> 217 + skip-concat (general) -> 256 (plain) -> 256 (plain)."""
    from nero_b200 import ops
    from nero_b200.ops import Mat, chain, chain_layer as CL
    dev = torch.device('cuda')
    Ls = [_mk_layer(ops, n, k, dev, seed=41 + i)[0] for i, (n, k) in enumerate(((256, 39), (217, 256), (256, 256), (256, 256)))]
    U0 = torch.zeros(cap, 64, device=dev)
    U0[:, :39] = _inputs(M, cap, 39, dev, M + 6, 1.0)
    H = [_inputs(M, cap, 256, dev, M + 10 + i, 0.04).abs() for i in range(4)]
    V = [_inputs(M, cap, 256, dev, M + 20 + i, 1.0) for i in range(4)]
    skip = _inputs(M, cap, 39, dev, M + 7, 1.0)
    names = [('u1', 'q0'), ('u2', 'q1'), ('u3', 'q2'), ('u4', 'q3')]
    B = {k: _buf(cap, dev) for pair in names for k in pair}
    m_ptr, m_cap = _mcount(M, cap, dev)
    descs = []

    def make(off):
        B['u2'][:M, off + 217:off + 256] = skip[:M]
        w = lambda k, n=256: Mat(B[k], off, n)
        ls = []
        for i, (u, q) in enumerate(names):
            kw = dict(oscale=0.70710678, hscale=1.41421356, csrc=w(u)) if i == 1 else {}
            ls.append(CL(Ls[i], ops.EK_TANGENT, 217 if i == 1 else 256, use_bias=False, H=Mat(H[i]), V=Mat(V[i]),
                         out2=w(q), save=w(u), **kw))
        descs[:] = ls
        chain(Mat(U0), 40, ls, m_ptr=m_ptr, m_cap=m_cap)

    got = _run_twice(make, B, {k: 256 for k in B})
    for k in got:
        assert bool((got[k][M:] == SENT).all()), f'{k}: rows past the row count written'
    A = U0[:M].double()
    for i, (u, q) in enumerate(names):
        d = descs[i]
        nm = d['ncol_out']
        nmain = _check_layer(d, A, M, got[u], got2=got[q], ins={'H': H[i][:M, :nm].double(), 'V': V[i][:M, :nm].double()})
        A = _next_a(got[u], nmain, M, csrc=got[u] if d['csrc'] is not None else None)
