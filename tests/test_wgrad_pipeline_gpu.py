"""nero_wgrad + its finish against the fp64 restatement in gemm_ref.py, at the shapes a training step uses and at the edges
of the operand stream: aligned operands arrive by tensor copies (16-row boxes that zero-fill columns past the limit and
rows past m_cap; rows in [M, m_cap) are zeroed as they are converted), unaligned ones by per-thread copies.  Each case
runs twice and must give the same bits both times."""
import pytest
import torch

import gemm_ref as R
from test_gemm_gpu import _mk_layer

pytestmark = pytest.mark.gpu

# (M, cap, N, K, two, column offset of dY / X).  P = 66 CTAs per 128-row tile, 32-sample chunks.
CASES = {
    'step_one_pair': (127217, 127217, 256, 256, False, 0),    # the bench row count; the last CTA holds 5 chunks
    'step_two_pairs': (127217, 127217, 256, 256, True, 0),
    'nerf_layer': (36600, 36600, 256, 283, False, 0),         # <256> + <64> launches, X columns past k_valid
    'M_not_chunk_multiple': (1031, 1031, 256, 128, False, 0),  # one <128> launch; a partial 16-row box
    'empty_ctas': (33, 33, 217, 64, True, 0),                  # one <64> launch; 64 of 66 CTAs have no samples
    'device_count_below_cap': (5003, 9000, 256, 256, False, 0),  # rows [M, cap) hold NaN / inf
    'unaligned_operands': (4097, 4097, 200, 256, True, 1),     # the per-thread (scalar) copies
    'aligned_offset': (4097, 4097, 256, 256, False, 4),        # 16-byte aligned column windows
}


def _run(ops, ws, L, dY, N, X, dY2, X2, m_ptr, cap, off):
    gw, gg, gb = torch.zeros_like(L.weight), torch.zeros_like(L.g), torch.zeros(N, device=dY.device)
    ops.wgrad(ws, ops.Mat(dY, off), N, ops.Mat(X, off), L.k_valid, L, gw, gg, gb,
              None if dY2 is None else ops.Mat(dY2, off), None if X2 is None else ops.Mat(X2, off), m_ptr=m_ptr, m_cap=cap)
    torch.cuda.synchronize()
    return gw, gg, gb


@pytest.mark.parametrize('case', sorted(CASES))
def test_wgrad_matches_fp64_and_repeats(case):
    from nero_b200 import ops
    M, cap, N, K, two, off = CASES[case]
    dev = torch.device('cuda')
    L, _, _ = _mk_layer(ops, N, K, dev, seed=M + K)
    gen = torch.Generator(device=dev).manual_seed(M)
    mk = lambda cols, s: torch.randn(cap, cols + off, device=dev, generator=gen) * s
    dY, X = mk(256, 0.1), mk(320, 1.0)
    dY2, X2 = (mk(256, 0.1), mk(320, 1.0)) if two else (None, None)
    for t in (dY, X, dY2, X2):
        if t is not None:
            t[M:] = float('nan')                    # rows past the device count are never read
    m_ptr = torch.tensor([M], dtype=torch.int32, device=dev)
    ws = ops.WgradWorkspace(dev)
    first = _run(ops, ws, L, dY, N, X, dY2, X2, m_ptr, cap, off)
    second = _run(ops, ws, L, dY, N, X, dY2, X2, m_ptr, cap, off)
    for a, b in zip(first, second):
        assert torch.equal(a, b)

    win = lambda t: None if t is None else t[:M, off:]
    dW, dWa, db, dba = R.wgrad_layout(win(dY), N, win(X), L.k_valid, win(dY2), win(X2))
    fv, fg, fb = R.wgrad_finish(L, dW, dWa, db, dba, 2.0 ** -24 * R.ceil_div(max(M, 1), ws.P) ** 0.5)
    for name, got, f in (('dv', first[0], fv), ('dg', first[1], fg), ('bias', first[2], fb)):
        assert torch.isfinite(got).all(), name
        ok, err, bound = R.frob_ok(got.double().reshape(f[0].shape), *f)
        assert ok, f'{case} {name}: ||got - ref||_F = {err:.3e} > {bound:.3e}'
