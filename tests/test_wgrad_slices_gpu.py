"""Write-once split-K slices of nero_wgrad: every launch stores its whole window of every slice (zeros where a CTA has no
samples), so the workspace slots are never zeroed.  Slots filled with NaN must give the same gradients, bit for bit, as
zeroed slots: stand-alone calls (device row counts that leave trailing CTAs without rows, M = 0, one row past a chunk
boundary), a deferred training step, and a graph replay."""
import pytest
import torch

from test_gemm_gpu import _mk_layer
from test_graph_gpu import make, one_step

pytestmark = pytest.mark.gpu


def _fill_slots(ws, value):
    for s in ws.slots:
        s.fill_(value)


# P = 66 CTAs per tile, 32-sample chunks: 2113 rows = 67 chunks (2 per CTA, CTAs 34..65 empty, one row past a boundary),
# 33 rows = 2 chunks (64 empty CTAs), 0 rows (every CTA empty), 127217 rows (the bench count: the last CTA holds 5 chunks)
@pytest.mark.parametrize('M', [0, 1, 33, 2113, 127217])
@pytest.mark.parametrize('N,K,two', [(256, 256, True), (217, 283, False), (3, 39, False)])
def test_standalone_wgrad_ignores_slot_contents(M, N, K, two):
    from nero_b200 import ops
    dev = torch.device('cuda')
    cap = max(M, 1) + 40
    L, _, _ = _mk_layer(ops, N, K, dev, seed=M + N)
    gen = torch.Generator(device=dev).manual_seed(7)
    dY = torch.randn(cap, 256, device=dev, generator=gen) * 0.1
    X = torch.randn(cap, 320, device=dev, generator=gen)
    dY2 = torch.randn(cap, 256, device=dev, generator=gen) * 0.1 if two else None
    X2 = torch.randn(cap, 320, device=dev, generator=gen) if two else None
    dY[M:], X[M:] = float('nan'), float('inf')        # rows past the device count are never read
    m_ptr = torch.tensor([M], dtype=torch.int32, device=dev)
    ws = ops.WgradWorkspace(dev)
    ws.partial                                          # make slot 0
    grads = []
    for fill in (0.0, float('nan')):
        _fill_slots(ws, fill)
        gw, gg, gb = torch.zeros_like(L.weight), torch.zeros_like(L.g), torch.zeros(N, device=dev)
        ops.wgrad(ws, ops.Mat(dY), N, ops.Mat(X), L.k_valid, L, gw, gg, gb, ops.Mat(dY2) if two else None,
                  ops.Mat(X2) if two else None, m_ptr=m_ptr, m_cap=cap)
        torch.cuda.synchronize()
        grads.append((gw, gg, gb))
    for a, b in zip(*grads):
        assert torch.isfinite(b).all() and torch.equal(a, b)
    if M == 0:
        assert all(float(t.abs().max()) == 0.0 for t in grads[1])


def test_deferred_step_and_graph_replay_ignore_slot_contents():
    net, R = make('shape_bell_r32', {'perturb': 0.0})
    ws = net.engine.ws
    net.cfg['cuda_graph'] = False
    one_step(net, 30000)                                # makes the slots
    res = []
    for fill in (0.0, float('nan')):
        _fill_slots(ws, fill)
        net.train_batch_i = 0
        res.append(one_step(net, 30000))
    (o0, l0, g0), (o1, l1, g1) = res
    assert l0 == l1 and all(torch.equal(g0[n], g1[n]) for n in g0)

    net.cfg['cuda_graph'] = True
    net.train_batch_i = 0
    one_step(net, 30000)                                # capture
    res = []
    for fill in (0.0, float('nan')):
        _fill_slots(ws, fill)
        net.train_batch_i = 0
        res.append(one_step(net, 30000))                # replay
    (o0, l0, g0), (o1, l1, g1) = res
    assert l0 == l1 and torch.equal(o0['ray_rgb'], o1['ray_rgb'])
    for n in g0:
        assert torch.isfinite(g1[n]).all() and torch.equal(g0[n], g1[n]), n
