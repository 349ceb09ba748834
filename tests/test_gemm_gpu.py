"""GPU parity of the wgmma GEMM kernels (nero_linear / nero_wgrad) against fp64 torch on the same inputs.
Tolerance: the split-bf16 3-MMA scheme carries ~2^-17 relative error per product (DESIGN.md); we require
max|err| <= 2e-5 * (|A| @ |W|^T) element-wise scale, i.e. far below the 1e-4 output tolerance of north_star."""
import numpy as np
import pytest
import torch

from helpers import act_ref, dact_ref

pytestmark = pytest.mark.gpu


def _mk_layer(ops, N, K, dev, wn=True, kmap=None, k_layout=None, t_cols=None, row0=0, nrows=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    v = (torch.randn(N, K, generator=g) / np.sqrt(K)).to(dev)
    gg = (1.0 + 0.1 * torch.randn(N, 1, generator=g)).to(dev) if wn else None
    b = (0.1 * torch.randn(N, generator=g)).to(dev)
    L = ops.PreparedLayer(v, gg, b, dev, row0=row0, nrows=nrows, kmap=kmap, k_layout=k_layout, t_cols=t_cols)
    L.prep()
    W = (gg * v / v.norm(dim=1, keepdim=True)) if wn else v
    return L, W.double(), b.double()


def _err(got, want, scale):
    e = (got.double() - want).abs()
    return float((e / (scale + 1e-30)).max()), float(e.max())


@pytest.mark.parametrize('M,K,N,act', [(1000, 39, 256, 1), (4113, 256, 256, 1), (300, 256, 217, 1), (2500, 256, 1, 0),
                                       (777, 256, 3, 3), (129, 72, 256, 2), (5000, 283, 128, 2), (40000, 256, 256, 2)])
def test_linear_bias_act(M, K, N, act):
    from nero_b200 import ops
    dev = torch.device('cuda')
    torch.manual_seed(M)
    k_layout = K
    L, W, b = _mk_layer(ops, N, K, dev, k_layout=k_layout)
    lda = ops.ceil_div(K, 64) * 64 + 8
    A = torch.randn(M + 5, lda, device=dev)
    out = torch.full((M + 5, 264), -7.0, device=dev)
    ops.linear(ops.Mat(A), L, ops.Mat(out, 4), N, act=act, act_param=0.0, m_cap=M)
    torch.cuda.synchronize()
    acc = A[:M, :K].double() @ W.t() + b
    want = act_ref(acc, act, 0.0)
    scale = A[:M, :K].double().abs() @ W.abs().t() + b.abs()
    rel, ab = _err(out[:M, 4:4 + N], want, scale)
    print(f'linear M={M} K={K} N={N} act={act}: rel {rel:.2e} abs {ab:.2e}')
    assert rel < 2e-5
    assert float(out[M:, :].min()) == -7.0 and float(out[:, :4].max()) == -7.0 and float(out[:, 4 + N:].max()) == -7.0


def test_linear_kmap_and_device_count():
    from nero_b200 import ops
    dev = torch.device('cuda')
    K, N, k_layout = 259, 256, 264
    kmap = list(range(4, 260)) + [0, 1, 2]          # reference [feat(256), x(3)] -> layout [x(3), pad, feat...]
    L, W, b = _mk_layer(ops, N, K, dev, kmap=kmap, k_layout=k_layout)
    A = torch.randn(3000, 320, device=dev)
    out = torch.zeros(3000, 256, device=dev)
    mcount = torch.tensor([1234], dtype=torch.int32, device=dev)
    ops.linear(ops.Mat(A), L, ops.Mat(out), N, act=2, m_ptr=mcount, m_cap=3000)
    torch.cuda.synchronize()
    Ar = A[:1234][:, kmap].double()
    want = torch.relu(Ar @ W.t() + b)
    rel, ab = _err(out[:1234], want, Ar.abs() @ W.abs().t() + 1)
    print(f'kmap: rel {rel:.2e}')
    assert rel < 2e-5 and float(out[1234:].abs().max()) == 0.0


def test_linear_transposed_modes():
    from nero_b200 import ops
    dev = torch.device('cuda')
    M, K, N = 2100, 256, 217
    L, W, b = _mk_layer(ops, N, K, dev, t_cols=(0, 256))
    dY = torch.randn(M, 224, device=dev)
    H = torch.rand(M, 256, device=dev) * 0.05
    V = torch.randn(M, 256, device=dev)
    add = torch.randn(M, 256, device=dev)
    out = torch.zeros(M, 256, device=dev)
    out2 = torch.zeros(M, 256, device=dev)
    tail = torch.zeros(M, 64, device=dev)
    acc = dY[:, :N].double() @ W            # [M, 256]
    s = dact_ref(H.double() * 1.4142135, 1)
    scale = dY[:, :N].double().abs() @ W.abs()
    # MUL_DACT with addend, tail split at 217
    ops.linear(ops.Mat(dY), L, ops.Mat(out), 256, transposed=True, mode=ops.EPI_MUL_DACT, oscale=0.70710678, H=ops.Mat(H),
               hscale=1.4142135, dact=1, addend=ops.Mat(add), ncol_main=217, tail=ops.Mat(tail))
    torch.cuda.synchronize()
    want = 0.70710678 * s[:, :217] * acc[:, :217] + add[:, :217].double()
    rel, _ = _err(out[:, :217], want, scale[:, :217] + 1)
    relt, _ = _err(tail[:, :39], 0.70710678 * acc[:, 217:], scale[:, 217:] + 1e-3)
    print(f'mul_dact rel {rel:.2e} tail {relt:.2e}')
    assert rel < 2e-5 and relt < 2e-5
    # TANGENT
    ops.linear(ops.Mat(dY), L, ops.Mat(out), 256, transposed=True, mode=ops.EPI_TANGENT, H=ops.Mat(H), hscale=1.0, dact=1,
               V=ops.Mat(V), out2=ops.Mat(out2))
    torch.cuda.synchronize()
    s1 = dact_ref(H.double(), 1)
    rel1, _ = _err(out, s1 * acc, scale + 1e-3)
    rel2, _ = _err(out2, 100 * (1 - s1) * V.double() * acc, 100 * V.double().abs() * scale + 1e-3)
    print(f'tangent rel {rel1:.2e} {rel2:.2e}')
    assert rel1 < 2e-5 and rel2 < 2e-5


@pytest.mark.parametrize('M,N,K,two', [(5000, 256, 256, False), (70001, 256, 256, True), (3000, 217, 256, False),
                                       (999, 3, 259, False), (20000, 128, 283, False), (4000, 256, 39, True)])
def test_wgrad(M, N, K, two):
    from nero_b200 import ops
    dev = torch.device('cuda')
    L, W, b = _mk_layer(ops, N, K, dev)
    ws = ops.WgradWorkspace(dev)
    dY = torch.randn(M, 256 + 8, device=dev) * 0.1
    X = torch.randn(M, 320, device=dev)
    dY2 = torch.randn(M, 256, device=dev) * 0.1 if two else None
    X2 = torch.randn(M, 320, device=dev) if two else None
    gw, gg, gb = torch.zeros_like(L.weight), torch.zeros_like(L.g), torch.zeros(N, device=dev)
    ops.wgrad(ws, ops.Mat(dY, 4), N, ops.Mat(X), L.k_valid, L, gw, gg, gb, ops.Mat(dY2) if two else None,
              ops.Mat(X2) if two else None)
    torch.cuda.synchronize()
    # reference through autograd of weight norm in fp64
    v = L.weight.double().requires_grad_(True)
    g = L.g.double().requires_grad_(True)
    Wd = g * v / v.norm(dim=1, keepdim=True)
    dW = dY[:, 4:4 + N].double().t() @ X[:, :K].double()
    if two:
        dW = dW + dY2[:, :N].double().t() @ X2[:, :K].double()
    (Wd * dW).sum().backward()
    sc = float(dW.abs().max())
    e_v = float((gw.double() - v.grad).abs().max()) / sc
    e_g = float((gg.double() - g.grad).abs().max()) / sc
    e_b = float((gb.double() - dY[:, 4:4 + N].double().sum(0)).abs().max()) / (float(dY.abs().sum(0).max()))
    print(f'wgrad M={M} N={N} K={K}: v {e_v:.2e} g {e_g:.2e} b {e_b:.2e}')
    assert e_v < 3e-5 and e_g < 3e-5 and e_b < 1e-5


def test_wgrad_device_row_count_masks_stale_rows():
    """Rows >= the device-side count hold stale data (here NaN / inf): the producers must zero them while converting."""
    from nero_b200 import ops
    dev = torch.device('cuda')
    M, cap, N, K = 12345, 20000, 256, 256
    L, W, b = _mk_layer(ops, N, K, dev)
    ws = ops.WgradWorkspace(dev)
    dY = torch.randn(cap, 256, device=dev) * 0.1
    X = torch.randn(cap, 256, device=dev)
    dY[M:] = float('nan')
    X[M:] = float('inf')
    m_ptr = torch.tensor([M], dtype=torch.int32, device=dev)
    gw, gg, gb = torch.zeros_like(L.weight), torch.zeros_like(L.g), torch.zeros(N, device=dev)
    ops.wgrad(ws, ops.Mat(dY), N, ops.Mat(X), L.k_valid, L, gw, gg, gb, m_ptr=m_ptr, m_cap=cap)
    torch.cuda.synchronize()
    v = L.weight.double().requires_grad_(True)
    g = L.g.double().requires_grad_(True)
    dW = dY[:M].double().t() @ X[:M].double()
    ((g * v / v.norm(dim=1, keepdim=True)) * dW).sum().backward()
    sc = float(dW.abs().max())
    assert torch.isfinite(gw).all() and torch.isfinite(gb).all()
    assert float((gw.double() - v.grad).abs().max()) / sc < 3e-5
    assert float((gb.double() - dY[:M].double().sum(0)).abs().max()) / float(dY[:M].abs().sum(0).max()) < 1e-5


@pytest.mark.parametrize('M', [3000, 45001])
def test_chain_matches_layerwise_and_fp64(M):
    """Fused chain (A operand in shared memory) and its one-nero_linear-per-layer expansion (ops.mlp) vs fp64 torch:
    3 softplus layers with the skip-concat, then a linear head; then a derivative (DACT) chain in the reverse direction with
    addend / tail.  M = 45001 is 352 row tiles: every one of the 132 persistent CTAs loops over at least two tiles (mbarrier
    phases across tiles) and the last tile is ragged."""
    from nero_b200 import ops
    from nero_b200.ops import Mat, mlp, chain_layer as CL
    dev = torch.device('cuda')
    L0, W0, b0 = _mk_layer(ops, 256, 39, dev, seed=1, t_cols=(0, 39))
    L1, W1, b1 = _mk_layer(ops, 217, 256, dev, seed=2, t_cols=(0, 256))
    L2, W2, b2 = _mk_layer(ops, 256, 256, dev, seed=3, t_cols=(0, 256))
    L3, W3, b3 = _mk_layer(ops, 3, 256, dev, seed=4, t_cols=(0, 256))
    X = torch.zeros(M, 64, device=dev)
    X[:, :39] = torch.randn(M, 39, device=dev) * 0.5
    H1, H2, H3 = torch.zeros(M, 256, device=dev), torch.zeros(M, 256, device=dev), torch.zeros(M, 256, device=dev)
    out = torch.zeros(M, 32, device=dev)
    sp = lambda x: torch.nn.functional.softplus(x, beta=100)
    h1 = sp(X[:, :39].double() @ W0.t() + b0)
    h2 = torch.cat([0.70710678 * sp(h1 @ W1.t() + b1), X[:, :39].double() * 0.5], -1)
    h3 = sp(h2 @ W2.t() + b2)
    o = torch.sigmoid(h3 @ W3.t() + b3)
    for fused in (True, False):
        for t in (H1, H2, H3, out):
            t.zero_()
        H2[:, 217:] = X[:, :39] * 0.5                 # concat source pre-filled in the save buffer
        mlp(Mat(X), [CL(L0, ops.EK_BIAS_SOFTPLUS, 256, save=Mat(H1)),
                     CL(L1, ops.EK_BIAS_SOFTPLUS, 217, oscale=0.70710678, save=Mat(H2), csrc=Mat(H2)),
                     CL(L2, ops.EK_BIAS_SOFTPLUS, 256, save=Mat(H3)),
                     CL(L3, ops.EK_BIAS_GENERIC, 3, act=3, save=Mat(out, 8), write_a=False)], fused=fused)
        torch.cuda.synchronize()
        for nm, got, want in [('h1', H1, h1), ('h2', H2, h2), ('h3', H3, h3), ('out', out[:, 8:11], o)]:
            e = float((got.double() - want).abs().max())
            print(f'{"chain" if fused else "layerwise"} fwd {nm}: max abs err {e:.2e} (|want| max {float(want.abs().max()):.2e})')
            assert e < 3e-5 * max(1.0, float(want.abs().max()))
    # derivative chain: g2 = dact(H3) * (G @ W2) [217 main + tail], g1 = dact(H2*sqrt2)*... , g0 = g1 @ W0 (no dact)
    G = torch.randn(M, 256, device=dev)
    V2, V1, U0, TL = torch.zeros(M, 256, device=dev), torch.zeros(M, 256, device=dev), torch.zeros(M, 64, device=dev), torch.zeros(M, 64, device=dev)
    add = torch.randn(M, 256, device=dev)
    acc2 = G.double() @ W2
    s2 = dact_ref(H2.double()[:, :217] * 1.41421356, 1)
    g2 = 0.70710678 * s2 * acc2[:, :217]
    tl = 0.70710678 * acc2[:, 217:]
    g1 = dact_ref(H1.double(), 1) * (g2 @ W1) + add.double()
    g0 = g1 @ W0
    for fused in (True, False):
        for t in (V2, U0, TL):
            t.zero_()
        V1.copy_(add)
        mlp(Mat(G), [CL(L2, ops.EK_DACT_SOFTPLUS, 256, transposed=True, oscale=0.70710678, H=Mat(H2), hscale=1.41421356, ncol_main=217,
                        tail=Mat(TL), save=Mat(V2)),
                     CL(L1, ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H1), addend=Mat(V1), save=Mat(V1)),
                     CL(L0, ops.EK_DACT_NONE, 39, transposed=True, save=Mat(U0))], fused=fused)
        torch.cuda.synchronize()
        for nm, got, want in [('g2', V2[:, :217], g2), ('tail', TL[:, :39], tl), ('g1', V1, g1), ('g0', U0[:, :39], g0)]:
            e = float((got.double() - want).abs().max())
            print(f'{"chain" if fused else "layerwise"} dact {nm}: max abs err {e:.2e} (|want| max {float(want.abs().max()):.2e})')
            assert e < 3e-5 * max(1.0, float(want.abs().max()))


@pytest.mark.parametrize('M', [1500, 40007])
def test_tangent_chain_matches_fp64(M):
    """Tangent-sweep chain (EK_TANGENT: out = s*acc, out2 = 100*(1-s)*V*acc with s = sigma(100 a) recovered from the stored
    softplus output) over three layers incl. the skip-concat split, vs fp64 torch; M = 40007 gives every CTA >= 2 tiles."""
    from nero_b200 import ops
    from nero_b200.ops import Mat, chain, chain_layer as CL
    dev = torch.device('cuda')
    L0, W0, _ = _mk_layer(ops, 256, 39, dev, seed=11)
    L1, W1, _ = _mk_layer(ops, 217, 256, dev, seed=12)
    L2, W2, _ = _mk_layer(ops, 256, 256, dev, seed=13)
    g = torch.Generator().manual_seed(M)
    U0 = torch.zeros(M, 64, device=dev)
    U0[:, :39] = torch.randn(M, 39, generator=g).to(dev)
    H = [(torch.rand(M, 256, generator=g) * 0.04).to(dev) for _ in range(3)]
    V = [torch.randn(M, 256, generator=g).to(dev) for _ in range(3)]
    UB = [torch.zeros(M, 256, device=dev) for _ in range(3)]
    AB = [torch.zeros(M, 256, device=dev) for _ in range(3)]
    skip = torch.randn(M, 39, generator=g).to(dev)
    UB[1][:, 217:] = skip                                   # tangent of the PE/sqrt2 tail, pre-stored like pe_tangent does
    chain(Mat(U0), 40, [CL(L0, ops.EK_TANGENT, 256, use_bias=False, H=Mat(H[0]), V=Mat(V[0]), out2=Mat(AB[0]), save=Mat(UB[0])),
                        CL(L1, ops.EK_TANGENT, 217, use_bias=False, oscale=0.70710678, H=Mat(H[1]), hscale=1.41421356, V=Mat(V[1]),
                           out2=Mat(AB[1]), save=Mat(UB[1]), csrc=Mat(UB[1])),
                        CL(L2, ops.EK_TANGENT, 256, use_bias=False, H=Mat(H[2]), V=Mat(V[2]), out2=Mat(AB[2]), save=Mat(UB[2]))])
    torch.cuda.synchronize()
    s0 = dact_ref(H[0].double(), 1)
    a0 = U0[:, :39].double() @ W0.t()
    u1 = s0 * a0
    q0 = 100 * (1 - s0) * V[0].double() * a0
    s1 = dact_ref(H[1].double()[:, :217] * 1.41421356, 1)
    a1 = u1 @ W1.t()
    u2 = torch.cat([0.70710678 * s1 * a1, skip.double()], -1)
    q1 = 100 * (1 - s1) * V[1].double()[:, :217] * a1
    s2 = dact_ref(H[2].double(), 1)
    a2 = u2 @ W2.t()
    u3 = s2 * a2
    q2 = 100 * (1 - s2) * V[2].double() * a2
    for nm, got, want in [('u1', UB[0], u1), ('q0', AB[0], q0), ('u2', UB[1], u2), ('q1', AB[1][:, :217], q1), ('u3', UB[2], u3), ('q2', AB[2], q2)]:
        e = float((got.double() - want).abs().max())
        sc = max(1.0, float(want.abs().max()))
        print(f'tangent chain {nm} (M={M}): max abs err {e:.2e} (|want| max {sc:.2e})')
        assert e < 3e-5 * sc, nm


def test_flat_adam_matches_torch_adam():
    """nero_adam_flat over the flat parameter buffer vs torch.optim.Adam on the same gradients (train/trainer.py:73-76)."""
    import nero_oracle as O
    from helpers import build_params
    from nero_b200.renderer import NeROShapeRenderer
    from nero_b200.optim import FlatAdam
    cfg = {'n_samples': 32, 'n_importance': 32}
    net = NeROShapeRenderer(cfg, training=False)
    net.load_state_dict(build_params(cfg))
    net = net.cuda()
    ref = [p.detach().clone().requires_grad_(True) for p in net.parameters()]
    opt_ref = torch.optim.Adam(ref, lr=5e-4)
    opt = FlatAdam(net, lr=5e-4)
    r = {k: v.cuda() for k, v in O.synthetic_rays(32, seed=6033).items()}
    for it in range(3):
        opt.zero_grad()
        out = net.render(r['rays_o'], r['rays_d'], r['near'], r['far'], r['human_poses'], 0, 1.0, True, 30000)
        (torch.mean(net.compute_rgb_loss(out['ray_rgb'], r['rgb'])) + torch.mean(out['gradient_error'] * 0.1)).backward()
        for q, p in zip(ref, net.parameters()):
            q.grad = p.grad.detach().clone()
        opt.param_groups[0]['lr'] = opt_ref.param_groups[0]['lr'] = 5e-4 * (it + 1)      # the trainer sets the lr every step
        opt.step()
        opt_ref.step()
        for q, p in zip(ref, net.parameters()):
            assert float((q - p).abs().max()) <= 1e-6 * float(q.abs().max()) + 1e-9
    sd = opt.state_dict()
    assert len(sd['state']) == len(ref) and int(float(sd['state'][0]['step'])) == 3
    fresh = torch.optim.Adam([q.detach().clone().requires_grad_(True) for q in ref], lr=1e-3)
    fresh.load_state_dict(sd)                                   # interchangeable with torch's optimizer checkpoints
    opt2 = FlatAdam(net, lr=1e-3)
    opt2.load_state_dict(opt_ref.state_dict())
    assert opt2.t == 3 and float((opt2.exp_avg - opt.exp_avg).abs().max()) <= 1e-7
