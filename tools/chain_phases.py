"""Developer tool (run on the GPU box): where the time of a fused-chain layer-tile goes.

Loads the diagnostic library built with NERO_CHAIN_PHASES (nero_b200/build.py: build_phases), in which thread 0 of each
warpgroup of `gemm_chain_kernel` adds the SM cycles of five phases of every layer to device counters:
  a0    the first A operand's load and split (layer 0 of a tile only)
  wait  from the start of the layer until its first weight stage has landed
  mma   from there until the layer's last MMA has completed
  epi   the epilogue, from the last MMA's completion to the end of the next-A writes (including the barrier before it)
  bar   the closing barrier of the layer
Each CTA's cycles and %globaltimer nanoseconds convert cycles to time.  Prints, per case, microseconds per layer-tile (the
mean of a warpgroup's time over the layers and tiles of the launch) for each phase.

Cases: the tools/bench_chain.py launches (8 fused 256-wide layers over ROWS rows; each runs once after a warm-up), then
every chain launch of one resident bell training step (bench.py's workload), summed per family and per tag.

    python tools/chain_phases.py [--no-step] [--rows N] [--out FILE.json]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
from nero_b200 import build as B

if 'NERO_LIB' not in os.environ:
    os.environ['NERO_LIB'] = B.build_phases()
import numpy as np
import torch

from nero_b200 import ops

PHASES = ('a0', 'wait', 'mma', 'epi', 'bar')
N_SM, N_LAYERS_MAX = 132, 10           # kNumSMs, kMaxChainLayers (k_gemm_chain.cu)
N_CNT = N_SM * 2 * N_LAYERS_MAX * len(PHASES)
FAMILY = {0: 'forward', 1: 'forward', 2: 'forward', 3: 'gradient', 4: 'gradient', 5: 'gradient', 6: 'tangent'}


def counters(dev):
    return torch.zeros(N_CNT + 2 * N_SM, dtype=torch.int64, device=dev)


def decode(buf, rows, n_layers):
    """-> ({phase: cycles summed over CTAs, warpgroups and layers}, ns per cycle, layer-tiles per warpgroup)."""
    c = buf.cpu().numpy().astype(np.float64)
    ph = c[:N_CNT].reshape(N_SM, 2, N_LAYERS_MAX, len(PHASES))
    cta = c[N_CNT:].reshape(N_SM, 2)
    assert cta[:, 0].sum() > 0, 'no phase counters written: the library was not built with NERO_CHAIN_PHASES'
    tiles = -(-rows // 128)
    return {p: ph[:, :, :, i].sum() for i, p in enumerate(PHASES)}, cta[:, 1].sum() / cta[:, 0].sum(), 2 * tiles * n_layers


def us_per_layer_tile(acc):
    cyc, ns_per_cyc, lt = acc
    return {p: round(cyc[p] * ns_per_cyc / lt / 1e3, 2) for p in PHASES} | {
        'sum': round(sum(cyc.values()) * ns_per_cyc / lt / 1e3, 2)}


def bench_chain_cases(dev, M, NL=8):
    from nero_b200.ops import Mat, chain, chain_layer as CL
    from test_gemm_gpu import _mk_layer
    Ls = [_mk_layer(ops, 256, 256, dev, seed=10 + i, t_cols=(0, 256))[0] for i in range(NL)]
    X = torch.randn(M, 256, device=dev) * 0.3
    H = [torch.rand(M, 256, device=dev) * 0.05 for _ in range(NL)]
    V = [torch.randn(M, 256, device=dev) for _ in range(NL)]
    O1 = [torch.zeros(M, 256, device=dev) for _ in range(NL)]
    O2 = [torch.zeros(M, 256, device=dev) for _ in range(NL)]
    cases = {   # the same launches as tools/bench_chain.py
        'forward_nosave': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_BIAS_SOFTPLUS, 256) for i in range(NL)]),
        'forward_save': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_BIAS_SOFTPLUS, 256, save=Mat(O1[i])) for i in range(NL)]),
        'reverse': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[i]), save=Mat(O1[i]))
                                               for i in range(NL)]),
        'reverse_addend': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[i]), addend=Mat(V[i]),
                                                         save=Mat(O1[i])) for i in range(NL)]),
        'tangent': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_TANGENT, 256, use_bias=False, H=Mat(H[i]), V=Mat(V[i]), out2=Mat(O2[i]),
                                                  save=Mat(O1[i])) for i in range(NL)]),
    }
    res = {}
    for name, fn in cases.items():
        ops.CHAIN_PHASES = None
        fn()                                  # warm-up
        buf = counters(dev)
        ops.CHAIN_PHASES = buf
        fn()
        torch.cuda.synchronize()
        ops.CHAIN_PHASES = None
        res[name] = us_per_layer_tile(decode(buf, M, NL))
    return res


def bell_step(dev):
    import bench
    from nero_b200 import synthetic as O
    net, _ = bench.build_net({}, dev)
    r = {k: v.to(dev).contiguous() for k, v in O.synthetic_rays(1024, seed=6033).items()}
    car = net.get_anneal_val(bench.STEP)

    def step():
        net.zero_grad()
        z = net.sample_ray(r['rays_o'], r['rays_d'], r['near'], r['far'], 0)
        out = net.render_core(r['rays_o'], r['rays_d'], z, r['human_poses'], car, bench.STEP)
        bench.training_loss(net, out, r['rgb']).backward()
        torch.cuda.synchronize()
    step()                                    # warm-up
    launches = []
    orig = ops.chain

    def chain(A0, k_valid0, layers, m_ptr=None, m_cap=None, tag=''):
        buf = counters(dev)
        ops.CHAIN_PHASES = buf
        orig(A0, k_valid0, layers, m_ptr, m_cap, tag=tag)
        ops.CHAIN_PHASES = None
        launches.append((tag or '-', FAMILY[layers[0]['kind']], buf, m_ptr, A0.t.shape[0] if m_cap is None else m_cap, len(layers)))
    ops.chain = chain          # the engine's passes launch their chains through ops.mlp
    try:
        step()
    finally:
        ops.chain = orig
    by = {}
    for tag, fam, buf, m_ptr, m_cap, nl in launches:
        rows = min(int(m_ptr.item()), m_cap) if m_ptr is not None else m_cap
        if rows <= 0:
            continue
        cyc, ns_per_cyc, lt = decode(buf, rows, nl)
        for key in (f'family:{fam}', f'tag:{tag}'):
            a = by.setdefault(key, [dict.fromkeys(PHASES, 0.0), 0.0, 0, 0])
            for p in PHASES:
                a[0][p] += cyc[p] * ns_per_cyc
            a[2] += lt
            a[3] += 1
    out = {}
    for key, (ns, _, lt, n) in sorted(by.items()):
        out[key] = {p: round(ns[p] / lt / 1e3, 2) for p in PHASES} | {'sum': round(sum(ns.values()) / lt / 1e3, 2), 'launches': n}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--rows', type=int, default=127232)
    ap.add_argument('--no-step', action='store_true', help='only the tools/bench_chain.py cases')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda')
    res = {'gpu': torch.cuda.get_device_name(), 'lib': os.environ['NERO_LIB'], 'rows': args.rows, 'unit': 'us per layer-tile',
           'bench_chain': bench_chain_cases(dev, args.rows)}
    if not args.no_step:
        res['bell_step'] = bell_step(dev)
    txt = json.dumps(res, indent=1)
    print(txt)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(txt)


if __name__ == '__main__':
    main()
