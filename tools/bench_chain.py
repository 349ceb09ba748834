"""Developer micro-benchmark of the fused MLP-chain kernel alone (run on the GPU box): 8 fused 256-wide layers over M rows
in the four shapes the training step uses -- forward without saves (sampling), forward with saved activations, the
derivative sweep (H in, V out per layer) and the tangent sweep (H, V in; two outputs) -- and three variants of the
derivative sweep that locate the cost of its H operand (see the comments at the cases).  Prints microseconds per launch,
the algorithmic TFLOP/s (2*M*K*N per layer) and the time of one layer on one 128-row tile in one CTA."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests')); sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import numpy as np, torch
from nero_b200 import ops
from nero_b200.ops import Mat, chain, chain_layer as CL
from test_gemm_gpu import _mk_layer
dev = torch.device('cuda')
M = int(os.environ.get('ROWS', 127232))
NL = int(os.environ.get('LAYERS', 8))
reps = int(os.environ.get('REPS', 10))
only = os.environ.get('ONLY', '')
Ls = [_mk_layer(ops, 256, 256, dev, seed=10 + i, t_cols=(0, 256))[0] for i in range(NL)]
X = torch.randn(M, 256, device=dev) * 0.3
H = [torch.rand(M, 256, device=dev) * 0.05 for _ in range(NL)]
V = [torch.randn(M, 256, device=dev) for _ in range(NL)]
HP = [torch.nn.functional.pad(h, (0, 8)) for h in H]     # H with a 264-float row stride
O1 = [torch.zeros(M, 256, device=dev) for _ in range(NL)]
O2 = [torch.zeros(M, 256, device=dev) for _ in range(NL)]
cases = {
    'forward_nosave': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_BIAS_SOFTPLUS, 256) for i in range(NL)]),
    'forward_save': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_BIAS_SOFTPLUS, 256, save=Mat(O1[i])) for i in range(NL)]),
    'relu_save': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_BIAS_RELU, 256, save=Mat(O1[i])) for i in range(NL)]),
    'reverse': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[i]), save=Mat(O1[i])) for i in range(NL)]),
    # `reverse` with every layer reading H[0]: at one tile per CTA (ROWS=16896) H[0] stays in L2 after the first layer, so
    # the gap to `reverse` is the most that fetching the epilogue operands from HBM costs the sweep
    'reverse_l2hot': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[0]), save=Mat(O1[i])) for i in range(NL)]),
    # `reverse` reading H through rows 1056 B apart instead of 1024 B: whether the row stride concentrates the epilogue's
    # loads on a few L2 slices
    'reverse_ld264': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(HP[i], 0, 256), save=Mat(O1[i])) for i in range(NL)]),
    # `reverse` without the H operand (and without the softplus derivative): what the sweep costs when its epilogue loads
    # nothing
    'reverse_noh': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_NONE, 256, transposed=True, save=Mat(O1[i])) for i in range(NL)]),
    'reverse_addend': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_DACT_SOFTPLUS, 256, transposed=True, H=Mat(H[i]), addend=Mat(V[i]), save=Mat(O1[i])) for i in range(NL)]),
    'tangent': lambda: chain(Mat(X), 256, [CL(Ls[i], ops.EK_TANGENT, 256, use_bias=False, H=Mat(H[i]), V=Mat(V[i]), out2=Mat(O2[i]), save=Mat(O1[i])) for i in range(NL)]),
}
res = {}
for name, fn in cases.items():
    if only and name not in only.split(','):
        continue
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    res[name] = {'us': round(us, 1), 'tflops': round(2.0 * M * 256 * 256 * NL / us / 1e6, 1), 'us_per_layer_tile': round(us / NL / max(1.0, np.ceil(M / 128) / 132), 2)}
print(json.dumps({'rows': M, 'layers': NL, 'lib': os.environ.get('NERO_LIB', 'default'), **res}))
