"""Environment-light export on one H100: the stage-II outer light of the perturbed bell-like parameters as a 2048 x 1024 map at
ssaa 4 (33.6 M sub-sample rows) and at ssaa 1.

    python tools/bench_envmap.py [--width 2048] [--height 1024] [--repeats 3] [--sphere] [--out DIR]

Times the three stages over the whole map (CUDA events, median over warm repeats; each stage runs alone over every batch of
the default row cap): the row encoder (nero_env_rows), the outer-light chain and the texel resolve, and the whole export as
NeROMaterialRenderer.export_lighting runs it (the three interleaved per batch).  Reports rows per second and the chain's
algorithmic TFLOP/s (150 272 MAC per row, 168 704 with --sphere), with the card's name, power limit and maximum SM clock read
in the same run.  Prints one JSON line (and writes it to DIR/bench_envmap.json with --out).
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tools')):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch

from bench_mesh import card
from bench_texmap import timed

MAC_PER_ROW = {False: 72 * 256 + 2 * 256 * 256 + 256 * 3, True: 144 * 256 + 2 * 256 * 256 + 256 * 3}


def stages(ol, width, height, ssaa, repeats, center):
    """{stage: median ms} of the export of `ol` (an envmap.OuterLight) at this size."""
    from nero_b200 import envmap as EM, ops
    s2 = ssaa * ssaa
    n_tex = width * height
    per = min(EM.MAX_ROWS // s2, n_tex)
    ol.pred.prep()
    ol._alloc(per * s2)
    env = torch.empty(height, width, 3, device='cuda')
    batches = [(t0, min(per, n_tex - t0)) for t0 in range(0, n_tex, per)]

    def rows():
        for t0, nt in batches:
            ops.K('nero_env_rows', t0 * s2, nt * s2, width, height, ssaa, None, 0.0, ol.mode, *center, ol.ws['A'], ol.lda, None)

    def mlp():
        for _, nt in batches:
            ol._chain(nt * s2)

    def resolve():
        for t0, nt in batches:
            ops.K('nero_env_resolve', ol.ws['OUT'], 4, t0, nt, width, height, ssaa, env)
    out = {}
    for name, fn in (('rows', rows), ('chain', mlp), ('resolve', resolve)):
        out[name] = timed(fn, repeats)[0] * 1e3
    out['total'], m = timed(lambda: ol.map(width, height, ssaa, 0.0, center), repeats)
    out['total'] *= 1e3
    assert torch.isfinite(m).all()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--width', type=int, default=2048)
    ap.add_argument('--height', type=int, default=1024)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--sphere', action='store_true', help='a sphere_direction light seen from a point off the origin')
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_envmap: needs a CUDA device')
    from nero_b200 import params as P, synthetic
    from nero_b200 import envmap as EM
    gpu = card()
    scfg = {'human_lights': False, 'outer_light_version': 'sphere_direction' if args.sphere else 'direction'}
    sd = synthetic.perturb_params(P.build_material_state_dict(scfg, seed=6033))
    shader = P.MCShadingParams(scfg)
    shader.load_state_dict({k[len('shader_network.'):]: v for k, v in sd.items()})
    shader = shader.cuda()
    ol = EM.OuterLight(shader.outer_light, shader.cfg['light_exp_max'], 'stage2' if args.sphere else None)
    center = (0.1, -0.2, 0.15) if args.sphere else (0.0, 0.0, 0.0)
    line = {'metric': 'envmap_export', 'gpu': gpu, 'width': args.width, 'height': args.height, 'sphere': args.sphere,
            'max_rows': EM.MAX_ROWS}
    for ssaa in (4, 1):
        n = args.width * args.height * ssaa * ssaa
        t = stages(ol, args.width, args.height, ssaa, args.repeats, center)
        line[f'ssaa{ssaa}'] = {'rows': n, **{f'{k}_ms': round(v, 3) for k, v in t.items()},
                               'rows_per_s': round(n / (t['total'] * 1e-3), 0),
                               'chain_tflops': round(2.0 * MAC_PER_ROW[args.sphere] * n / (t['chain'] * 1e-3) / 1e12, 2)}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_envmap.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
