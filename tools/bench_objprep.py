"""Custom-object preparation on one H100: crop, plane hypotheses and inlier counts, refit, voxel components and compaction.

    python tools/bench_objprep.py [--points 5000000] [--hypotheses 1024] [--repeats 5] [--out DIR]

Workload: the synthetic scene of oracle/nero_oracle_objprep.scene (tilted table, box-and-sphere object, 10 % uniform
outliers) with --points points, uploaded once, cropped to the default sphere (CROP_FRAC of the camera distance around the
object centre).  Stages, each the median over the repeats between CUDA events after a warm call:
  crop        crop kernel + ordered compaction of the kept points (including the read of their count)
  counts      hypotheses + the H x m point-plane inlier counts (the hot loop; m = kept points)
  refit       two least-squares refit rounds (four fixed-order moment passes, host eigen-solves)
  components  height test and voxel keys, key sort and unique (torch), voxel union-find, component selection, point flags
  compaction  ordered compaction of the object's points
The counts are reported as point-plane tests per second against the fp64 roof of the card: SMs x 64 fp64 lanes x the max
SM clock, divided by the 7 fp64 instructions of one uncontracted test (3 DMUL, 3 DADD, 1 DSETP).  Prints one JSON line
with the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'oracle')):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np
import torch

from bench_mesh import card, timed

FP64_PER_TEST = 7


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--points', type=int, default=5_000_000)
    ap.add_argument('--hypotheses', type=int, default=1024)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--out', type=str, default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_objprep: needs a CUDA device')
    import nero_oracle_objprep as O
    from nero_b200 import objprep as OP, ops
    gpu = card()
    n = args.points
    sc = O.scene(n_table=int(n * 0.55) + 10, n_obj=int(n * 0.35) + 10, seed=0)
    p = torch.from_numpy(np.ascontiguousarray(sc['points'][:n])).cuda()
    D = 3.0                                                   # the scene's camera distance
    sphere = list(sc['center']) + [OP.CROP_FRAC * D]
    tol, voxel = OP.TOL_FRAC * D, OP.VOXEL_FRAC * D
    above = OP.ABOVE_TOLS * tol
    H = args.hypotheses
    res = {}

    def crop():
        res['keep'], _, res['kept'] = OP.crop_points(p, sphere)
    t_crop = timed(crop, args.repeats)
    keep, kept = res['keep'], res['kept']
    m = kept.shape[0]
    planes = torch.empty(H, 4, dtype=torch.float64, device='cuda')
    sample = torch.empty(H, 3, dtype=torch.int32, device='cuda')
    valid = torch.empty(H, dtype=torch.uint8, device='cuda')
    counts = torch.empty(H, dtype=torch.int64, device='cuda')

    def hyp_counts():
        ops.K('nero_objprep_hypotheses', kept, m, H, 0, planes, sample, valid)
        ops.K('nero_objprep_counts', kept, m, planes, H, tol, counts)
    t_counts = timed(hyp_counts, args.repeats)
    plane0 = planes[int(torch.argmax(counts))].cpu().numpy()

    def refit():
        pl = plane0
        for _ in range(2):
            pl = OP.refit(kept, pl, tol)[0]
        res['plane'] = pl
    t_refit = timed(refit, args.repeats)
    plane = res['plane'] if res['plane'][:3] @ sc['up'] > 0 else -res['plane']
    origin = np.ascontiguousarray(kept.amin(0).cpu().numpy())

    def components():
        flag = torch.empty(n, dtype=torch.uint8, device='cuda')
        keys = torch.empty(n, dtype=torch.int64, device='cuda')
        ops.K('nero_objprep_above', p, n, keep, plane, above, origin, voxel, flag, keys)
        ukeys, vcount = torch.unique_consecutive(torch.sort(keys)[0], return_counts=True)
        ukeys, vcount = ukeys[:-1].contiguous(), vcount[:-1].contiguous()      # the last key is the unflagged sentinel
        nv = ukeys.shape[0]
        parent = torch.empty(nv, dtype=torch.int32, device='cuda')
        label = torch.empty(nv, dtype=torch.int32, device='cuda')
        ops.K('nero_objprep_voxel_components', ukeys, nv, parent, label)
        cc = torch.empty(nv, dtype=torch.int64, device='cuda')
        vk = torch.empty(nv, dtype=torch.uint8, device='cuda')
        ops.K('nero_objprep_component_select', label, vcount, nv, 1.0, cc, vk)
        pk = torch.empty(n, dtype=torch.uint8, device='cuda')
        ops.K('nero_objprep_point_keep', keys, flag, n, ukeys, nv, vk, pk)
        res['pk'], res['voxels'] = pk, nv
    t_comp = timed(components, args.repeats)
    t_compact = timed(lambda: res.__setitem__('obj', OP._compact(p, res['pk'], True)), args.repeats)
    _, iinfo = OP.isolate_object(p, plane, above, voxel, sphere, None, 1.0)
    same = bool(torch.equal(iinfo['index'], res['obj'][0]))

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    mhz = re.search(r'(\d+) MHz', gpu)
    roof = sms * 64 * float(mhz.group(1)) * 1e6 / FP64_PER_TEST if mhz else None
    tests = float(H) * m
    ms = lambda x: round(x * 1e3, 3)
    line = {'metric': 'objprep', 'gpu': gpu, 'points': n, 'kept': m, 'hypotheses': H, 'voxels': res['voxels'],
            'object_points': int(res['obj'][0].shape[0]), 'crop_ms': ms(t_crop), 'counts_ms': ms(t_counts), 'refit_ms': ms(t_refit),
            'components_ms': ms(t_comp), 'compaction_ms': ms(t_compact), 'tests_per_s': tests / t_counts,
            'fp64_roof_tests_per_s': roof, 'fraction_of_roof': (tests / t_counts / roof) if roof else None,
            'isolate_equal_stages': same}
    print(json.dumps(line), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, 'bench_objprep.json'), 'w') as f:
            json.dump(line, f, indent=1)


if __name__ == '__main__':
    main()
