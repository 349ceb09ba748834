"""Distances from points to a triangle mesh on the GPU (k_meshdist.cu, include/nero_meshdist.h), and the reconstruction
metrics built on them: accuracy, completeness, Chamfer, Hausdorff and F-score between two meshes.

The reference's Chamfer distance (evaluate.nearest_dist_cuda) measures point set against point set, so it cannot go below
the spacing of the samples.  Here one side is a surface: the distance of a sample to the other mesh is exact up to
rounding, whatever the sample count.

Convention
----------
  * Queries are float64 points [n,3] (what evaluate.sample_surface returns); the mesh is verts [V,3] float32 and tris [T,3]
    int32, each vertex converted exactly to float64.
  * The distance to a triangle is Ericson's Voronoi-region closest point (Real-Time Collision Detection, 5.1.5), every
    float64 operation correctly rounded and never fused, so oracle/nero_oracle_meshdist.py reproduces every bit.  A
    triangle with cross(b - a, c - a) = 0 (zero-length edges, collinear or repeated vertices: marching cubes emits such
    triangles where grid values sit on the isovalue), or whose region denominators vanish, is taken as its three edge
    segments.  No finite input gives NaN.  include/nero_meshdist.h states every operation.
  * Result per query: dist = sqrt of the least squared distance over the triangles, tri = the original index of the
    minimising triangle (ties to the lowest index, so the result depends neither on the BVH nor on the traversal), and
    optionally the closest point.  With max_dist, a query with no triangle within it gets dist = +inf, tri = -1 and a NaN
    point.
  * The search is a one-thread-per-query traversal of the BVH that nero_bvh_build_host builds (ops.bvh_build).  A node is
    skipped only when no triangle under it can produce a computed distance <= the current best: the box bound uses directed
    rounding plus margins larger than the routine's rounding error, so the result equals brute force bit for bit.

Metrics (compare, metrics)
--------------------------
  * accuracy: distances of `samples` area-uniform samples of the predicted mesh (sample_surface, seed s) to the reference
    surface; completeness: samples of the reference (seed s + 1) to the predicted surface.  Each is summarised by mean,
    median, RMS, p90, p95, p99 (numpy's default percentile definition) and max, in float64 on the host.
  * chamfer = (accuracy.mean + completeness.mean) / 2: the reference's convention (eval_synthetic_shape.py:95), with
    point-to-surface distances.
  * hausdorff = max(accuracy.max, completeness.max).  It is an estimate from the samples, so it is a lower bound of the
    true Hausdorff distance.
  * Per threshold t: precision = the share of accuracy distances < t, recall = that of completeness distances, fscore =
    2 P R / (P + R), 0 when both are 0 (Tanks and Temples).
THRESHOLDS are choices, not tuned values: 1, 2 and 5 thousandths of the unit sphere's radius the objects are fitted into.

Error map (error_colors, mesh.write_ply): the colour of distance d at threshold t is floor(255 (s, 0, 1 - s) + 0.5) with s =
min(d / t, 1): blue on the surface, red at t and beyond.  The distance itself goes to the PLY's per-vertex `quality`.
"""
import numpy as np

THRESHOLDS = (0.001, 0.002, 0.005)
PERCENTILES = (90, 95, 99)


class MeshDistance:
    """A triangle mesh resident on the GPU with its BVH, so that several query sets reuse one host build.  verts [V,3] /
    tris [T,3] as numpy arrays or tensors, checked by evaluate._mesh_cuda."""

    def __init__(self, verts, tris):
        from . import ops
        from .evaluate import _mesh_cuda
        self.verts, self.tris = _mesh_cuda(verts, tris, 'MeshDistance')
        self.nodes, _, self.tri_ids = ops.bvh_cuda(self.verts, self.tris)

    def query(self, points, max_dist=float('inf'), closest=False):
        """Distances of points [n,3] (numpy or tensor, converted to float64) to the mesh -> (dist CUDA float64 [n], tri CUDA
        int32 [n]) or, with closest=True, (dist, tri, point CUDA float64 [n,3]).  Reads one status word back."""
        import torch
        from . import ops
        max_dist = float(max_dist)
        if not max_dist >= 0.0:
            raise ValueError(f'max_dist must be >= 0 (or inf), got {max_dist}')
        dev = self.verts.device
        p = torch.as_tensor(points).detach().to(dev, torch.float64)
        if p.ndim != 2 or p.shape[1] != 3:
            raise ValueError(f'query points must be [n,3], got {tuple(p.shape)}')
        if not bool(torch.isfinite(p).all()):
            raise ValueError('query points must be finite')
        p = p.contiguous()
        n = p.shape[0]
        dist = torch.empty(n, dtype=torch.float64, device=dev)
        tri = torch.empty(n, dtype=torch.int32, device=dev)
        point = torch.empty(n, 3, dtype=torch.float64, device=dev) if closest else None
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            ops.K('nero_meshdist_query', p, n, self.nodes, self.tri_ids, self.verts, self.tris, max_dist, dist, tri, point, status,
                  launches=int(n > 0))
        if int(status.item()) != 0:
            raise RuntimeError('nero_meshdist_query: a traversal overran its stack (the BVH is deeper than the kernel supports)')
        return (dist, tri, point) if closest else (dist, tri)


def _summary(d):
    s = {'mean': float(np.mean(d)), 'median': float(np.median(d)), 'rms': float(np.sqrt(np.mean(d * d)))}
    for q, v in zip(PERCENTILES, np.percentile(d, PERCENTILES)):
        s[f'p{q}'] = float(v)
    s['max'] = float(np.max(d))
    return s


def metrics(accuracy, completeness, thresholds=THRESHOLDS):
    """Every metric of the module docstring from the two distance arrays (numpy or tensors, non-empty) -> dict with
    accuracy / completeness summaries, chamfer, hausdorff and per threshold {threshold, precision, recall, fscore}."""
    acc = np.asarray(accuracy.cpu() if hasattr(accuracy, 'cpu') else accuracy, np.float64).reshape(-1)
    comp = np.asarray(completeness.cpu() if hasattr(completeness, 'cpu') else completeness, np.float64).reshape(-1)
    if acc.size == 0 or comp.size == 0:
        raise ValueError('metrics need non-empty distance arrays')
    a, c = _summary(acc), _summary(comp)
    per = []
    for t in thresholds:
        t = float(t)
        if not (np.isfinite(t) and t > 0):
            raise ValueError(f'thresholds must be positive and finite, got {t}')
        pr, rc = float(np.count_nonzero(acc < t)) / acc.size, float(np.count_nonzero(comp < t)) / comp.size
        per.append({'threshold': t, 'precision': pr, 'recall': rc, 'fscore': 2 * pr * rc / (pr + rc) if pr + rc > 0 else 0.0})
    return {'accuracy': a, 'completeness': c, 'chamfer': (a['mean'] + c['mean']) / 2, 'hausdorff': max(a['max'], c['max']),
            'thresholds': per}


def compare_index(pr, gt, samples=1_000_000, seed=0, thresholds=THRESHOLDS):
    """compare() on meshes already resident as MeshDistance objects (pr: the predicted mesh, gt: the reference)."""
    from .evaluate import sample_surface
    if not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 32 - 1:
        raise ValueError(f'seed must be an integer in [0, 2^32 - 1), got {seed}')
    acc = gt.query(sample_surface(pr.verts, pr.tris, samples, seed))[0]
    comp = pr.query(sample_surface(gt.verts, gt.tris, samples, seed + 1))[0]
    out = metrics(acc, comp, thresholds)
    out['samples'], out['seed'] = int(samples), int(seed)
    return out


def compare(pr_verts, pr_tris, gt_verts, gt_tris, samples=1_000_000, seed=0, thresholds=THRESHOLDS):
    """Accuracy, completeness, Chamfer, Hausdorff and F-score of the predicted mesh against the reference mesh (module
    docstring) -> the dict of metrics(), plus samples and seed."""
    return compare_index(MeshDistance(pr_verts, pr_tris), MeshDistance(gt_verts, gt_tris), samples, seed, thresholds)


def error_colors(dist, threshold):
    """uint8 [n,3] RGB of distances [n] at a threshold: floor(255 (s, 0, 1 - s) + 0.5), s = min(d / threshold, 1)."""
    t = float(threshold)
    if not (np.isfinite(t) and t > 0):
        raise ValueError(f'threshold must be positive and finite, got {t}')
    d = np.asarray(dist.cpu() if hasattr(dist, 'cpu') else dist, np.float64).reshape(-1)
    s = np.minimum(d / t, 1.0)
    out = np.zeros((d.size, 3), np.uint8)
    out[:, 0] = np.floor(255.0 * s + 0.5)
    out[:, 2] = np.floor(255.0 * (1.0 - s) + 0.5)
    return out
