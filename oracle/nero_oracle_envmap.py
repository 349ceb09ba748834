"""CPU oracle of the environment-light export (nero_b200/envmap.py, k_envmap.cu) in numpy / torch CPU.

TEST INFRASTRUCTURE ONLY.  Sub-sample directions through nero_oracle_relight.env_dir (the inverse of relight's lookup), the
MLP input rows through nero_oracle.ide, the radiance through nero_oracle.predictor / nero_oracle_mat.outer_lights, the
cos(elevation)-weighted texel mean in float64 and the Radiance RGBE encoding.  Pinned against the unmodified reference by
tests/golden/envmap_*.npz (oracle/make_golden_envmap.py).
"""
import numpy as np
import torch
import torch.nn.functional as F

import nero_oracle as O
import nero_oracle_mat as OM
import nero_oracle_relight as ORl


def subsample_uv(width, height, ssaa):
    """(u, v) float64 [width * height * ssaa^2] in row order: texel t = y * width + x (row 0 at the top), sub-sample
    k = b * ssaa + a at u = (x + (a + 1/2) / ssaa) / width, v = (j + (b + 1/2) / ssaa) / height, j = height - 1 - y."""
    t = np.arange(width * height)
    y, x = t // width, t % width
    j = height - 1 - y
    k = np.arange(ssaa * ssaa)
    a, b = k % ssaa, k // ssaa
    u = (x[:, None] + (a[None] + 0.5) / ssaa) / width
    v = (j[:, None] + (b[None] + 0.5) / ssaa) / height
    return u.reshape(-1), v.reshape(-1)


def directions(width, height, ssaa, frame=None):
    """float32 [rows, 3]: env_dir in float64, rotated by `frame` (3x3, summed left to right, no fused multiply-add), rounded once."""
    d, _ = ORl.env_dir(*subsample_uv(width, height, ssaa))
    if frame is not None:
        Fm = np.asarray(frame, np.float64)
        d = np.stack([(Fm[i, 0] * d[:, 0] + Fm[i, 1] * d[:, 1]) + Fm[i, 2] * d[:, 2] for i in range(3)], -1)
    return d.astype(np.float32)


def sphere_points(d, sphere, center):
    """The second encoded point of a sphere_direction light for directions d [n,3] (torch float32) seen from `center`."""
    c = torch.as_tensor(np.asarray(center, np.float32)).expand(d.shape[0], 3)
    if sphere == 'stage2':         # network/field.py:843-850
        far = (torch.norm(c, dim=-1) > 0.999).unsqueeze(-1)
        p = torch.where(far, c * 0.999, c)
        return p + d * O.get_sphere_intersection(p, d)
    if sphere == 'stage1':         # network/field.py:559-561
        p = O.offset_points_to_sphere(c)
        return F.normalize(p + d * O.get_sphere_intersection(p, d), dim=-1)
    raise ValueError(sphere)


def rows(d, kappa_inv=0.0, sphere=None, center=(0.0, 0.0, 0.0)):
    """The outer-light input [n, 72 or 144] (torch float32) of directions d [n,3]."""
    d = torch.as_tensor(d)
    enc = O.ide(d, kappa_inv)
    if sphere is None:
        return enc
    return torch.cat([enc, O.ide(sphere_points(d, sphere, center), 0.0 if sphere == 'stage2' else kappa_inv)], -1)


def radiance(p, prefix, d, kappa_inv=0.0, sphere=None, center=(0.0, 0.0, 0.0), exp_max=0.0):
    """outer_light(rows(...)) -> float32 [n, 3] numpy.  Stage II goes through nero_oracle_mat.outer_lights."""
    d = torch.as_tensor(d)
    with torch.no_grad():
        if sphere == 'stage2' or (sphere is None and prefix.startswith('shader_network')):
            scfg = {'outer_light_version': 'sphere_direction' if sphere else 'direction', 'light_exp_max': exp_max}
            pts = torch.as_tensor(np.asarray(center, np.float32)).expand(d.shape[0], 3)
            out = OM.outer_lights(p, scfg, pts, d, prefix=prefix[:-len('.outer_light')])
        else:
            out = O.predictor(p, prefix, rows(d, kappa_inv, sphere, center), 'exp', exp_max)
    return out.float().numpy()


def weights(width, height, ssaa):
    """float64 [height * width, ssaa^2]: cos(elevation) of every sub-sample."""
    _, v = subsample_uv(width, height, ssaa)
    return np.cos((v - 0.5) * np.pi).reshape(width * height, ssaa * ssaa)


def resolve(rad, width, height, ssaa):
    """[rows, 3] sub-sample radiance -> float32 [height, width, 3], the weighted texel means in float64."""
    w = weights(width, height, ssaa)
    r = np.asarray(rad, np.float64).reshape(width * height, ssaa * ssaa, 3)
    return ((w[..., None] * r).sum(1) / w.sum(1)[:, None]).astype(np.float32).reshape(height, width, 3)


def envmap(p, prefix, width, height, ssaa, kappa_inv=0.0, sphere=None, center=(0.0, 0.0, 0.0), frame=None, exp_max=0.0):
    """The whole export: float32 [height, width, 3]."""
    d = directions(width, height, ssaa, frame)
    return resolve(radiance(p, prefix, torch.from_numpy(d), kappa_inv, sphere, center, exp_max), width, height, ssaa)


def fixture_params(g):
    """(state dict, MLP prefix, sphere mode) of a tests/golden/envmap_*.npz fixture, regenerated from its seeds."""
    from nero_b200 import params as P
    sph = bool(g['sphere'])
    if int(g['stage']) == 2:
        scfg = {'human_lights': False, 'outer_light_version': 'sphere_direction' if sph else 'direction'}
        sd = P.build_material_state_dict(scfg, seed=int(g['seed']))
        return O.perturb_params(sd, seed=int(g['pseed']), rel=float(g['rel'])), 'shader_network.outer_light', 'stage2' if sph else None
    sd = P.build_shape_state_dict({'shader_config': {'sphere_direction': sph}}, seed=int(g['seed']))
    return O.perturb_params(sd, seed=int(g['pseed']), rel=float(g['rel'])), 'color_network.outer_light', 'stage1' if sph else None


def rgbe(env):
    """[H,W,3] -> [H,W,4] uint8 RGBE, pixel by pixel with math.frexp (Greg Ward's float2rgbe)."""
    import math
    e = np.asarray(env, np.float64)
    out = np.zeros(e.shape[:2] + (4,), np.uint8)
    for y in range(e.shape[0]):
        for x in range(e.shape[1]):
            m = e[y, x].max()
            if m <= 1e-32:
                continue
            _, ex = math.frexp(m)
            out[y, x, :3] = [min(255, int(math.floor(max(c, 0.0) * 256.0 / 2.0 ** ex))) for c in e[y, x]]
            out[y, x, 3] = ex + 128
    return out


def rgbe_decode(px):
    """Radiance's decoding, as nero_b200.relight reads it: (byte + 1/2) 2^(e - 136), 0 where e = 0."""
    e = px[..., 3].astype(np.int32)
    return ((px[..., :3] + 0.5) * np.where(e > 0, np.ldexp(1.0, e - 136), 0.0)[..., None]).astype(np.float32)
