"""GPU: the glTF export's kernels against the numpy oracle (the weld exactly, tangent frames to 2e-6 of float64, converted
bytes exactly, the metallic-roughness texture exactly), and texture export -> tools/bake_normal_map.py ->
tools/export_gltf.py end to end: positions, winding against NORMAL, the decode bound on the file and identical bytes on two
runs."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import nero_oracle_gltf as OG
import nero_oracle_normalmap as ON
from nero_b200 import gltf as GL
from nero_b200 import normalmap as NM
from nero_b200 import relight as RL
from nero_b200 import texmap as TX
from nero_b200.simplify import _vertex_triangles, simplify
from test_normalmap_gpu import low_and_detail, mc_mesh

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unwrapped(kind, faces=1500, size=128):
    """A 64^3 marching-cubes mesh simplified to `faces` triangles and unwrapped at size^2, vt as the OBJ stores it."""
    v, t, _ = simplify(*mc_mesh(64, kind), faces)
    vt_atlas, ft = TX.uv_atlas(v, t, size, size, 2)
    return v, t, np.stack([vt_atlas[:, 0], np.float32(1) - vt_atlas[:, 1]], -1), ft


def gpu_stages(v, t, vt, ft):
    dev = torch.device('cuda')
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    v_d, t_d, vt_d, ft_d = up(v), up(t), up(vt), up(ft)
    ptr, tri = _vertex_triangles(t_d, v.shape[0])
    normals = NM.vertex_normals_cuda(v_d, t_d)
    wv, wt, wf = GL.weld_cuda(t_d, ft_d, v.shape[0], ptr, tri)
    wn, wtan = GL.frames_cuda(v_d, t_d, vt_d, ft_d, ptr, tri, normals, wv, wt)
    return dict(normals=normals.cpu().numpy(), wv=wv.cpu().numpy(), wt=wt.cpu().numpy(), wf=wf, wn=wn, wtan=wtan)


@pytest.mark.parametrize('kind', ['bumpy', 'torus'])
def test_weld_and_frames_match_the_oracle(kind):
    v, t, vt, ft = unwrapped(kind)
    g = gpu_stages(v, t, vt, ft)
    wv, wt, wf = OG.weld(t, ft, v.shape[0])
    assert np.array_equal(g['wv'], wv) and np.array_equal(g['wt'], wt) and np.array_equal(g['wf'].cpu().numpy(), wf)
    assert wv.size == np.unique(np.stack([t.reshape(-1), ft.reshape(-1)], -1), axis=0).shape[0] > v.shape[0]
    wn, wtan = OG.frames(v, t, vt, ft, g['normals'], wv, wt, wf)
    got_n, got_t = g['wn'].cpu().numpy().astype(np.float64), g['wtan'].cpu().numpy().astype(np.float64)
    assert np.array_equal(got_n, wn)
    err = np.abs(got_t[:, :3] - wtan[:, :3]).max(1)
    print(f'{kind}: {wv.size} welded of {v.shape[0]} vertices, max |tangent - float64| {err.max():.2e}, '
          f'{int((got_t[:, 3] < 0).sum())} with w = -1')
    assert err.max() <= 2e-6 and np.array_equal(got_t[:, 3], wtan[:, 3])


@pytest.mark.parametrize('kind', ['bumpy', 'torus'])
def test_tangent_space_bytes_match_the_oracle(kind):
    v, t, vt, ft = unwrapped(kind)
    g = gpu_stages(v, t, vt, ft)
    wn, wtan = g['wn'].cpu().numpy(), g['wtan'].cpu().numpy()
    rng = np.random.RandomState(2)
    omap = rng.randint(0, 256, (96, 128, 3)).astype(np.uint8)
    c = GL.tangent_space_cuda(v, t, vt, ft, g['wf'], g['wn'], g['wtan'], omap)
    ref, fr = OG.tangent_space(vt, ft, g['wf'].cpu().numpy(), wn, wtan, omap)
    assert np.array_equal(c['raster']['texel'].cpu().numpy(), fr['texel']) and fr['texel'].size > 3000
    assert np.array_equal(c['img'].cpu().numpy(), ref)


def test_metal_rough_texture_is_the_tables_applied():
    rng = np.random.RandomState(4)
    m, r = rng.randint(0, 256, (2, 40, 56)).astype(np.uint8)
    got = GL.metal_rough_cuda(m, r).cpu().numpy()
    lut_m, lut_r = OG.material_tables()
    assert np.array_equal(got, np.stack([np.full_like(m, 255), lut_r[r], lut_m[m]], -1))


def export(tmp_path, *extra):
    env = dict(os.environ, PYTHONPATH=ROOT)
    return subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'export_gltf.py'), '--obj', 'n2m/mesh_0.obj', *extra],
                          cwd=tmp_path, env=env, capture_output=True, text=True, check=True).stdout


def test_tools_end_to_end(tmp_path):
    """write_textured_obj -> tools/bake_normal_map.py -> tools/export_gltf.py, read back with read_glb."""
    from nero_b200.mesh import write_ply
    lv, lt, dv, dt = low_and_detail(64, 48, 1200)
    vt_atlas, ft = TX.uv_atlas(lv, lt, 128, 128, 2)
    rng = np.random.RandomState(1)
    maps = (rng.randint(60, 200, (64, 64, 3)).astype(np.uint8), np.repeat(rng.randint(0, 256, (64, 64, 1)), 3, -1).astype(np.uint8),
            np.repeat(rng.randint(0, 256, (64, 64, 1)), 3, -1).astype(np.uint8))
    TX.write_textured_obj(str(tmp_path / 'n2m'), lv, lt, vt_atlas, ft, maps)
    write_ply(str(tmp_path / 'detail.ply'), dv, dt)
    env = dict(os.environ, PYTHONPATH=ROOT)
    subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'bake_normal_map.py'), '--obj', 'n2m/mesh_0.obj', '--detail', 'detail.ply'],
                   cwd=tmp_path, env=env, check=True, capture_output=True)
    out = export(tmp_path, '--normal-map', 'n2m/normal_0.png')
    print(out)
    assert 'welded vertices' in out and 'covered texels' in out
    first = (tmp_path / 'n2m' / 'mesh_0.glb').read_bytes()
    export(tmp_path, '--normal-map', 'n2m/normal_0.png')
    assert (tmp_path / 'n2m' / 'mesh_0.glb').read_bytes() == first
    g = GL.read_glb(str(tmp_path / 'n2m' / 'mesh_0.glb'))
    v, t, vt, ft_f, _ = RL.load_textured_obj(str(tmp_path / 'n2m' / 'mesh_0.obj'))
    wv, wt, wf = OG.weld(t, ft_f, v.shape[0])
    assert np.array_equal(g['positions'], v[wv]) and np.array_equal(g['indices'], wf[:, [0, 2, 1]])
    assert np.array_equal(g['texcoords'], np.stack([vt[wt, 0], np.float32(1) - vt[wt, 1]], -1))
    assert g['rotation'] == GL.Z_UP_ROTATION and g['tangents'] is not None
    # glTF's counter-clockwise faces point the way NORMAL does on this closed mesh
    p = g['positions'].astype(np.float64)[g['indices']]
    fn = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
    ok = np.linalg.norm(fn, axis=1) > 1e-12
    dots = (g['normals'][g['indices']] * fn[:, None]).sum(-1)
    assert (dots[ok] > 0).all(), f'{int((dots[ok] <= 0).any(1).sum())} faces against NORMAL'
    # the images: base colour = feat0's bytes, metallic-roughness = the tables, the normal texture decodes to the map
    assert np.array_equal(g['images']['base_color'], maps[0])
    lut_m, lut_r = OG.material_tables()
    assert np.array_equal(g['images']['metallic_roughness'][..., 1], lut_r[maps[2][..., 0]])
    assert np.array_equal(g['images']['metallic_roughness'][..., 2], lut_m[maps[1][..., 0]])
    omap = NM.read_normal_map_bytes(str(tmp_path / 'n2m' / 'normal_0.png'))
    h, w = omap.shape[:2]
    ind = g['indices'][:, [0, 2, 1]].astype(np.int64)
    fr = OG.texel_frames(g['texcoords'], ind, ind, g['normals'], g['tangents'], w, h, np.float64)
    got = OG.viewer_decode(g['images']['normal'], fr)
    err = OG.angle_deg(got, ON.decode(omap.reshape(-1, 3)[fr['texel']]).astype(np.float64))
    print(f'decode: {err.size} texels, median {np.median(err):.3f} deg, 99.9th percentile {np.percentile(err, 99.9):.3f}')
    assert (err <= 1.0).mean() >= 0.999 and np.median(err) <= 0.4
    # without a map: no TANGENT, no normal texture; --trans: no rotation
    export(tmp_path, '--trans', '--out', 'plain.glb')
    p = GL.read_glb(str(tmp_path / 'plain.glb'))
    assert p['tangents'] is None and 'normal' not in p['images'] and p['rotation'] is None
    assert np.array_equal(p['positions'], g['positions']) and np.array_equal(p['normals'], g['normals'])
