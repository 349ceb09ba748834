"""UV texture-map export on the GPU: the raster, encode, inpaint and down-sample kernels against the numpy oracle, the whole
bake against the reference fixtures, texture / vertex consistency, the tool end to end and its refusals."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_mat as OM
import nero_oracle_texmap as OT
from nero_b200 import texmap as TX

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
FIXTURES = ['texmap_scene_32x32', 'texmap_blob_40x64']
SHADER_CFG = {'human_lights': False, 'diffuse_sample_num': 16, 'specular_sample_num': 16}


def grid_on_texel_centres(n=6, w=48, h=40):
    """A plane grid whose uv vertices sit exactly on texel centres and edges: every shared edge and corner is hit."""
    ij = np.stack(np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing='ij'), -1).reshape(-1, 2)
    verts = np.concatenate([ij.astype(np.float32) / n, np.zeros((ij.shape[0], 1), np.float32)], 1)
    vt = np.stack([(4 + 6 * ij[:, 0] + 0.5) / w, (3 + 5 * ij[:, 1] + 0.5) / h], 1).astype(np.float32)
    q = np.arange(n)
    a = (q[:, None] * (n + 1) + q[None, :]).reshape(-1)
    tris = np.concatenate([np.stack([a, a + n + 1, a + n + 2], 1), np.stack([a, a + n + 2, a + 1], 1)]).astype(np.int32)
    tris[::3] = tris[::3, [0, 2, 1]]           # both windings
    return verts, tris, vt, tris.copy(), w, h


def atlas_cases():
    verts, tris = OM.test_scene(2)
    vt, ft = TX.uv_atlas(verts, tris, 256, 192, 4)
    yield verts, tris, vt, ft, 256, 192
    yield grid_on_texel_centres()
    for name in FIXTURES:
        g = np.load(os.path.join(GOLD, name + '.npz'))
        h, w = g['mask'].shape
        yield g['verts'], g['tris'], g['vt'], g['ft'], w, h


def material_renderer(verts, tris, seed=6033, pseed=11):
    from nero_b200 import params as P
    from nero_b200.material import NeROMaterialRenderer
    sd = O.perturb_params(P.build_material_state_dict(SHADER_CFG, seed=seed), seed=pseed)
    net = NeROMaterialRenderer({'shader_cfg': dict(SHADER_CFG)}, is_train=False, mesh=(verts, tris))
    net.load_state_dict(sd)
    return net.cuda(), sd


def test_raster_matches_oracle():
    for verts, tris, vt, ft, w, h in atlas_cases():
        r = TX.raster(vt, ft, verts, tris, w, h)
        owner, count, bary = OT.rasterize(vt, ft, w, h)
        np.testing.assert_array_equal(r['owner'].cpu().numpy(), owner)
        np.testing.assert_array_equal(r['cover'].cpu().numpy(), count)
        assert count.max() <= 1 and (owner >= 0).any()
        np.testing.assert_array_equal(r['texel'].cpu().numpy(), np.flatnonzero(owner >= 0))
        want = OT.interpolate(verts, tris, owner, bary)[owner >= 0]
        ext = float(np.abs(verts).max())
        assert np.abs(r['xyz'].cpu().numpy() - want).max() <= 1e-6 * ext


def test_shared_edges_and_corners_are_owned_once():
    verts, tris, vt, ft, w, h = grid_on_texel_centres()
    r = TX.raster(vt, ft, verts, tris, w, h)
    cover = r['cover'].cpu().numpy()
    # every texel centre strictly inside the grid's rectangle [4, 40] x [3, 33] is covered exactly once
    inner = np.zeros((h, w), bool)
    inner[4:33, 5:40] = True
    assert cover.max() == 1 and (cover[inner] == 1).all()


def test_encode_inpaint_downsample_match_oracle_bit_for_bit():
    rng = np.random.RandomState(5)
    for verts, tris, vt, ft, w, h in atlas_cases():
        if w % 2 or h % 2:
            continue
        r = TX.raster(vt, ft, verts, tris, w, h)
        owner = r['owner'].cpu().numpy()
        mask = owner >= 0
        n = int(mask.sum())
        mat = rng.rand(n, 5).astype(np.float32)
        mat[: n // 8] *= 0.004                   # the linear branch of the transfer
        img = TX.encode(torch.from_numpy(mat).cuda(), r['texel'], w, h)
        want = OT.encode(mat, mask)
        np.testing.assert_array_equal(img.cpu().numpy(), want)
        out, src = TX.inpaint(img, r['owner'])
        wout, wsrc = OT.inpaint(want, mask)
        np.testing.assert_array_equal(src.cpu().numpy(), wsrc)
        np.testing.assert_array_equal(out.cpu().numpy(), wout)
        np.testing.assert_array_equal(TX.downsample(out).cpu().numpy(), OT.downsample(wout))


@pytest.mark.parametrize('name', FIXTURES)
def test_bake_matches_reference_fixture(name):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    h0, w0 = (int(x) for x in g['hw0'])
    h, w = g['mask'].shape
    net, _ = material_renderer(g['verts'], g['tris'], int(g['seed']), int(g['pseed']))
    r = TX.raster(g['vt'], g['ft'], g['verts'], g['tris'], w, h)
    mask = r['owner'].cpu().numpy() >= 0
    np.testing.assert_array_equal(mask, g['mask'])
    np.testing.assert_array_equal(r['xyz'].cpu().numpy(), g['xyzs'])
    img = TX.encode(TX.query_materials(net, r['xyz']), r['texel'], w, h)
    d = img.cpu().numpy().astype(int) - g['img_before'].astype(int)
    assert np.abs(d).max() <= 1 and (d == 0).mean() >= 0.995
    out, src = TX.inpaint(img, r['owner'])
    src = src.cpu().numpy().reshape(-1)
    ti, ts = g['inpaint_texels'], g['inpaint_src']
    np.testing.assert_array_equal(np.flatnonzero(src >= 0), np.sort(ti))
    d2 = lambda a, b: (a // w - b // w) ** 2 + (a % w - b % w) ** 2
    np.testing.assert_array_equal(d2(ti, src[ti]), d2(ti, ts))
    same = src[ti] == ts
    o = out.cpu().numpy().reshape(-1, 5)
    dd = o[ti[same]].astype(int) - g['img_after'].reshape(-1, 5)[ti[same]].astype(int)
    assert np.abs(dd).max() <= 1 and (dd == 0).mean() >= 0.995
    alb, met, rough = TX.bake_textures(net, g['verts'], g['tris'], g['vt'], g['ft'], (h0, w0), 2)
    for mine, ref in ((alb, g['feat0'][..., ::-1]), (met, g['feat1']), (rough, g['feat2'])):
        e = mine.astype(int) - ref.astype(int)
        assert mine.shape == (h0, w0, 3) and np.abs(e).max() <= 1 and (e == 0).mean() >= 0.99


def test_textures_agree_with_vertex_materials():
    """Bilinear samples of the written albedo and metallic textures at each vertex's vt agree with the vertex materials."""
    from nero_b200.relight import linear_to_srgb
    verts, tris = OM.test_scene(3)
    net, _ = material_renderer(verts, tris)
    h0 = w0 = 256
    vt, ft = TX.uv_atlas(verts, tris, 2 * w0, 2 * h0, 4)
    alb, met, rough = (im.astype(np.float64) / 255 for im in TX.bake_textures(net, verts, tris, vt, ft, (h0, w0), 2))
    m, r, a = (t.cpu().numpy().astype(np.float64) for t in net.query_materials(torch.from_numpy(verts).cuda()))
    uv = vt[ft.reshape(-1)].astype(np.float64)
    vid = tris.reshape(-1)
    x, y = uv[:, 0] * w0 - 0.5, uv[:, 1] * h0 - 0.5
    x0, y0 = np.floor(x).astype(int), np.floor(y).astype(int)
    fx, fy = x - x0, y - y0

    def sample(img):
        g = lambda yy, xx: img[np.clip(yy, 0, h0 - 1), np.clip(xx, 0, w0 - 1)]
        return ((1 - fy)[:, None] * ((1 - fx)[:, None] * g(y0, x0) + fx[:, None] * g(y0, x0 + 1)) +
                fy[:, None] * ((1 - fx)[:, None] * g(y0 + 1, x0) + fx[:, None] * g(y0 + 1, x0 + 1)))
    for img, want in ((alb, a), (met, np.repeat(m, 3, 1)), (rough, np.repeat(r, 3, 1))):
        err = np.abs(sample(img) - linear_to_srgb(want[vid]))
        assert np.median(err) <= 2 / 255, np.median(err)


def read_png_rgb(path):
    data = open(path, 'rb').read()
    assert data[:8] == b'\x89PNG\r\n\x1a\n'
    w, h = int.from_bytes(data[16:20], 'big'), int.from_bytes(data[20:24], 'big')
    assert data[24:26] == bytes([8, 2])
    i, idat = 8, b''
    while i < len(data):
        n = int.from_bytes(data[i:i + 4], 'big')
        if data[i + 4:i + 8] == b'IDAT':
            idat += data[i + 8:i + 8 + n]
        i += 12 + n
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 3 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 3)


def test_tool_end_to_end(tmp_path):
    import yaml
    from nero_b200.mesh import write_ply
    verts, tris = OM.test_scene(2)
    _, sd = material_renderer(verts, tris)
    os.makedirs(tmp_path / 'data' / 'model' / 'tex', exist_ok=True)
    torch.save({'step': 77, 'network_state_dict': sd}, tmp_path / 'data' / 'model' / 'tex' / 'model_best.pth')
    write_ply(str(tmp_path / 'mesh.ply'), verts, tris)
    cfg = {'name': 'tex', 'network': 'material', 'mesh': str(tmp_path / 'mesh.ply'), 'shader_cfg': dict(SHADER_CFG)}
    (tmp_path / 'cfg.yaml').write_text(yaml.safe_dump(cfg))
    env = dict(os.environ, PYTHONPATH=ROOT)
    tool = os.path.join(ROOT, 'tools', 'extract_materials_texture_map.py')
    files = ['feat0_0.png', 'feat1_0.png', 'feat2_0.png', 'mesh_0.obj', 'mesh_0.mtl']
    runs = []
    for out in ('a', 'b'):
        subprocess.check_call([sys.executable, tool, '--cfg', 'cfg.yaml', '--size', '96', '--out', out], cwd=tmp_path, env=env)
        runs.append([(tmp_path / out / f).read_bytes() for f in files])
    assert runs[0] == runs[1]
    lines = runs[0][3].decode().splitlines()
    n_vt = sum(l.startswith('vt ') for l in lines)
    assert sum(l.startswith('v ') for l in lines) == verts.shape[0] and sum(l.startswith('f ') for l in lines) == tris.shape[0]
    assert verts.shape[0] <= n_vt <= 3 * tris.shape[0]
    for f in files[:3]:
        assert read_png_rgb(tmp_path / 'a' / f).shape == (96, 96, 3)
    assert 'map_Kd feat0_0.png' in runs[0][4].decode()
    cfg['network'] = 'shape'
    (tmp_path / 'bad.yaml').write_text(yaml.safe_dump(cfg))
    p = subprocess.run([sys.executable, tool, '--cfg', 'bad.yaml'], cwd=tmp_path, env=env, capture_output=True, text=True)
    assert p.returncode != 0 and 'material network' in p.stderr


def test_empty_atlas_raises():
    verts, tris = OM.test_scene(1)
    net, _ = material_renderer(verts, tris)
    vt = np.zeros((3, 2), np.float32)            # every triangle collapsed onto one point: no texel is covered
    ft = np.zeros_like(tris)
    with pytest.raises(ValueError, match='no texel'):
        TX.bake_textures(net, verts, tris, vt, ft, (16, 16), 2)
