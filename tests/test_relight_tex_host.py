"""CPU checks of relighting from UV textures: the textured-OBJ reader against texmap's writer (PNG) and OpenCV JPEGs under the
reference's names, its refusals, the oracle's texture lookup, the UVMaterials refusals, the bindings of
include/nero_relight_tex.h and the argument handling of tools/relight.py.  No GPU."""
import os
import sys

import numpy as np
import pytest

import nero_oracle_relight as OR
import nero_oracle_relight_tex as ORT
from nero_b200 import relight as RL
from nero_b200 import texmap as TX

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def random_asset(seed=0, V=40, T=60, N=70, H=12, W=20):
    rng = np.random.RandomState(seed)
    verts = rng.randn(V, 3).astype(np.float32)
    tris = rng.randint(0, V, (T, 3)).astype(np.int32)
    vt = rng.rand(N, 2).astype(np.float32)
    ft = rng.randint(0, N, (T, 3)).astype(np.int32)
    images = (rng.randint(0, 256, (H, W, 3)).astype(np.uint8),) + tuple(
        np.repeat(rng.randint(0, 256, (H, W, 1)).astype(np.uint8), 3, -1) for _ in range(2))
    return verts, tris, vt, ft, images


def decoded(img8):
    return RL.srgb_to_linear(img8.astype(np.float64) / 255).astype(np.float32)


def test_obj_round_trip_through_the_texture_writer(tmp_path):
    verts, tris, vt, ft, images = random_asset()
    TX.write_textured_obj(str(tmp_path), verts, tris, vt, ft, images)
    v, t, vt2, ft2, maps = RL.load_textured_obj(str(tmp_path / 'mesh_0.obj'))
    assert v.dtype == np.float32 and t.dtype == np.int32 and vt2.dtype == np.float32 and ft2.dtype == np.int32
    np.testing.assert_array_equal(v, verts)
    np.testing.assert_array_equal(t, tris)
    np.testing.assert_array_equal(ft2, ft)
    np.testing.assert_array_equal(vt2[:, 0], vt[:, 0])
    np.testing.assert_array_equal(vt2[:, 1], np.float32(1) - vt[:, 1])       # the file stores 1 - v of the atlas
    np.testing.assert_array_equal(maps['albedo'], decoded(images[0]))
    np.testing.assert_array_equal(maps['metallic'], decoded(images[1][..., :1]))
    np.testing.assert_array_equal(maps['roughness'], decoded(images[2][..., :1]))
    # the a/b/n face form is accepted and its normal index ignored
    obj = (tmp_path / 'mesh_0.obj').read_text().splitlines()
    obj = [' '.join(c + '/1' if i else c for i, c in enumerate(l.split())) if l.startswith('f ') else l for l in obj]
    (tmp_path / 'mesh_0.obj').write_text('\n'.join(obj + ['vn 0 0 1']) + '\n')
    _, t3, _, ft3, _ = RL.load_textured_obj(str(tmp_path / 'mesh_0.obj'))
    np.testing.assert_array_equal(t3, tris)
    np.testing.assert_array_equal(ft3, ft)


def test_reference_jpeg_names(tmp_path):
    """The reference writes feat{0,1,2}_0.jpg with OpenCV (BGR albedo, grey metallic and roughness) and names the JPEG in
    map_Kd.  The maps are what OpenCV reads back: albedo in RGB order, metallic and roughness from the red channel."""
    import cv2
    verts, tris, vt, ft, images = random_asset(1)
    y, x = np.mgrid[:12, :20]
    images = (np.stack([40 + 8 * x, 200 - 5 * y, 90 + 0 * x], -1).astype(np.uint8),) + images[1:]   # smooth: JPEG keeps it
    TX.write_textured_obj(str(tmp_path), verts, tris, vt, ft, images)
    for k in range(3):
        os.remove(tmp_path / f'feat{k}_0.png')
    cv2.imwrite(str(tmp_path / 'feat0_0.jpg'), images[0][..., ::-1])
    cv2.imwrite(str(tmp_path / 'feat1_0.jpg'), images[1][..., 0])
    cv2.imwrite(str(tmp_path / 'feat2_0.jpg'), images[2][..., 0])
    mtl = (tmp_path / 'mesh_0.mtl').read_text().replace('feat0_0.png', 'feat0_0.jpg')
    (tmp_path / 'mesh_0.mtl').write_text(mtl)
    _, _, _, _, maps = RL.load_textured_obj(str(tmp_path / 'mesh_0.obj'))
    back = [cv2.imread(str(tmp_path / f'feat{k}_0.jpg'), cv2.IMREAD_COLOR)[..., ::-1] for k in range(3)]
    np.testing.assert_array_equal(maps['albedo'], decoded(back[0]))
    np.testing.assert_array_equal(maps['metallic'], decoded(back[1][..., :1]))
    np.testing.assert_array_equal(maps['roughness'], decoded(back[2][..., :1]))
    assert np.abs(maps['albedo'] - decoded(images[0])).max() < 0.05               # lossy, but in RGB order


def edited_asset(tmp_path, edit):
    verts, tris, vt, ft, images = random_asset(2)
    TX.write_textured_obj(str(tmp_path), verts, tris, vt, ft, images)
    path = tmp_path / 'mesh_0.obj'
    lines = path.read_text().splitlines()
    edit(lines, tmp_path)
    path.write_text('\n'.join(lines) + '\n')
    return str(path)


def first(lines, prefix):
    return next(i for i, l in enumerate(lines) if l.startswith(prefix))


def _quad(lines, _):
    i = first(lines, 'f ')
    lines[i] += ' 1/1'


def _no_uv(lines, _):
    i = first(lines, 'f ')
    lines[i] = 'f ' + ' '.join(c.split('/')[0] for c in lines[i].split()[1:])


def _no_uv_with_normal(lines, _):
    i = first(lines, 'f ')
    lines[i] = 'f ' + ' '.join(c.split('/')[0] + '//1' for c in lines[i].split()[1:])


def _vertex_out_of_range(lines, _):
    i = first(lines, 'f ')
    lines[i] = 'f 41/1 1/1 2/2'


def _uv_out_of_range(lines, _):
    i = first(lines, 'f ')
    lines[i] = 'f 1/71 2/1 3/2'


def _zero_index(lines, _):
    i = first(lines, 'f ')
    lines[i] = 'f 0/1 2/1 3/2'


def _nan_vertex(lines, _):
    lines[first(lines, 'v ')] = 'v nan 0 0'


def _inf_uv(lines, _):
    lines[first(lines, 'vt ')] = 'vt inf 0.5'


def _missing_texture(_, d):
    os.remove(d / 'feat2_0.png')


def _sizes_differ(_, d):
    RL.write_png(str(d / 'feat1_0.png'), np.zeros((5, 7, 3), np.uint8))


def _missing_mtl(_, d):
    os.remove(d / 'mesh_0.mtl')


@pytest.mark.parametrize('edit, match', [
    (_quad, 'only triangles'), (_no_uv, 'no uv index'), (_no_uv_with_normal, 'no uv index'),
    (_vertex_out_of_range, 'vertex index 41 is out of range'), (_uv_out_of_range, 'uv index 71 is out of range'),
    (_zero_index, 'vertex index 0 is out of range'), (_nan_vertex, 'non-finite vertex'), (_inf_uv, 'non-finite texture vertex'),
    (_missing_texture, 'feat2_0.png: texture file is missing'), (_sizes_differ, 'texture maps differ in size'),
    (_missing_mtl, 'mesh_0.mtl: material file is missing')])
def test_reader_refusals(tmp_path, edit, match):
    path = edited_asset(tmp_path, edit)
    with pytest.raises(ValueError, match=match) as e:
        RL.load_textured_obj(path)
    assert str(tmp_path) in str(e.value)              # the message names the file


# ------------------------------------------------------------------------------------------------ the oracle's lookup
def test_lookup_is_exact_on_affine_textures_at_interior_points():
    H, W = 9, 14
    y, x = np.mgrid[:H, :W].astype(np.float64)
    tex = np.stack([0.3 + 0.02 * x - 0.05 * y, 1.0 - 0.01 * x + 0.07 * y], -1)
    rng = np.random.RandomState(0)
    s, t = rng.uniform(0, W - 1, 500), rng.uniform(0, H - 1, 500)
    uv = np.stack([(s + 0.5) / W, 1 - (t + 0.5) / H], -1)
    got = ORT.texture_lookup(tex, uv)
    s, t = uv[:, 0] * W - 0.5, (1 - uv[:, 1]) * H - 0.5
    want = np.stack([0.3 + 0.02 * s - 0.05 * t, 1.0 - 0.01 * s + 0.07 * t], -1)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-14)
    # texel centres return the texel; row 0 of the image is v = 1
    np.testing.assert_array_equal(ORT.texture_lookup(tex, [[0.5 / W, 1 - 0.5 / H]])[0], tex[0, 0])
    np.testing.assert_array_equal(ORT.texture_lookup(tex, [[(W - 0.5) / W, 0.5 / H]])[0], tex[H - 1, W - 1])


def test_lookup_wraps_continuously_and_keeps_constants():
    rng = np.random.RandomState(1)
    tex = rng.rand(6, 10, 5)
    v = rng.rand(200)
    for e in (0.0, 1e-9):
        a = ORT.texture_lookup(tex, np.stack([np.full_like(v, e), v], -1))
        b = ORT.texture_lookup(tex, np.stack([np.full_like(v, 1 - e), v], -1))
        assert np.abs(a - b).max() <= 1e-7
    shifted = ORT.texture_lookup(tex, np.stack([v * 0 + 3, v - 2], -1))                    # whole periods away
    np.testing.assert_allclose(ORT.texture_lookup(tex, np.stack([v * 0, v], -1)), shifted, rtol=0, atol=1e-12)
    c = np.float64(np.float32(0.123456789))
    uv = rng.uniform(-3, 4, (300, 2))
    assert (ORT.texture_lookup(np.full((5, 7, 1), c), uv) == c).all()


def test_textured_oracle_reproduces_the_vertex_oracle_on_constant_materials():
    """Constant materials given per vertex (roughness r, squared to alpha) and as a constant texture (alpha = r^2 stored)
    describe one scene, so the textured oracle's loop must give the per-vertex oracle's image: the same coverage, and
    colours equal up to the rounding of the barycentric sum of three equal values."""
    import nero_oracle_mat as OM
    verts, tris = OM.test_scene(1)
    V, T = verts.shape[0], tris.shape[0]
    alb, met, r = np.asarray([0.7, 0.4, 0.2]), 0.3, 0.6
    vmat = np.zeros((V, 8))
    vmat[:, :3], vmat[:, 3], vmat[:, 4] = alb, met, r
    tex = np.zeros((3, 5, 8))
    tex[..., :3], tex[..., 3], tex[..., 4] = alb, met, r ** 2
    rng = np.random.RandomState(2)
    uvm = (rng.uniform(-1, 2, (7, 2)), rng.randint(0, 7, (T, 3)), tex)
    tables = RL.env_tables(np.exp(rng.randn(8, 16, 3)).astype(np.float32))
    pose, K = RL.relight_poses(3, 20.0, 30.0, 2.0)[1], RL.blender_default_K(12, 12)
    want = OR.render(verts, tris, vmat, tables, pose, K, 12, 12, 2, 3, seed=4, ggx_smith=1)
    got = ORT.render(verts, tris, uvm, tables, pose, K, 12, 12, 2, 3, seed=4, ggx_smith=1)
    assert want[..., 3].any() and not want[..., 3].all()
    np.testing.assert_array_equal(got[..., 3], want[..., 3])
    np.testing.assert_allclose(got[..., :3], want[..., :3], rtol=1e-12, atol=1e-15)


# ------------------------------------------------------------------------------------------------ API and bindings
def test_uv_materials_refusals():
    vt = np.random.RandomState(0).rand(5, 2)
    ft = np.asarray([[0, 1, 2], [2, 3, 4]])
    a, m = np.zeros((4, 6, 3)), np.zeros((4, 6))
    RL.UVMaterials(vt, ft, a, m, m[..., None])
    for bad, match in (((vt, ft + 1, a, m, m), 'outside'), ((vt, ft - 1, a, m, m), 'outside'), ((vt, ft, a, m[:3], m), 'metallic'),
                       ((vt, ft, a[..., :2], m, m), 'albedo'), ((vt * np.nan, ft, a, m, m), 'non-finite'),
                       ((vt[:, :1], ft, a, m, m), 'vt')):
        with pytest.raises(ValueError, match=match):
            RL.UVMaterials(*bad)
    verts = np.random.RandomState(1).rand(5, 3)
    with pytest.raises(ValueError, match='ft has shape'):
        RL.Relighter(verts, np.asarray([[0, 1, 2]]), RL.UVMaterials(vt, ft, a, m, m), np.ones((2, 4, 3), np.float32))
    t = RL.UVMaterials(vt, ft, a + 0.25, m + 0.5, m + 0.75).texel_table()
    assert t.shape == (4, 6, 8) and (t[..., :3] == 0.25).all() and (t[..., 3] == 0.5).all() and (t[..., 4] == 0.75).all()
    assert (t[..., 5:] == 0).all()


def test_textured_entry_point_binding():
    from nero_b200 import ops
    assert set(ops.RELIGHT_TEX_PROTOS) == {'nero_relight_render_textured'}
    argtypes = ops.RELIGHT_TEX_PROTOS['nero_relight_render_textured']
    assert getattr(ops.lib, 'nero_relight_render_textured').argtypes == argtypes          # the library exports it
    assert [a.__name__ for a in argtypes] == ['Ptr', 'Ptr', 'Ptr', 'c_int', 'Ptr', 'c_int', 'c_int', 'Ptr']
    # the per-vertex entry point and its record are unchanged
    assert ops.lib.nero_relight_render.argtypes == [ops.Ptr, ops.Ptr]
    assert ops.ctypes.sizeof(ops.RelightParams) == ops.lib.nero_abi_sizeof(ops.ABI_RECORDS.index('nero_relight_params'))


# ------------------------------------------------------------------------------------------------ the tool
def tool():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import relight
    return relight


def test_tool_arguments(tmp_path):
    t = tool()
    common = ['--hdr', 'e.hdr', '--name', 'n']
    f = t.parse(['--mesh', 'm.ply', '--material', 'mat'] + common)
    assert (f.mesh, f.material, f.obj) == ('m.ply', 'mat', None)
    f = t.parse(['--obj', 'x/mesh_0.obj', '--trans'] + common)
    assert (f.mesh, f.material, f.obj, f.trans) == (None, None, 'x/mesh_0.obj', True)
    for bad in (['--obj', 'o.obj', '--mesh', 'm.ply'], ['--obj', 'o.obj', '--material', 'mat'],
                ['--obj', 'o.obj', '--mesh', 'm.ply', '--material', 'mat'], ['--mesh', 'm.ply'], ['--material', 'mat'], []):
        with pytest.raises(SystemExit):
            t.parse(bad + common)
    # --obj without its texture files fails before anything is rendered
    verts, tris, vt, ft, images = random_asset(3)
    TX.write_textured_obj(str(tmp_path), verts, tris, vt, ft, images)
    os.remove(tmp_path / 'feat0_0.png')
    with pytest.raises(ValueError, match='texture file is missing'):
        t.main(['--obj', str(tmp_path / 'mesh_0.obj')] + common)
    with pytest.raises(FileNotFoundError):
        t.main(['--obj', str(tmp_path / 'none.obj')] + common)


def test_textured_entry_point_refusals():
    """Every refusal returns 1 before anything reaches the GPU; with spp = 0 a valid call returns 0 and launches nothing."""
    from nero_b200 import ops
    fake = 0x1000                                     # never dereferenced: the checks return first
    q = ops.RelightParams().set(nodes=fake, tris=fake, tri_ids=fake, faces=fake, env=fake, env_p=fake, cdf_rows=fake, cdf_cols=fake,
                                accum=fake)
    q.env_w, q.env_h, q.width, q.height, q.spp0, q.spp, q.max_bounces = 4, 2, 8, 8, 0, 0, 1
    f = ops.lib.nero_relight_render_textured
    ok = (ops.ctypes.byref(q), fake, fake, 3, fake, 4, 2, None)
    assert f(*ok) == 0
    for i, bad in ((0, None), (1, None), (2, None), (3, 0), (4, None), (5, 0), (6, 0)):
        args = list(ok)
        args[i] = bad
        assert f(*args) == 1, i
    q.vmat = fake                                     # the per-vertex table must not be set
    assert f(*ok) == 1
    q.vmat = None
    q.max_bounces = 0                                 # a check the per-vertex entry point makes
    assert f(*ok) == 1 and ops.lib.nero_relight_render(ops.ctypes.byref(q), None) == 1
