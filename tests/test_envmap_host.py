"""CPU: the environment-light oracle against the reference fixtures (tests/golden/envmap_*.npz), the map's directions against
relight's own lookup, the .hdr / .exr writers read back by relight.load_env_map (and OpenCV), the bindings of
include/nero_envmap.h and the argument handling of tools/extract_lighting.py.  No GPU."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

import nero_oracle_envmap as OE
import nero_oracle_relight as ORl
from nero_b200 import envmap as EM
from nero_b200.relight import MESH_TRANS, env_tables, load_env_map

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden')
FIXTURES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, 'envmap_*.npz')))


def test_seven_fixtures():
    assert len(FIXTURES) == 7


@pytest.mark.parametrize('name', FIXTURES)
def test_oracle_matches_reference_fixture(name):
    g = np.load(os.path.join(GOLD, name + '.npz'))
    W, H, s = int(g['width']), int(g['height']), int(g['ssaa'])
    d = OE.directions(W, H, s)
    np.testing.assert_array_equal(d, g['dirs'])
    sd, prefix, sphere = OE.fixture_params(g)
    rad = OE.radiance(sd, prefix, torch.from_numpy(d), float(g['kappa_inv']), sphere, g['center'], float(g['exp_max']))
    np.testing.assert_allclose(rad, g['rad'], rtol=1e-6, atol=1e-7)
    env = OE.resolve(rad, W, H, s)
    np.testing.assert_allclose(env, g['env'], rtol=1e-6, atol=1e-7)
    assert np.ptp(g['rad']) > 0.005           # the light varies over the sphere


@pytest.mark.parametrize('trans', [False, True])
@pytest.mark.parametrize('W,H,s', [(16, 8, 2), (37, 19, 3), (64, 32, 4), (5, 3, 1)])
def test_subsample_directions_map_back_to_their_texel(W, H, s, trans):
    """Through relight's own lookup (env_uv, texel) and the row flip of env_tables, every sub-sample of texel (x, y) lands in
    (x, y); with --trans the map's direction is MESH_TRANS applied to the queried (network) direction."""
    frame = EM.trans_frame(trans)
    d = OE.directions(W, H, s, frame).astype(np.float64)
    scene = d @ MESH_TRANS.T if trans else d
    u, v = ORl.env_uv(scene)
    t = ORl.texel(u, v, W, H)                    # j * W + i with j counted from the bottom (env_tables' row order)
    j, i = t // W, t % W
    want = np.repeat(np.arange(W * H), s * s)
    np.testing.assert_array_equal((H - 1 - j) * W + i, want)
    # the flip is the one env_tables makes: its rows run from the bottom
    env = np.random.RandomState(1).rand(H, W, 3).astype(np.float32)
    tab = env_tables(env)['env'].reshape(-1, 4)[:, :3]
    np.testing.assert_array_equal(tab[t], env.reshape(-1, 3)[want])
    np.testing.assert_allclose(np.linalg.norm(d, axis=-1), 1.0, atol=1e-6)


def test_weights_are_cos_elevation_within_the_texel():
    w = OE.weights(4, 6, 3)
    assert w.shape == (24, 9) and (w > 0).all()
    np.testing.assert_allclose(w[:, 0], w[:, 2])                 # a only moves along u
    assert (w[:4, 0] > w[:4, 3]).all() and (w[-4:, 0] < w[-4:, 3]).all()     # b rises towards +z: row 0 is the top


def hdr_values(rng):
    mag = 10.0 ** rng.uniform(-6, 4, size=(7, 33, 1))
    env = (mag * rng.rand(7, 33, 3)).astype(np.float32)
    env[0, :5] = 0.0
    env[1, :] = env[1, :1]          # a constant scanline: one run per channel
    env[2, 3:9] = [1e4, 2e-6, 0.0]
    return env


def test_write_hdr_reads_back_within_the_rgbe_bound(tmp_path):
    env = hdr_values(np.random.RandomState(2))
    p = str(tmp_path / 'a.hdr')
    EM.write_hdr(p, env)
    back = load_env_map(p)
    assert back.shape == env.shape and back.dtype == np.float32
    np.testing.assert_array_equal(back, OE.rgbe_decode(OE.rgbe(env)))
    np.testing.assert_array_equal(EM.rgbe(env), OE.rgbe(env))
    top = env.max(-1, keepdims=True)
    assert (np.abs(back - env) <= top * 2.0 ** -8).all()
    zero = top[..., 0] == 0
    assert zero.any() and (back[zero] == 0).all()
    assert os.path.getsize(p) < 4 * env.size // 3 + 200            # run-length scanlines


def test_write_hdr_narrow_maps_are_flat(tmp_path):
    env = hdr_values(np.random.RandomState(3))[:, :6]
    p = str(tmp_path / 'b.hdr')
    EM.write_hdr(p, env)
    np.testing.assert_array_equal(load_env_map(p), OE.rgbe_decode(OE.rgbe(env)))


def test_opencv_reads_the_hdr(tmp_path):
    cv2 = pytest.importorskip('cv2')
    env = hdr_values(np.random.RandomState(4))
    p = str(tmp_path / 'c.hdr')
    EM.write_hdr(p, env)
    img = cv2.imread(p, cv2.IMREAD_ANYDEPTH | cv2.IMREAD_COLOR)
    assert img is not None and img.shape == env.shape
    ours = load_env_map(p)
    top = env.max(-1, keepdims=True)
    assert (np.abs(img[..., ::-1] - ours) <= top * 2.0 ** -8 + 1e-30).all()


@pytest.mark.parametrize('compression', ['none', 'zip'])
def test_write_exr_reads_back_bit_exact(tmp_path, compression):
    env = hdr_values(np.random.RandomState(5))
    env = np.concatenate([env] * 3, 0)                 # 21 rows: a partial last ZIP block
    env[3, 4] = [-0.0, np.float32(1e-40), np.float32(3.4e38)]
    p = str(tmp_path / f'd_{compression}.exr')
    EM.write_exr(p, env, compression)
    back = load_env_map(p)
    assert back.dtype == np.float32
    np.testing.assert_array_equal(back.view(np.uint32), env.view(np.uint32))


def test_preview_is_clamped_srgb(tmp_path):
    env = np.asarray([[[0.0, 0.5, 4.0], [1e-3, 1.0, 0.25]]], np.float32)
    img = EM.preview(env)
    assert img.dtype == np.uint8 and img[0, 0, 0] == 0 and img[0, 0, 2] == 255 and img[0, 1, 1] == 255
    assert EM.preview(env, exposure=-2.0)[0, 0, 2] == 255 and EM.preview(env, exposure=-4.0)[0, 0, 2] < 255
    EM.write_preview_png(str(tmp_path / 'p.png'), env)
    assert (tmp_path / 'p.png').read_bytes()[:8] == b'\x89PNG\r\n\x1a\n'


def test_argument_checks():
    with pytest.raises(ValueError):
        EM._sphere_mode('stage3')
    with pytest.raises(ValueError):
        EM._check_size(16, 8, 0)
    with pytest.raises(ValueError):
        EM._frame_tensor(np.eye(2), 'cpu')


def test_envmap_header_bindings():
    from nero_b200 import ops
    assert set(ops.ENVMAP_PROTOS) == {'nero_env_rows', 'nero_env_resolve'}
    for name, argtypes in ops.ENVMAP_PROTOS.items():
        fn = getattr(ops.lib, name)
        assert fn.argtypes == argtypes
    assert len(ops.ENVMAP_PROTOS['nero_env_rows']) == 15 and len(ops.ENVMAP_PROTOS['nero_env_resolve']) == 9


# ------------------------------------------------------------------------------------------------ the tool
def tool():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import extract_lighting
    return extract_lighting


def test_tool_arguments():
    t = tool()
    f = t.parse(['--cfg', 'x.yaml'])
    assert (f.width, f.height, f.ssaa, f.trans, f.exr) == (1024, 512, 4, False, False)
    assert tuple(f.center) == (0.0, 0.0, 0.0) and tuple(f.kappa) == (0.0, 0.1, 0.25, 0.5, 1.0)
    f = t.parse(['--cfg', 'x.yaml', '--width', '64', '--height', '32', '--ssaa', '2', '--trans', '--center', '0.1', '-0.2', '0.3',
                 '--kappa', '0', '1', '--exr'])
    assert (f.width, f.height, f.ssaa, f.trans, f.exr) == (64, 32, 2, True, True)
    assert list(f.center) == [0.1, -0.2, 0.3] and list(f.kappa) == [0.0, 1.0]
    for bad in (['--ssaa', '0'], ['--width', '0'], ['--kappa', '-1'], ['--center', '1', '2']):
        with pytest.raises(SystemExit):
            t.parse(['--cfg', 'x.yaml'] + bad)


def test_tool_refuses_a_config_without_an_outer_light(tmp_path):
    t = tool()
    p = tmp_path / 'nerf.yaml'
    p.write_text('name: lego\nnetwork: nerf\n')
    with pytest.raises(SystemExit, match='shape or a material'):
        t.main(['--cfg', str(p)])
    p.write_text('name: lego\n')
    with pytest.raises(SystemExit):
        t.main(['--cfg', str(p)])
    for net in ('shape', 'material'):
        p.write_text(f'name: bell\nnetwork: {net}\n')
        assert t.load_cfg(str(p))['network'] == net
