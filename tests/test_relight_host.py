"""CPU checks of relighting: the material export format, the image readers and writers, the cameras, the environment
sampler, the host-compiled math_relight.cuh against the numpy oracle, and the unbiasedness of the oracle's estimator."""
import ctypes
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest
import torch

import nero_oracle as O
import nero_oracle_relight as OR
from helpers import load_golden
from nero_b200 import relight as RL

HERE = os.path.dirname(os.path.abspath(__file__))


# ------------------------------------------------------------------------------------------------ writers used by the tests
def write_hdr(path, img, rle):
    """Radiance RGBE writer: flat scanlines or new-style run-length scanlines (runs for repeated bytes)."""
    img = np.asarray(img, np.float64)
    H, W = img.shape[:2]
    m = img.max(-1)
    f, e = np.frexp(m)
    rgbe = np.zeros((H, W, 4), np.uint8)
    ok = m > 1e-32
    scale = np.where(ok, f * 256.0 / np.where(ok, m, 1.0), 0.0)
    rgbe[..., :3] = np.where(ok[..., None], np.floor(img * scale[..., None]), 0).astype(np.uint8)
    rgbe[..., 3] = np.where(ok, e + 128, 0).astype(np.uint8)
    out = bytearray(b'#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n' + f'-Y {H} +X {W}\n'.encode())
    for y in range(H):
        if not rle:
            out += rgbe[y].tobytes()
            continue
        out += bytes([2, 2, W >> 8, W & 0xff])
        for c in range(4):
            row, x = rgbe[y, :, c], 0
            while x < W:
                n = 1
                while x + n < W and n < 127 and row[x + n] == row[x]:
                    n += 1
                if n >= 3:
                    out += bytes([128 + n, row[x]])
                    x += n
                else:
                    n = 1
                    while x + n < W and n < 128 and not (x + n + 2 < W and row[x + n] == row[x + n + 1] == row[x + n + 2]):
                        n += 1
                    out += bytes([n]) + row[x:x + n].tobytes()
                    x += n
    with open(path, 'wb') as fh:
        fh.write(bytes(out))
    ex = rgbe[..., 3].astype(np.int32)
    return ((rgbe[..., :3] + 0.5) * np.where(ex > 0, np.ldexp(1.0, ex - 136), 0.0)[..., None]).astype(np.float32)


def _attr(name, typ, body):
    return name.encode() + b'\0' + typ.encode() + b'\0' + struct.pack('<i', len(body)) + body


def write_exr(path, img, compression, ptype):
    """Scanline OpenEXR writer: channels B, G, R (stored alphabetically), NONE (0), ZIPS (2) or ZIP (3), half (1) / float (2)."""
    H, W = img.shape[:2]
    dt = {1: np.dtype('<f2'), 2: np.dtype('<f4')}[ptype]
    chl = b''.join(c.encode() + b'\0' + struct.pack('<iBBBBii', ptype, 0, 0, 0, 0, 1, 1) for c in 'BGR') + b'\0'
    hdr = struct.pack('<ii', 20000630, 2)
    hdr += _attr('channels', 'chlist', chl) + _attr('compression', 'compression', bytes([compression]))
    hdr += _attr('dataWindow', 'box2i', struct.pack('<4i', 0, 0, W - 1, H - 1))
    hdr += _attr('displayWindow', 'box2i', struct.pack('<4i', 0, 0, W - 1, H - 1))
    hdr += _attr('lineOrder', 'lineOrder', b'\0') + _attr('pixelAspectRatio', 'float', struct.pack('<f', 1.0))
    hdr += _attr('screenWindowCenter', 'v2f', struct.pack('<ff', 0, 0)) + _attr('screenWindowWidth', 'float', struct.pack('<f', 1.0)) + b'\0'
    lines = {0: 1, 2: 1, 3: 16}[compression]
    chunks = []
    for y in range(0, H, lines):
        raw = b''.join(img[r, :, c].astype(dt).tobytes() for r in range(y, min(y + lines, H)) for c in (2, 1, 0))
        if compression:
            b = np.frombuffer(raw, np.uint8)
            t = np.concatenate([b[0::2], b[1::2]]).astype(np.int64)
            d = t.copy()
            d[1:] = (t[1:] - t[:-1] + 128) & 0xff
            raw = zlib.compress(d.astype(np.uint8).tobytes())
        chunks.append(struct.pack('<ii', y, len(raw)) + raw)
    off = len(hdr) + 8 * len(chunks)
    table = b''
    for c in chunks:
        table += struct.pack('<Q', off)
        off += len(c)
    with open(path, 'wb') as fh:
        fh.write(hdr + table + b''.join(chunks))
    return img.astype(dt).astype(np.float32)


def read_png(path):
    """Minimal PNG decoder for 8-bit RGBA with filter type 0 (what write_png_rgba writes)."""
    data = open(path, 'rb').read()
    assert data[:8] == b'\x89PNG\r\n\x1a\n'
    pos, idat, ihdr = 8, b'', None
    while pos < len(data):
        n, tag = struct.unpack('>I4s', data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        assert struct.unpack('>I', data[pos + 8 + n:pos + 12 + n])[0] == zlib.crc32(tag + body) & 0xffffffff
        if tag == b'IHDR':
            ihdr = struct.unpack('>IIBBBBB', body)
        elif tag == b'IDAT':
            idat += body
        pos += 12 + n
    w, h, depth, ctype = ihdr[:4]
    assert depth == 8 and ctype == 6
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + 4 * w)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(h, w, 4)


def test_relighter_has_no_cpu_path():
    verts = np.zeros((3, 3), np.float32)
    mats = {'metallic': np.zeros((3, 1)), 'roughness': np.ones((3, 1)), 'albedo': np.ones((3, 3))}
    with pytest.raises(RuntimeError):
        RL.Relighter(verts, np.asarray([[0, 1, 2]]), mats, np.ones((2, 4, 3), np.float32), device='cpu')


# ------------------------------------------------------------------------------------------------ export format
def test_save_materials_writes_the_reference_format(tmp_path):
    rng = np.random.RandomState(0)
    V = 257
    mats = {'metallic': rng.rand(V, 1).astype(np.float32), 'roughness': rng.rand(V, 1).astype(np.float32),
            'albedo': rng.rand(V, 3).astype(np.float32)}
    mats['albedo'][:5] = 0.001                      # the linear segment of the transfer
    RL.save_materials(str(tmp_path / 'm'), mats)
    assert sorted(os.listdir(tmp_path / 'm')) == ['albedo.npy', 'metallic.npy', 'roughness.npy']
    for k, shape in (('metallic', (V, 1)), ('roughness', (V, 1)), ('albedo', (V, 3))):
        got = np.load(tmp_path / 'm' / f'{k}.npy')
        assert got.shape == shape and got.dtype == np.float32
        want = O.linear_to_srgb(torch.from_numpy(mats[k])).numpy()
        np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-7)
    back = RL.load_materials(str(tmp_path / 'm'))
    for k in mats:
        np.testing.assert_allclose(back[k], mats[k], rtol=1e-5, atol=1e-6)


# ------------------------------------------------------------------------------------------------ image files
def _test_image(H=9, W=37, seed=1):
    rng = np.random.RandomState(seed)
    img = np.exp(rng.randn(H, W, 3) * 2).astype(np.float32)
    img[:, 5:20] = img[:, 5:6]                     # runs for the run-length coder
    img[2, :] = 0.0
    return img


@pytest.mark.parametrize('rle', [False, True])
def test_hdr_round_trip(tmp_path, rle):
    img = _test_image()
    want = write_hdr(tmp_path / 'a.hdr', img, rle)
    got = RL.load_env_map(str(tmp_path / 'a.hdr'))
    assert got.dtype == np.float32 and got.shape == img.shape
    np.testing.assert_array_equal(got, want)
    assert np.all(np.abs(got - img) <= img.max(-1, keepdims=True) / 128.0)


@pytest.mark.parametrize('compression', [0, 2, 3])
@pytest.mark.parametrize('ptype', [1, 2])
def test_exr_round_trip(tmp_path, compression, ptype):
    img = _test_image(H=21, W=13) * 0.01
    want = write_exr(tmp_path / 'a.exr', img, compression, ptype)
    got = RL.load_env_map(str(tmp_path / 'a.exr'))
    assert got.dtype == np.float32 and got.shape == img.shape
    np.testing.assert_array_equal(got, want)


def test_exr_unsupported_compression_raises(tmp_path):
    write_exr(tmp_path / 'a.exr', _test_image(), 0, 1)
    data = bytearray(open(tmp_path / 'a.exr', 'rb').read())
    i = data.index(b'compression\0compression\0') + len('compression\0compression\0') + 4
    data[i] = 4
    open(tmp_path / 'piz.exr', 'wb').write(bytes(data))
    with pytest.raises(ValueError, match='PIZ'):
        RL.load_env_map(str(tmp_path / 'piz.exr'))


def test_png_round_trip(tmp_path):
    rgba = np.random.RandomState(2).randint(0, 256, (11, 23, 4)).astype(np.uint8)
    RL.write_png_rgba(str(tmp_path / 'a.png'), rgba)
    np.testing.assert_array_equal(read_png(tmp_path / 'a.png'), rgba)
    img = np.zeros((1, 3, 4))
    img[0, 1] = [0.25, 0.5, 0.0, 0.5]             # premultiplied: straight colour (0.5, 1, 0)
    img[0, 2] = [2.0, 0.0, 0.0, 1.0]
    q = RL.to_rgba8(img)
    assert q[0, 0].tolist() == [0, 0, 0, 0]
    assert q[0, 1].tolist() == [round(float(RL.linear_to_srgb(np.float64(0.5))) * 255), 255, 0, 128]
    assert q[0, 2].tolist() == [255, 0, 0, 255]


# ------------------------------------------------------------------------------------------------ cameras
def test_relight_poses_match_the_reference():
    g = load_golden('relight_poses')
    for c in range(3):
        num, az, el, dist = g[f'config{c}']
        np.testing.assert_allclose(RL.relight_poses(int(num), az, el, dist), g[f'poses{c}'], atol=1e-12)
    p = RL.relight_poses(5, 10.0, 30.0, 2.0)
    centre = -np.einsum('nji,nj->ni', p[:, :, :3], p[:, :, 3])
    np.testing.assert_allclose(np.linalg.norm(centre, axis=-1), 2.0)
    np.testing.assert_allclose(centre[:, 2], 2.0 * np.sin(np.deg2rad(30.0)))


def test_blender_default_K():
    K = RL.blender_default_K(800, 800)
    assert abs(K[0, 0] - 1111.1111) < 1e-3 and K[0, 0] == K[1, 1] and K[0, 2] == 400 and K[1, 2] == 400
    K = RL.blender_default_K(600, 900)
    assert abs(K[0, 0] - 1250.0) < 1e-9 and K[0, 2] == 450 and K[1, 2] == 300


# ------------------------------------------------------------------------------------------------ environment sampling
def _smooth_env(H=32, W=64):
    v = (np.arange(H)[::-1] + 0.5) / H            # row 0 at the top
    u = (np.arange(W) + 0.5) / W
    d, _ = OR.env_dir(u[None, :], v[:, None])
    base = 0.3 + np.maximum(d[..., 2], 0) + 2.0 * np.exp(-8 * np.sum((d - np.asarray([0.6, 0.0, 0.8])) ** 2, -1))
    return np.stack([base, base * 0.8 + 0.1, base * 0.6 + 0.2 * d[..., 0] ** 2], -1).astype(np.float32)


def test_env_pdf_integrates_to_one():
    tab = RL.env_tables(_smooth_env())
    n = 1024
    u, v = np.meshgrid((np.arange(2 * n) + 0.5) / (2 * n), (np.arange(n) + 0.5) / n)
    d, ce = OR.env_dir(u.reshape(-1), v.reshape(-1))
    _, pdf = OR.env_lookup_pdf(tab, d)
    total = np.sum(pdf * ce) * (2 * np.pi / (2 * n)) * (np.pi / n)
    assert abs(total - 1.0) < 1e-4, total
    assert abs(tab['p'].astype(np.float64).sum() - 1.0) < 1e-5
    assert tab['cdf_rows'][0] == 0 and tab['cdf_rows'][-1] == 1 and (tab['cdf_cols'][:, -1] == 1).all()


def test_env_sampler_chi_square():
    from scipy.stats import chi2
    tab = RL.env_tables(_smooth_env(8, 16))
    N = 10 ** 6
    r = np.stack([OR.uniform(5, np.arange(N), 0, 0, k) for k in (2, 3, 4, 5)], -1)
    d, tx, pdf = OR.sample_env(tab, r)
    np.testing.assert_array_equal(tx, OR.env_lookup_pdf(tab, d)[0])   # sampled directions fall in the chosen texel
    counts = np.bincount(tx, minlength=tab['p'].size)
    exp = tab['p'].reshape(-1).astype(np.float64) * N
    keep = exp >= 5
    stat = np.sum((counts[keep] - exp[keep]) ** 2 / exp[keep])
    assert chi2.sf(stat, keep.sum() - 1) > 1e-3, stat


def test_one_hot_map_round_trip():
    H, W = 8, 16
    for j, i in [(0, 0), (3, 5), (7, 15), (4, 8)]:
        env = np.zeros((H, W, 3), np.float32)
        env[j, i] = 1.0
        tab = RL.env_tables(env)
        row_from_bottom = H - 1 - j
        assert tab['p'].reshape(-1)[row_from_bottom * W + i] == 1.0
        r = np.stack([OR.uniform(1, np.arange(1000), 0, 0, k) for k in (2, 3, 4, 5)], -1)
        d, tx, _ = OR.sample_env(tab, r)
        assert (tx == row_from_bottom * W + i).all()
        u, v = OR.env_uv(d)
        assert ((u * W).astype(int) == i).all() and ((v * H).astype(int) == row_from_bottom).all()
    # the mapping itself: +x at u = 0.5, +y at u = 0.25, up at v = 1
    u, v = OR.env_uv(np.asarray([[1.0, 0, 0], [0, 1.0, 0], [0, 0, 1.0]]))
    np.testing.assert_allclose(u[:2], [0.5, 0.25])
    np.testing.assert_allclose(v, [0.5, 0.5, 1.0])


# ------------------------------------------------------------------------------------------------ host-compiled kernel math
@pytest.fixture(scope='module')
def hc():
    src = os.path.join(HERE, 'hostcheck', 'hostcheck_relight.cu')
    so = os.path.join(HERE, 'hostcheck', 'libhostcheck_relight.so')
    deps = [src] + [os.path.join(HERE, '..', 'nero_b200', 'csrc', f) for f in ('math_relight.cuh', 'math_mc.cuh', 'common.cuh')]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        subprocess.check_call(['/usr/local/cuda/bin/nvcc', '-O2', '-std=c++17', '-Xcompiler', '-fPIC', '-shared', '--fmad=false',
                               '-Wno-deprecated-gpu-targets', '-o', so, src])
    return ctypes.CDLL(so)


def P(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def f32(a):
    return np.ascontiguousarray(a, np.float32)


def i32(a):
    return np.ascontiguousarray(a, np.int32)


def test_hostcheck_rng_and_search_are_bit_identical(hc):
    rng = np.random.RandomState(3)
    n = 5000
    pix, smp, bnc, dim = rng.randint(0, 2 ** 31 - 1, n), rng.randint(0, 1 << 20, n), rng.randint(0, 8, n), rng.randint(0, 9, n)
    out = np.zeros(n, np.float32)
    hc.hc_rl_uniform(n, ctypes.c_uint(123456789), P(i32(pix)), P(i32(smp)), P(i32(bnc)), P(i32(dim)), P(out))
    want = OR.uniform(123456789, pix, smp, bnc, dim)
    np.testing.assert_array_equal(out.astype(np.float64), want)
    assert 0.49 < want.mean() < 0.51 and want.min() >= 0 and want.max() < 1
    tab = RL.env_tables(_smooth_env())
    env = np.zeros((8, 16, 3), np.float32)
    env[2, 3] = 1.0
    env[6, 9:12] = 2.0                             # zero-probability bins everywhere else
    for cdf in (tab['cdf_rows'], tab['cdf_cols'][7], RL.env_tables(env)['cdf_rows'], RL.env_tables(env)['cdf_cols'][1]):
        u = np.concatenate([want[:2000], cdf[:-1], np.nextafter(cdf[1:-1], 0, dtype=np.float32)]).astype(np.float32)
        u = u[u < 1]
        got = np.zeros(u.size, np.int32)
        hc.hc_rl_search(P(f32(cdf)), cdf.size - 1, u.size, P(f32(u)), P(got))
        np.testing.assert_array_equal(got, OR.search(cdf, u.astype(np.float64)))
        assert (cdf[got] < cdf[got + 1]).all()     # never an empty bin


def test_hostcheck_env_mapping(hc):
    rng = np.random.RandomState(4)
    n, W, H = 3000, 64, 32
    u, v = f32(rng.rand(n)), f32(rng.rand(n) * 0.98 + 0.01)
    d, ce, uv, tx = np.zeros((n, 3), np.float32), np.zeros(n, np.float32), np.zeros((n, 2), np.float32), np.zeros(n, np.int32)
    hc.hc_rl_env(n, P(u), P(v), W, H, P(d), P(ce), P(uv), P(tx))
    dw, cw = OR.env_dir(u.astype(np.float64), v.astype(np.float64))
    np.testing.assert_allclose(d, dw, atol=2e-6)
    np.testing.assert_allclose(ce, cw, atol=2e-6)
    np.testing.assert_allclose(uv, np.stack([u, v], -1), atol=3e-6)
    uo, vo = OR.env_uv(d.astype(np.float64))
    np.testing.assert_allclose(uv, np.stack([uo, vo], -1), atol=1e-6)
    inner = (np.abs(u * W - np.round(u * W)) > 1e-3) & (np.abs(v * H - np.round(v * H)) > 1e-3)
    np.testing.assert_array_equal(tx[inner], OR.texel(u.astype(np.float64), v.astype(np.float64), W, H)[inner])


def _surface_cases(n, seed):
    rng = np.random.RandomState(seed)
    nrm = OR.normalize(rng.randn(n, 3))
    view = OR.normalize(nrm + 0.9 * OR.normalize(rng.randn(n, 3)))
    view = np.where((OR.dot(view, nrm) < 0.05)[:, None], nrm, view)
    albedo = rng.rand(n, 3)
    metallic = rng.rand(n)
    metallic[:50], metallic[50:100], albedo[100:110] = 0.0, 1.0, 0.0
    alpha = (0.05 + 0.95 * rng.rand(n)) ** 2
    return f32(nrm), f32(view), f32(albedo), f32(metallic), f32(alpha)


def test_hostcheck_lobe_sampling_and_pdf(hc):
    n = 2000
    nrm, view, albedo, metallic, alpha = _surface_cases(n, 5)
    ps = np.zeros(n, np.float32)
    hc.hc_rl_lobe(n, P(albedo), P(metallic), P(ps))
    want = OR.spec_prob(albedo.astype(np.float64), metallic.astype(np.float64))
    np.testing.assert_allclose(ps, want, rtol=2e-6)
    assert (ps[metallic == 1.0] == 1.0).all() and (ps[(metallic < 1) & (albedo.sum(-1) > 0)] < 1).all() and (ps >= 0.25).all()
    r1, r2 = f32(OR.uniform(9, np.arange(n), 0, 0, 7)), f32(OR.uniform(9, np.arange(n), 0, 0, 8))
    spec = i32(np.arange(n) % 2)
    l, pdf = np.zeros((n, 3), np.float32), np.zeros(n, np.float32)
    hc.hc_rl_sample(n, P(nrm), P(view), P(alpha), P(r1), P(r2), P(spec), P(ps), P(l), P(pdf))
    N64, V64, A64 = nrm.astype(np.float64), view.astype(np.float64), alpha.astype(np.float64)
    lw = OR.normalize(np.where(spec[:, None] == 1, OR.sample_ggx(N64, V64, A64, r1.astype(np.float64), r2.astype(np.float64)),
                               OR.sample_diffuse(N64, r1.astype(np.float64), r2.astype(np.float64))))
    np.testing.assert_allclose(l, lw, atol=5e-4)     # fp32 sqrt(1 - cos^2) near the GGX peak
    assert np.mean(np.abs(l - lw).max(-1) < 1e-5) > 0.95
    pw = OR.bsdf_pdf(N64, V64, l.astype(np.float64), A64, ps.astype(np.float64))
    ok = pw > 0
    # below alpha ~ 0.03 the fp32 1 - NoH^2 of a peaked GGX lobe carries percent-level error (the rounding of NoH near 1)
    broad = ok & (alpha >= 0.03)
    np.testing.assert_allclose(pdf[broad], pw[broad], rtol=1e-3)
    np.testing.assert_allclose(pdf[ok], pw[ok], rtol=0.1)
    assert (pdf[~ok] == 0).all()


@pytest.mark.parametrize('ggx', [0, 1])
def test_hostcheck_brdf(hc, ggx):
    n = 2000
    nrm, view, albedo, metallic, alpha = _surface_cases(n, 6)
    l = f32(OR.normalize(OR.normalize(np.random.RandomState(7).randn(n, 3)) + nrm))
    f = np.zeros((n, 3), np.float32)
    hc.hc_rl_brdf(n, P(nrm), P(view), P(l), P(albedo), P(metallic), P(alpha), ggx, P(f))
    want = OR.brdf(*(a.astype(np.float64) for a in (nrm, view, l, albedo, metallic, alpha)), ggx)
    np.testing.assert_allclose(f, want, rtol=2e-3, atol=1e-6)
    # the terms equal NeRO's (oracle) distribution_ggx and geometry_term
    import nero_oracle_mat as OM
    h = OR.normalize(view.astype(np.float64) + l)
    NoH = torch.from_numpy(np.clip(OR.dot(nrm.astype(np.float64), h), 0, 1))
    D = OM.distribution_ggx(NoH, torch.from_numpy(alpha.astype(np.float64))).numpy()
    a2 = alpha.astype(np.float64) ** 2
    np.testing.assert_allclose(D, a2 / (np.pi * (NoH.numpy() ** 2 * (a2 - 1) + 1) ** 2 + 1e-4), rtol=1e-12)


# ------------------------------------------------------------------------------------------------ unbiased estimator
@pytest.mark.parametrize('case', ['diffuse', 'rough_metal', 'glossy_dielectric'])
def test_direct_light_estimator_is_unbiased(case):
    albedo, metallic, rough = {'diffuse': ((0.7, 0.5, 0.3), 0.0, 0.9), 'rough_metal': ((0.9, 0.6, 0.3), 1.0, 0.6),
                               'glossy_dielectric': ((0.2, 0.3, 0.5), 0.0, 0.3)}[case]
    env = _smooth_env(32, 64)
    tab = RL.env_tables(env)
    n = OR.normalize(np.asarray([0.3, -0.2, 0.9]))
    v = OR.normalize(np.asarray([-0.4, 0.5, 0.6]))
    alpha = rough ** 2
    N = 1 << 16
    rep = lambda a: np.broadcast_to(np.asarray(a, np.float64), (N,) + np.shape(a)).copy()
    rnd = lambda dim: OR.uniform(77, np.arange(N), 0, 0, dim)
    L, _, _, _, _ = OR.shade(rep(n), rep(v), rep(albedo), rep(metallic), rep(alpha), tab, 0, rnd,
                             lambda mask, l: np.zeros(N, bool), lambda mask, l: (np.zeros(N, bool), None))
    # quadrature of the integral of L f cos over the sphere, with the same piecewise-constant map
    qh = 1024
    u, vv = np.meshgrid((np.arange(2 * qh) + 0.5) / (2 * qh), (np.arange(qh) + 0.5) / qh)
    d, ce = OR.env_dir(u.reshape(-1), vv.reshape(-1))
    tx, _ = OR.env_lookup_pdf(tab, d)
    Le = tab['env'].reshape(-1, 4)[tx, :3].astype(np.float64)
    M = d.shape[0]
    f = OR.brdf(np.broadcast_to(n, (M, 3)), np.broadcast_to(v, (M, 3)), d, np.broadcast_to(np.asarray(albedo), (M, 3)),
                np.full(M, metallic), np.full(M, alpha), 0)
    cos = np.maximum(OR.dot(d, n), 0)
    ref = np.sum(Le * f * (cos * ce)[:, None], 0) * (2 * np.pi / (2 * qh)) * (np.pi / qh)
    mean, se = L.mean(0), L.std(0) / np.sqrt(N)
    assert (np.abs(mean - ref) < 3 * se + 1e-4 * ref).all(), (mean, ref, se)
