"""CPU: the image-metric oracle (oracle/nero_oracle_metrics.py) against scipy and the reference's compute_psnr
(tests/golden/metrics_reference.npz), the montage layout, the bindings of include/nero_metrics.h, the refusals that need no
GPU, the kernels' register use and the argument handling of tools/eval_synthetic_nvs.py.  No GPU."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

import make_golden_metrics as G
import nero_oracle_metrics as OM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, 'tests', 'golden', 'metrics_reference.npz')


@pytest.mark.parametrize('shape', [(11, 11), (12, 200), (37, 53)])
def test_explicit_recurrence_is_scipy_uniform_filter(shape):
    rng = np.random.RandomState(shape[0] * 1000 + shape[1])
    x = rng.randint(0, 256, shape).astype(np.float64)
    y = rng.randint(0, 256, shape).astype(np.float64)
    for plane in (x, y, x * x, y * y, x * y):
        assert np.array_equal(OM.uniform_filter_explicit(plane, 11), ndi.uniform_filter(plane, 11))
    for axis in (0, 1):
        assert np.array_equal(OM.uniform_filter1d_explicit(x * y, 11, axis), ndi.uniform_filter1d(x * y, 11, axis))


def test_oracle_ssim_identity_symmetry_and_refusals():
    rng = np.random.RandomState(3)
    a = rng.randint(0, 256, (23, 31, 3)).astype(np.uint8)
    b = np.clip(a.astype(int) + rng.randint(-30, 31, a.shape), 0, 255).astype(np.uint8)
    assert OM.ssim(a, a) == 1.0
    smap, chan = OM.ssim_map(a, a)
    assert (smap == 1.0).all() and (chan == 1.0).all()
    assert OM.ssim(a, b) == OM.ssim(b, a) and 0 < OM.ssim(a, b) < 1
    assert np.array_equal(OM.ssim_map(a, b)[0], OM.ssim_map(b, a)[0])
    for bad in ((a[:10], b[:10]), (a[:, :10], b[:, :10])):
        with pytest.raises(ValueError):
            OM.ssim(*bad)
    with pytest.raises(ValueError):
        OM.ssim(a, b, win_size=10)
    with pytest.raises(ValueError):
        OM.ssim(a, b[:-1])


def test_oracle_quantisation_matches_the_reference():
    g = np.load(GOLD)
    assert np.array_equal(OM.color_map_backward(g['quant_in']), g['quant_out'])
    k = np.arange(256, dtype=np.uint8)
    assert np.array_equal(OM.color_map_backward(k.astype(np.float32) / 255), k)     # color_map_forward round trip


def test_reference_psnr_and_the_exact_psnr():
    g = np.load(GOLD)
    for p, ref in zip(g['pairs'], g['psnr_reference']):
        gt, pr = G.image_pair(*p)
        assert OM.psnr_reference(gt, pr) == ref
        exact = OM.psnr_exact(gt, pr)
        # the reference's float32 sums lose squared error, so its PSNR is higher; by at most 0.02 dB at 800^2
        assert -1e-5 <= float(ref) - exact <= 0.02, (p, ref, exact)
        if p[1] * p[2] * 255 ** 2 < 1 << 24:       # every partial sum exact in float32: only the final rounding differs
            assert abs(float(ref) - exact) <= 1e-5
    gt, _ = G.image_pair(1, 48, 64, 20)
    assert OM.psnr_exact(gt, gt) == np.inf


def test_montage_layout():
    from nero_b200 import metrics as M
    rng = np.random.RandomState(5)
    imgs = [rng.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((4, 6), (7, 3), (2, 5), (7, 6))]
    for vert in (False, True):
        mine = M.concat_images_list(*[torch.from_numpy(i) for i in imgs], vert=vert).numpy()
        assert np.array_equal(mine, OM.concat_images_list(*imgs, vert=vert))
    # cv2.copyMakeBorder, which the reference pads with, agrees with the oracle's np.pad
    import cv2
    a, b = imgs[0], imgs[1]
    ref = np.concatenate([cv2.copyMakeBorder(a, 0, 3, 0, 0, borderType=cv2.BORDER_CONSTANT, value=0), b], axis=1)
    assert np.array_equal(ref, OM.concat_images(a, b))


def test_metrics_header_bindings():
    from nero_b200 import ops
    assert set(ops.METRICS_PROTOS) == {'nero_metrics_quantize', 'nero_metrics_sse', 'nero_metrics_ssim'}
    for name, argtypes in ops.METRICS_PROTOS.items():
        assert getattr(ops.lib, name).argtypes == argtypes
    assert [len(ops.METRICS_PROTOS[n]) for n in ('nero_metrics_quantize', 'nero_metrics_sse', 'nero_metrics_ssim')] == [4, 8, 14]


def test_cpu_tensors_are_refused():
    from nero_b200 import metrics as M
    a = torch.zeros(16, 16, 3, dtype=torch.uint8)
    for f in (M.psnr, M.ssim):
        with pytest.raises(RuntimeError, match='CUDA'):
            f(a, a)
    with pytest.raises(RuntimeError, match='CUDA'):
        M.color_map_backward(torch.zeros(4))
    with pytest.raises(TypeError):
        M.psnr(a.numpy(), a.numpy())


def test_metrics_kernels_do_not_spill():
    out = subprocess.run(['/usr/local/cuda/bin/nvcc', '-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-std=c++17',
                          '--expt-relaxed-constexpr', '-Xptxas', '-v', '-c', os.path.join(ROOT, 'nero_b200', 'csrc', 'k_metrics.cu'),
                          '-o', os.devnull], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    blocks = re.findall(r'Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads',
                        out.stderr)
    names = ('quantize_kernel', 'sse_kernel', 'ssim_cols_kernel', 'ssim_rows_kernel', 'ssim_finish_kernel')
    assert sorted(n for n in names if any(n in b[0] for b in blocks)) == sorted(names)
    for name, stack, stores, loads in blocks:
        assert (stack, stores, loads) == ('0', '0', '0'), name


# ------------------------------------------------------------------------------------------------ the tool
def tool():
    sys.path.insert(0, os.path.join(ROOT, 'tools'))
    import eval_synthetic_nvs
    return eval_synthetic_nvs


def test_tool_arguments_and_refusals(tmp_path):
    t = tool()
    assert t.parse(['--cfg', 'x.yaml']).ids is None
    assert t.parse(['--cfg', 'x.yaml', '--ids', '3', '7']).ids == ['3', '7']
    p = tmp_path / 'c.yaml'
    for body, match in (('name: a\nnetwork: nerf\ndatabase_name: syn/bell\n', 'shape or a material'),
                        ('name: a\nnetwork: shape\ndatabase_name: real/bear/raw_1024\n', 'GlossySynthetic'),
                        ('name: a\nnetwork: material\ndatabase_name: custom/obj/raw_1024\n', 'GlossySynthetic'),
                        ('name: a\nnetwork: shape\n', 'GlossySynthetic')):
        p.write_text(body)
        with pytest.raises(SystemExit, match=match):
            t.main(['--cfg', str(p)])
    p.write_text('name: a\nnetwork: material\ndatabase_name: syn/bell\n')
    assert t.load_cfg(str(p))['database_name'] == 'syn/bell'


def test_gt_image_reader(tmp_path):
    import cv2
    from nero_b200 import evaluate as E
    rng = np.random.RandomState(9)
    rgba = rng.randint(0, 256, (5, 7, 4)).astype(np.uint8)
    cv2.imwrite(str(tmp_path / '0.png'), rgba[..., [2, 1, 0, 3]])
    cv2.imwrite(str(tmp_path / '1.png'), rgba[..., 2::-1])
    for i in ('0', '1'):
        assert np.array_equal(E.read_gt_image(str(tmp_path), i), rgba[..., :3])
    cv2.imwrite(str(tmp_path / '2.png'), rgba[..., :3].astype(np.uint16) * 257)
    with pytest.raises(ValueError):
        E.read_gt_image(str(tmp_path), '2')
