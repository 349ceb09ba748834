"""Generate tests/golden/metrics_reference.npz by running the UNMODIFIED reference's compute_psnr (network/metrics.py:11-17) and
color_map_backward (utils/base_utils.py:453-456) through oracle/ref_shim.py (skimage is stubbed there).

The image pairs are not stored: they are regenerated from their seeds by `image_pair` (numpy's RandomState is stable across
versions), so the fixture holds only the seeds, the sizes and the reference's outputs.

    python oracle/make_golden_metrics.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), 'tests', 'golden', 'metrics_reference.npz')

# (seed, h, w, noise): small images, and 800^2 ones where numpy's float32 sums pass 2^24
PAIRS = [(1, 48, 64, 20), (2, 37, 53, 3), (3, 800, 800, 3), (4, 800, 800, 9), (5, 800, 800, 18)]


def image_pair(seed, h, w, noise):
    """A uint8 [h,w,3] image and a copy with uniform integer noise in [-noise, noise], clipped to [0, 255]."""
    rng = np.random.RandomState(seed)
    gt = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
    pr = np.clip(gt.astype(np.int64) + rng.randint(-noise, noise + 1, (h, w, 3)), 0, 255).astype(np.uint8)
    return gt, pr


def quant_inputs():
    """float32 values for color_map_backward: k/255, NaN, +-inf, out of range and values just below integers."""
    k = np.arange(256, dtype=np.float32) / np.float32(255)
    special = np.asarray([np.nan, np.inf, -np.inf, -1e30, -1.0, -1e-7, 1.0000001, 2.0, 1e30, 0.5, 0.99999994,
                          np.nextafter(np.float32(1 / 255), np.float32(0))], np.float32)
    rng = np.random.RandomState(7)
    return np.concatenate([k, special, rng.uniform(-0.2, 1.2, 4096).astype(np.float32)])


def main():
    sys.path.insert(0, HERE)
    import ref_shim
    ref_shim.install()
    # utils/draw_utils.py needs matplotlib, which the shim stubs without its submodules; only its montage helper is imported
    # by network/metrics.py, and the montage is not part of this fixture
    import types
    sys.modules['utils.draw_utils'] = types.SimpleNamespace(concat_images_list=None)
    from network.metrics import compute_psnr
    from utils.base_utils import color_map_backward
    x = quant_inputs()
    with np.errstate(invalid='ignore'):
        q = color_map_backward(x)
    psnrs = [compute_psnr(*image_pair(*p)) for p in PAIRS]
    assert all(isinstance(v, np.float32) for v in psnrs)
    np.savez_compressed(OUT, pairs=np.asarray(PAIRS, np.int64), psnr_reference=np.asarray(psnrs, np.float32), quant_in=x,
                        quant_out=q)
    print(OUT, psnrs)


if __name__ == '__main__':
    main()
