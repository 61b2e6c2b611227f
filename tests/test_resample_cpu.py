"""The coefficient tables of the device resampler (style_transfer.resample_coeffs) against the installed Pillow, without
a GPU: the two fixed-point passes restated in numpy and driven by the product's tables must give
`Image.resize((w, h), Image.BICUBIC)` exactly.  This pins the double arithmetic of the weights (the order of the sum and
the division decide their last bit) and the window bounds where they can be debugged; the kernels that run the same two
passes on the device are held against Pillow in test_gpu_resample.py."""
import re
from pathlib import Path

import numpy as np
import pytest
from PIL import Image

from style_transfer_b200 import _lib
from style_transfer_b200.style_transfer import resample_coeffs

ROOT = Path(__file__).resolve().parent.parent

# (source w, h) -> (w, h)
GRID = [
    ((1500, 900), (16, 16)),       # strong reduction: 375 taps per output
    ((1000, 700), (707, 495)),     # mild reduction
    ((64, 48), (64, 48)),          # identity: copied
    ((300, 200), (300, 77)),       # the height only
    ((300, 200), (111, 200)),      # the width only
    ((16, 16), (128, 128)),        # enlargement: 5 taps, windows cut at both edges
    ((181, 136), (256, 192)),
    ((1, 50), (7, 20)),            # 1-pixel axes, source and result
    ((50, 1), (20, 7)),
    ((1500, 3), (1, 1)),
    ((997, 13), (101, 31)),        # primes
    ((900, 700), (128, 100)),      # the sizes a default pyramid asks for
    ((777, 1100), (90, 128)),
    ((33, 77), (33, 200)),
]


def saturating_image(w, h, seed):
    """Noise with flat 0 and 255 regions side by side: next to such an edge the negative lobes of the bicubic kernel
    drive the accumulator below 0 and above 255, so the clamp of either pass acts."""
    a = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
    a[:h // 2, :w // 2] = 0
    a[:h // 2, w // 2:w // 2 + max(w // 8, 1)] = 255
    a[h // 2:h // 2 + max(h // 8, 1), :w // 3] = 255
    return a


def one_pass(a, k, bounds):
    """A fixed-point pass along axis 1 of a [rows][samples][3] uint8 array."""
    out = np.empty((a.shape[0], k.shape[0], 3), np.uint8)
    for x, (first, count) in enumerate(bounds):
        acc = (a[:, first:first + count].astype(np.int64) * k[x, :count, None]).sum(axis=1) + (1 << 21)
        assert np.abs(acc).max() < 2 ** 31          # the device accumulates in int32
        out[:, x] = np.clip(acc >> 22, 0, 255)
    return out


def two_passes(a, w, h):
    hs, ws, _ = a.shape
    if ws != w:
        a = one_pass(a, *resample_coeffs(ws, w))
    if hs != h:
        a = one_pass(a.transpose(1, 0, 2), *resample_coeffs(hs, h)).transpose(1, 0, 2)
    return a


@pytest.mark.parametrize('src,dst', GRID)
def test_tables_reproduce_pillow_bicubic(src, dst):
    a = saturating_image(*src, seed=src[0] * 7 + dst[1])
    ref = np.asarray(Image.fromarray(a).resize(dst, Image.BICUBIC))
    got = two_passes(a, *dst)
    assert got.shape == ref.shape
    assert np.array_equal(got, ref), f'{int((got != ref).sum())} samples differ'


def test_tables_reproduce_pillow_on_random_sizes():
    rng = np.random.default_rng(5)
    for _ in range(25):
        ws, hs, w, h = (int(v) for v in rng.integers(1, 400, 4))
        a = saturating_image(ws, hs, seed=ws + h)
        assert np.array_equal(two_passes(a, w, h), np.asarray(Image.fromarray(a).resize((w, h), Image.BICUBIC))), \
            (ws, hs, w, h)


@pytest.mark.parametrize('n_in,n_out', [(6000, 128), (4000, 2731), (16, 128), (1, 9), (9, 1)])
def test_table_shapes_and_bounds(n_in, n_out):
    k, bounds = resample_coeffs(n_in, n_out)
    ksize = 2 * int(np.ceil(2.0 * max(n_in / n_out, 1.0))) + 1
    assert k.dtype == np.int32 and bounds.dtype == np.int32
    assert k.shape == (n_out, ksize) and bounds.shape == (n_out, 2)
    first, count = bounds[:, 0], bounds[:, 1]
    assert (first >= 0).all() and (count >= 1).all() and (count <= ksize).all() and (first + count <= n_in).all()
    # the row window of a band relies on this: the first and the last row of a window bound the source rows it reads
    assert (np.diff(first) >= 0).all() and (np.diff(first + count) >= 0).all()
    assert (k[np.arange(ksize)[None, :] >= count[:, None]] == 0).all()
    assert np.abs(k.sum(axis=1) - (1 << 22)).max() <= ksize       # weights sum to one, up to their rounding


def test_resample_entry_points_are_declared_everywhere():
    header = (ROOT / 'include' / 'stb200.h').read_text()
    for name in ('stb_resample_rgb8', 'stb_resample_tmp_bytes'):
        assert re.search(rf'STB_API int {name}\(', header)
        assert name in _lib.EXPORTS
