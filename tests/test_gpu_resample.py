"""-m gpu: the source images on the device (stb_resample_rgb8, style_transfer.SourceImage).

Every tensor stylize() makes from the content and style images must be, bit for bit, what
`_pil_to_tensor(img.resize((w, h), Image.BICUBIC), device)` makes: whole, and per row window of a band.  The kernels
are held against the installed Pillow here; the tables they are driven by are held against it without a GPU in
test_resample_cpu.py."""
import contextlib
import ctypes
import io

import numpy as np
import pytest
import torch
from PIL import Image

import style_transfer_b200 as stb
from style_transfer_b200 import _lib
from style_transfer_b200 import distributed as D
from style_transfer_b200 import style_transfer as ST
from oracle import st_oracle as O
from test_resample_cpu import GRID, saturating_image

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
SAME_GPU = ['cuda:0', 'cuda:0']

PRODUCTION = [
    ((4000, 3000), (128, 96)),       # a camera photo at the scales of a pyramid
    ((4000, 3000), (512, 384)),
    ((4000, 3000), (2048, 1536)),
    ((1024, 1024), (4096, 4096)),    # a small content image brought up to the scale
    ((4000, 6), (16, 6)),            # 250 : 1, the span of a tile's outputs is read from global memory
    ((4001, 7), (16, 3)),
]


def pil_tensor(img, w, h):
    return ST._pil_to_tensor(img.resize((w, h), Image.BICUBIC), DEV)


def pil_resized(self, w, h, row0=0, rows=None):
    """SourceImage.resized as stylize() computed it before: resize on the host, upload, convert, cut the rows."""
    rows = h - row0 if rows is None else rows
    return pil_tensor(self.img, w, h)[:, :, row0:row0 + rows].contiguous()


@pytest.mark.parametrize('src,dst', GRID + PRODUCTION)
def test_resized_equals_pillow_bit_for_bit(src, dst):
    img = Image.fromarray(saturating_image(*src, seed=src[1] + dst[0]))
    got = ST.SourceImage(img, DEV).resized(*dst)
    ref = pil_tensor(img, *dst)
    assert got.shape == ref.shape == (1, 3, dst[1], dst[0]) and got.dtype == torch.float32 and got.is_contiguous()
    assert torch.equal(got, ref), f'{int((got != ref).sum())} of {ref.numel()} values differ'


def test_every_byte_value_converts_as_torch_does():
    a = np.arange(256, dtype=np.uint8).repeat(3).reshape(1, 256, 3)
    img = Image.fromarray(a)
    for w, h in ((256, 1), (256, 2), (512, 1)):    # copied; the vertical kernel alone; both
        got = ST.SourceImage(img, DEV).resized(w, h)
        assert torch.equal(got, pil_tensor(img, w, h))
    assert set(ST.SourceImage(img, DEV).resized(256, 1).mul(255).round().flatten().tolist()) == set(range(256))


@pytest.mark.parametrize('src,dst', [((900, 700), (288, 384)), ((300, 2000), (300, 640)), ((200, 150), (640, 480)),
                                     ((640, 480), (640, 480)), ((4000, 3000), (512, 384))])
def test_row_windows_equal_slices_of_the_whole(src, dst):
    img = Image.fromarray(saturating_image(*src, seed=3))
    holder = ST.SourceImage(img, DEV)
    w, h = dst
    full = pil_tensor(img, w, h)
    windows = [(0, 1), (h - 1, 1), (0, h), (h // 3, 1), (5, h - 9), (h // 2 - 7, 31)]
    for world in (2, 3):
        for rank in range(world):
            band = D.make_band(h, rank, world)
            assert band is not None
            windows.append((band.loc_begin, band.h_local))
    for row0, rows in windows:
        got = holder.resized(w, h, row0, rows)
        assert got.shape == (1, 3, rows, w)
        assert torch.equal(got, full[:, :, row0:row0 + rows]), (row0, rows)
    band = D.make_band(h, 1, 2)
    assert torch.equal(holder.resized(w, h, band.loc_begin, band.h_local), D.local_slice(full, band))


def test_other_modes_keep_the_host_path():
    a = saturating_image(333, 222, seed=9)
    for img in (Image.fromarray(a).convert('L'), Image.fromarray(np.dstack([a, a[:, :, :1]])),
                Image.fromarray(a).convert('P')):
        holder = ST.SourceImage(img, DEV)
        assert holder.data is None
        assert torch.equal(holder.resized(100, 64), pil_tensor(img, 100, 64))
        assert torch.equal(holder.resized(100, 64, 10, 20), pil_tensor(img, 100, 64)[:, :, 10:30])


def test_argument_errors_launch_nothing():
    lib = _lib.load()
    hs, ws, ho, wo = 40, 60, 20, 30
    holder = ST.SourceImage(Image.fromarray(saturating_image(ws, hs, seed=1)), DEV)
    tabs = [torch.from_numpy(t).to(DEV) for axis in ((ws, wo), (hs, ho)) for t in ST.resample_coeffs(*axis)]
    ks = [tabs[0].shape[1], tabs[2].shape[1]]
    need = ctypes.c_size_t()
    _lib.check(lib.stb_resample_tmp_bytes(hs, ws, ho, wo, 0, ho, ctypes.byref(need)))
    assert need.value == hs * wo * 3
    _lib.check(lib.stb_resample_tmp_bytes(hs, wo, ho, wo, 0, ho, ctypes.byref(need)))
    assert need.value == 0                                   # a kept width needs no scratch
    _lib.check(lib.stb_resample_tmp_bytes(hs, ws, ho, wo, 3, 2, ctypes.byref(need)))
    assert 0 < need.value < hs * wo * 3                      # a window costs the source rows it reads only
    _lib.check(lib.stb_resample_tmp_bytes(hs, ws, ho, wo, 0, ho, ctypes.byref(need)))
    tmp = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    out = torch.full((1, 3, ho, wo), float('nan'), device=DEV)

    def call(src=holder.data, size=(hs, ws, ho, wo), window=(0, ho), kx=tabs[0], bx=tabs[1], ky=tabs[2], by=tabs[3],
             scratch=tmp, scratch_bytes=None, dst=out):
        return lib.stb_resample_rgb8(_lib.ptr(src), *size, *window, _lib.ptr(kx), _lib.ptr(bx), ks[0], _lib.ptr(ky),
                                     _lib.ptr(by), ks[1], _lib.ptr(scratch),
                                     need.value if scratch_bytes is None else scratch_bytes, _lib.ptr(dst),
                                     _lib.cur_stream())

    bad = [dict(src=None), dict(dst=None), dict(kx=None), dict(by=None), dict(scratch=None),
           dict(scratch_bytes=need.value - 1), dict(size=(hs, 0, ho, wo)), dict(size=(hs, ws, 0, wo)),
           dict(window=(-1, 2)), dict(window=(0, 0)), dict(window=(ho - 1, 2)), dict(window=(ho, 1))]
    for kw in bad:
        with pytest.raises(ValueError, match='resample'):
            _lib.check(call(**kw))
    for window in ((-1, 2), (ho, 1), (0, ho + 1)):
        with pytest.raises(ValueError, match='resample'):
            _lib.check(lib.stb_resample_tmp_bytes(hs, ws, ho, wo, *window, ctypes.byref(need)))
    torch.cuda.synchronize()
    assert torch.isnan(out).all()                            # none of the refused calls wrote a value
    _lib.check(call())
    assert torch.equal(out, pil_tensor(holder.img, wo, ho))


def test_a_band_never_holds_the_full_height_tensor():
    """A tall, narrow scale on two ranks: the content step of a band allocates its own rows (and the source rows they
    read, as uint8), not the [1,3,H,W] fp32 tensor that used to be formed and then sliced."""
    w, h = 512, 8192
    holder = ST.SourceImage(Image.fromarray(saturating_image(256, 4096, seed=4)), DEV)
    band = D.make_band(h, 0, 2)
    full_bytes = 3 * h * w * 4
    holder.resized(w, h, band.loc_begin, band.h_local)        # first use loads the kernels
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(DEV)
    base = torch.cuda.memory_allocated(DEV)
    local = holder.resized(w, h, band.loc_begin, band.h_local)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(DEV) - base
    assert local.shape == (1, 3, band.h_local, w)
    assert local.numel() * 4 <= peak < full_bytes, (peak, full_bytes)
    assert peak < 0.65 * full_bytes


# ------------------------------------------------------------------------------------------------ end to end
def _stylize(devices, wts, content, style, kw):
    st = stb.StyleTransfer(devices=devices, pooling='max', vgg_weights=wts,
                           **({'distributed': False} if len(devices) == 1 else {}))
    trace = []
    with contextlib.redirect_stdout(io.StringIO()):
        img = st.stylize(content, [style], callback=lambda it: trace.append((it.w, it.h, it.loss)), **kw)
    return trace, st.average.get().clone(), np.asarray(img)


def _no_host_resize(monkeypatch):
    def refuse(self, *a, **k):
        raise AssertionError('Image.resize called inside stylize()')
    monkeypatch.setattr(Image.Image, 'resize', refuse)


def _spy_windows(monkeypatch):
    """Record (h, rows) of every SourceImage.resized call of the device path."""
    seen, inner = [], ST.SourceImage.resized

    def resized(self, w, h, row0=0, rows=None):
        seen.append((h, h - row0 if rows is None else rows))
        return inner(self, w, h, row0, rows)
    monkeypatch.setattr(ST.SourceImage, 'resized', resized)
    return seen


def test_stylize_equals_the_host_resize_path(vgg_weights):
    """Three scales, each of which resamples both images (900x700 content, 777x1100 style): the run on the device path,
    in which Pillow's resize may not be called at all, equals the run with the holder patched back to the host path."""
    content, style = O.synth_image(1, 16, 900, 700), O.synth_image(2, 32, 777, 1100)
    kw = dict(min_scale=64, end_scale=128, iterations=3, initial_iterations=4)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ST.SourceImage, 'resized', pil_resized)
        tr_h, avg_h, img_h = _stylize(['cuda:0'], vgg_weights, content, style, kw)
    with pytest.MonkeyPatch.context() as mp:
        _no_host_resize(mp)
        tr_d, avg_d, img_d = _stylize(['cuda:0'], vgg_weights, content, style, kw)
    assert len({(w, h) for w, h, _ in tr_d}) == 3 and len(tr_d) == 4 + 3 + 3
    assert tr_d == tr_h
    assert torch.equal(avg_d, avg_h) and np.array_equal(img_d, img_h)


def test_stylize_with_a_grayscale_style_image(vgg_weights):
    """An 'L' style image is resized on the host in its own mode, as before; the RGB content beside it on the device."""
    content, style = O.synth_image(1, 16, 900, 700), O.synth_image(2, 32, 777, 1100).convert('L')
    kw = dict(min_scale=64, end_scale=91, iterations=3, initial_iterations=3)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ST.SourceImage, 'resized', pil_resized)
        tr_h, avg_h, _ = _stylize(['cuda:0'], vgg_weights, content, style, kw)
    tr_d, avg_d, _ = _stylize(['cuda:0'], vgg_weights, content, style, kw)
    assert tr_d == tr_h and torch.equal(avg_d, avg_h)


def test_tiled_stylize_equals_the_host_resize_path(vgg_weights):
    """Two ranks on one GPU, 128 -> 384 of a 600x800 content image: the small scales replicated, the large ones banded.
    On a banded scale each rank resamples its band's rows only, and the run equals the host-path run bit for bit."""
    content, style = O.synth_image(1, 16, 600, 800), O.synth_image(2, 32, 777, 1100)
    kw = dict(min_scale=128, end_scale=384, iterations=3, initial_iterations=4)
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(ST.SourceImage, 'resized', pil_resized)
        tr_h, avg_h, img_h = _stylize(SAME_GPU, vgg_weights, content, style, kw)
    with pytest.MonkeyPatch.context() as mp:
        _no_host_resize(mp)
        seen = _spy_windows(mp)
        tr_d, avg_d, img_d = _stylize(SAME_GPU, vgg_weights, content, style, kw)
    assert D.make_band(tr_d[-1][1], 0, 2) is not None and D.make_band(tr_d[0][1], 0, 2) is None
    assert tr_d == tr_h
    assert torch.equal(avg_d, avg_h) and np.array_equal(img_d, img_h)
    # content and style are both 384 rows at the last scale, and banded: nobody asked for all of them
    last = [(h, rows) for h, rows in seen if h == tr_d[-1][1]]
    assert len(last) == 4 and all(rows < h for h, rows in last), last
