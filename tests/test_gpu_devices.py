"""-m gpu: StyleTransfer(devices=[a, b]) -- one process, one rank per listed device, the large scales tiled across them.

The public two-device call builds rank 1 on the second device and drives it from a thread of its own, in lockstep
with rank 0 on the caller's thread.  A list naming one GPU twice is legal and gives two ranks on that GPU, so these
tests cover the driver on a one-GPU box; the tests marked for two GPUs run where there are two.  The tiled path
itself is held against the untiled one in test_gpu_tiled.py / test_gpu_lbfgs_tiled.py; here the two-device call must
give exactly what the thread-group run of the same job gives.
"""
import contextlib
import ctypes
import io
import json
import signal
import threading

import numpy as np
import pytest
import torch

import style_transfer_b200 as stb
from style_transfer_b200 import _lib
from style_transfer_b200 import distributed as D
from oracle import st_oracle as O
from test_gpu_tiled import run_single, run_tiled

pytestmark = pytest.mark.gpu

SAME_GPU = ['cuda:0', 'cuda:0']
TWO_GPUS = ['cuda:0', 'cuda:1']
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')


def _comm_info(model):
    """(pdl, device of the own mailbox, device of the own peer-mapped workspace or -1)"""
    out = [ctypes.c_int(-2) for _ in range(3)]
    _lib.check(_lib.load_test().stb_test_comm_info(model.ctx, *map(ctypes.byref, out)), test_lib=True)
    return tuple(v.value for v in out)


def _run_devices(devices, content, style, wts, kw, callback=None):
    st = stb.StyleTransfer(devices=devices, pooling='max', vgg_weights=wts)
    trace = []

    def cb(it):
        trace.append(it.loss)
        if callback is not None:
            callback(st, it)

    with contextlib.redirect_stdout(io.StringIO()):
        img = st.stylize(content, [style], callback=cb, **kw)
    return st, np.array(trace), np.asarray(img, dtype=np.float32)


def _job(W, H):
    return O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)


@pytest.mark.parametrize('tile', ['halo', 'apron'])
@pytest.mark.parametrize('W,H', [(512, 384), (362, 384)])
def test_two_ranks_on_one_gpu_equal_thread_group_and_single(vgg_weights, monkeypatch, tile, W, H):
    """devices=['cuda:0', 'cuda:0']: bit-identical to run_tiled(2) of the same job, within the tiled bars of the
    untiled run; graphs replay on both ranks, and ranks sharing a GPU keep the early release of the exchanges off."""
    monkeypatch.setenv('STB_TILE', tile)
    content, style = _job(W, H)
    kw = dict(min_scale=max(W, H), end_scale=max(W, H), initial_iterations=6)
    before = threading.active_count()
    st, tr, img = _run_devices(SAME_GPU, content, style, vgg_weights, kw)
    assert threading.active_count() == before
    assert st._peer is not None and st._world == 2
    for m in (st.model, st._peer.model):
        gstat, note = m.graph_status()
        assert gstat == 1, note
        assert _comm_info(m) == (0, 0, 0 if tile == 'halo' else -1)
    assert st._halo_now == (tile == 'halo') and st._comm_mode == 'peer'
    tr_s, img_s = run_single(content, style, vgg_weights, kw)
    assert len(tr) == 6
    assert (np.abs(tr - tr_s) / np.abs(tr_s)).max() < 5e-4
    assert np.abs(img - img_s).mean() < 0.5
    tiled = run_tiled(2, content, style, vgg_weights, kw)
    np.testing.assert_array_equal(tr, tiled[0][0])
    np.testing.assert_array_equal(img, tiled[0][1])


def _lbfgs_bars(tr, tr_s, ema, ema_s):
    """The bars of test_gpu_lbfgs_tiled._check_end_to_end: L-BFGS amplifies the tiled closure's summation-order
    difference once it holds a pair."""
    drift = np.abs(tr - tr_s) / np.abs(tr_s)
    assert np.isfinite(tr).all()
    assert drift[:2].max() <= 5e-4, drift
    assert drift.max() <= 1e-2, drift
    assert (ema - ema_s).abs().mean().item() < 5e-3


@pytest.mark.parametrize('optimizer', ['adam', 'lbfgs'])
def test_pyramid_mixes_replicated_and_banded_scales(vgg_weights, optimizer):
    """128 -> 384: the small scales run replicated on both ranks, the large ones banded."""
    W, H = 288, 384
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, 260, 300)
    kw = dict(min_scale=128, end_scale=384, iterations=3, initial_iterations=4, optimizer=optimizer)
    sizes = []
    st, tr, img = _run_devices(SAME_GPU, content, style, vgg_weights, kw,
                               callback=lambda st, it: sizes.append(it.h))
    heights = sorted(set(sizes))
    assert D.make_band(heights[0], 0, 2) is None and D.make_band(heights[-1], 0, 2) is not None
    ref = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights, distributed=False)
    tr_s = []
    with contextlib.redirect_stdout(io.StringIO()):
        img_s = np.asarray(ref.stylize(content, [style], callback=lambda it: tr_s.append(it.loss), **kw),
                           dtype=np.float32)
    tr_s = np.array(tr_s)
    assert len(tr) == len(tr_s) == 4 + 3 * (len(heights) - 1)
    if optimizer == 'adam':
        np.testing.assert_allclose(tr, tr_s, rtol=2e-3)
        assert np.abs(img - img_s).mean() < 1.0
    else:
        _lbfgs_bars(tr, tr_s, st.average.get().cpu(), ref.average.get().cpu())


def test_callback_sees_the_whole_image_on_the_callers_thread(vgg_weights):
    W, H = 512, 384
    content, style = _job(W, H)
    kw = dict(min_scale=512, end_scale=512, initial_iterations=6)
    seen = []

    def cb(st, it):
        assert st._band is not None           # a banded scale: get_image() gathers rank 1's rows
        seen.append((threading.get_ident(), it.w, it.h, np.asarray(st.get_image(), dtype=np.float32)))

    st, tr, img = _run_devices(SAME_GPU, content, style, vgg_weights, kw, callback=cb)
    assert len(seen) == 6
    for ident, w, h, im in seen:
        assert ident == threading.get_ident()
        assert (w, h) == (W, H) and im.shape == (H, W, 3)
    np.testing.assert_array_equal(seen[-1][3], img)
    assert st.image.shape == (1, 3, H, W) and st.average.value.shape == (1, 3, H, W)


class _Stop(Exception):
    pass


def test_callback_error_stops_both_ranks_at_the_same_iteration(vgg_weights):
    """A callback that raises at iteration 3 of a banded scale: stylize() re-raises it, rank 1's thread is gone, and
    both ranks launched the same iterations (read before anything synchronises the device: no peer wait is left
    without its partner).  Afterwards the object holds the whole image of iteration 3, the image a run of three
    iterations ends with."""
    content, style = _job(512, 384)
    kw = dict(min_scale=512, end_scale=512)
    st = stb.StyleTransfer(devices=SAME_GPU, pooling='max', vgg_weights=vgg_weights)
    before = threading.active_count()

    def cb(it):
        if it.i == 3:
            raise _Stop()

    with contextlib.redirect_stdout(io.StringIO()), pytest.raises(_Stop):
        st.stylize(content, [style], initial_iterations=6, callback=cb, **kw)
    counts = (st.model.launch_count()[0], st._peer.model.launch_count()[0])
    assert threading.active_count() == before
    assert counts[0] == counts[1] > 0, counts
    torch.cuda.synchronize()
    assert st._band is None and st.average.value.shape == (1, 3, 384, 512)
    stopped = np.asarray(st.get_image(), dtype=np.float32)
    _, _, three = _run_devices(SAME_GPU, content, style, vgg_weights, dict(initial_iterations=3, **kw))
    np.testing.assert_array_equal(stopped, three)


@two_gpus
def test_cli_two_gpus(vgg_weights, tmp_path, monkeypatch):
    assert len(_cli(vgg_weights, tmp_path, monkeypatch, TWO_GPUS)) == 9


class _InterruptAt(io.StringIO):
    """stdout of the CLI that sends this process SIGINT (Ctrl-C) once `line` is printed."""

    def __init__(self, line):
        super().__init__()
        self.line = line

    def write(self, text):
        n = super().write(text)
        if self.line and self.line in self.getvalue():
            self.line = None
            signal.raise_signal(signal.SIGINT)
        return n


def _cli(wts, tmp_path, monkeypatch, devices, interrupt_at=None):
    from style_transfer_b200 import cli
    from style_transfer_b200 import style_transfer as S
    monkeypatch.setattr(S, 'load_vgg19_conv_weights', lambda: wts)   # no network for the ImageNet checkpoint
    monkeypatch.chdir(tmp_path)
    O.synth_image(1, 16, 256, 192).save('c.png')
    O.synth_image(2, 32, 200, 160).save('s.png')
    out = _InterruptAt(interrupt_at)
    with contextlib.redirect_stdout(out):
        cli.main(['c.png', 's.png', '--devices', *devices, '-s', '256', '-i', '3', '-ii', '3'])
    text = out.getvalue()
    assert 'GPU 0 type:' in text and 'GPU 1 RAM:' in text
    from PIL import Image
    assert Image.open('out.png').size == (256, 192)
    return json.load(open('trace.json'))['iterates']


def test_cli_two_ranks_on_one_gpu(vgg_weights, tmp_path, monkeypatch):
    trace = _cli(vgg_weights, tmp_path, monkeypatch, SAME_GPU)
    assert len(trace) == 3 + 3 + 3 and trace[-1]['w'] == 256 and trace[-1]['h'] == 192


def test_cli_ctrl_c_on_a_banded_scale_writes_the_image(vgg_weights, tmp_path, monkeypatch):
    """Ctrl-C during iteration 2 of the banded 256x192 scale takes effect at the next launch: the CLI still writes
    the whole image and the trace up to that iteration."""
    trace = _cli(vgg_weights, tmp_path, monkeypatch, SAME_GPU, interrupt_at='Size: 256x192, iteration: 2,')
    assert len(trace) == 3 + 3 + 2 and trace[-1]['w'] == 256 and trace[-1]['i'] == 2


@two_gpus
@pytest.mark.parametrize('tile', ['halo', 'apron'])
@pytest.mark.parametrize('W,H', [(512, 384), (362, 384)])
def test_two_gpus_equal_single(vgg_weights, monkeypatch, tile, W, H):
    monkeypatch.setenv('STB_TILE', tile)
    content, style = _job(W, H)
    kw = dict(min_scale=max(W, H), end_scale=max(W, H), initial_iterations=6)
    st, tr, img = _run_devices(TWO_GPUS, content, style, vgg_weights, kw)
    assert st._dev == torch.device('cuda:0') and st._peer._dev == torch.device('cuda:1')
    for m, dev in ((st.model, 0), (st._peer.model, 1)):
        gstat, note = m.graph_status()
        assert gstat == 1, note
        pdl, mailbox_dev, ws_dev = _comm_info(m)
        assert pdl == 1 and mailbox_dev == dev
        if tile == 'apron':                    # torch-owned workspace
            assert m._ws.device == torch.device('cuda', dev) and ws_dev == -1
        else:                                  # the library-owned, peer-mapped workspace
            assert m._ws_shared and ws_dev == dev
    assert torch.cuda.max_memory_allocated(1) > 0
    tr_s, img_s = run_single(content, style, vgg_weights, kw)
    assert (np.abs(tr - tr_s) / np.abs(tr_s)).max() < 5e-4
    assert np.abs(img - img_s).mean() < 0.5
