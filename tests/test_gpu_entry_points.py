"""-m gpu: the preconditions of the Adam iteration entry points, and which captured graphs a geometry change drops.

A band of a one-rank world (the whole image, no apron) needs no peer: its exchange kernels wait for nobody, so one
context on one stream can run stb_iterate_banded / stb_iterate_lbfgs_banded and have them captured as CUDA graphs.
"""
import ctypes

import pytest
import torch

import style_transfer_b200 as stb
from style_transfer_b200 import _lib
from style_transfer_b200 import distributed as D
import test_gpu_lbfgs as L

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
HL, W = 96, 64
LR, B1, B2, EPS = 0.02, 0.9, 0.99, 1e-8


def _whole_band():
    return D.Band(0, 1, HL, 0, HL, 0, HL)


def _banded_context(vgg_weights):
    """A context with targets for an HL x W band that is the whole image of a one-rank world."""
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights, distributed=False)
    m = st.model
    img, (ct, means, srms) = L._targets(st, HL, W)
    m.set_band(True, HL, 0, HL)
    m.set_targets(HL, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    return st, m, img, (ct, means, srms)


def test_adam_entry_point_errors_are_reported_before_any_launch(vgg_weights):
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights, distributed=False)
    m = st.model
    img, (ct, means, srms) = L._targets(st, HL, W)
    ea, eas, ema = torch.zeros_like(img), torch.zeros_like(img), img * 0.01

    def iterate(img_=img, ea_=ea, step=1):
        _lib.check(m.lib.stb_iterate(m.ctx, _lib.ptr(img_), _lib.ptr(ea_), _lib.ptr(eas), _lib.ptr(ema), step, LR, B1,
                                     B2, EPS, L.DECAY, None, _lib.cur_stream()))

    def banded(img_=img, ea_=ea, step=1):
        _lib.check(m.lib.stb_iterate_banded(m.ctx, _lib.ptr(img_), _lib.ptr(ea_), _lib.ptr(eas), _lib.ptr(ema), step,
                                            LR, B1, B2, EPS, L.DECAY, None, _lib.cur_stream()))

    with pytest.raises(_lib.NativeError, match='error -4'):     # no band
        banded()
    m.set_band(True, HL, 0, HL)
    m.set_targets(HL, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    with pytest.raises(_lib.NativeError, match='error -4'):     # stb_iterate updates the whole image, not a band
        iterate()
    with pytest.raises(_lib.NativeError, match='error -4'):     # no comm connection / geometry
        banded()
    _, p = m.comm_create(0, 1, HL, W)
    m.comm_connect_local([p])
    m.comm_set_geometry(W, D.Band(0, 1, HL, 0, HL - 16, 0, HL - 16), None, None, False)   # 80 own rows: not this band
    with pytest.raises(_lib.NativeError, match='error -4'):     # geometry does not match the band
        banded()
    m.comm_set_geometry(W, _whole_band(), None, None, False)
    for call, kw in ((banded, dict(img_=None)), (banded, dict(ea_=None)), (banded, dict(step=0)),
                     (iterate, dict(img_=None))):
        with pytest.raises(ValueError):
            call(**kw)
    torch.cuda.synchronize()
    assert st.model.graph_status()[0] == 2    # nothing was captured (or launched) by the refused calls


def test_geometry_change_drops_the_banded_lbfgs_graph(vgg_weights):
    """The banded L-BFGS graph bakes in the halo mode and the neighbours' heights: stb_comm_set_geometry drops it."""
    st, m, img, _ = _banded_context(vgg_weights)
    _, p = m.comm_create(0, 1, HL, W)
    m.comm_connect_local([p])
    m.comm_set_geometry(W, _whole_band(), None, None, False)
    stream = torch.cuda.Stream(device=DEV)     # graphs are captured on non-legacy streams only
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        m.comm_reset()
        n = ctypes.c_size_t()
        _lib.check(m.lib.stb_lbfgs_state_bytes(HL, W, ctypes.byref(n)))
        keep = torch.zeros(n.value + 512, dtype=torch.uint8, device=DEV)
        state = (keep.data_ptr() + 255) // 256 * 256
        _lib.check(m.lib.stb_lbfgs_reset(ctypes.c_void_p(state), HL, W, _lib.cur_stream()))
        ema = img * 0.01
        for step in range(1, 5):    # two eager iterations, then the capture, then a replay
            _lib.check(m.lib.stb_iterate_lbfgs_banded(m.ctx, _lib.ptr(img), _lib.ptr(ema), ctypes.c_void_p(state),
                                                      n.value, step, L.DECAY, None, _lib.cur_stream()))
        stream.synchronize()
    assert torch.isfinite(img).all() and torch.isfinite(ema).all()
    status, note = m.graph_status()
    assert status == 1, note
    m.comm_set_geometry(W, _whole_band(), None, None, False)
    assert m.graph_status()[0] == 2
