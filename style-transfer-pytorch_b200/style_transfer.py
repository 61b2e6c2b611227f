"""Drop-in `StyleTransfer` whose per-iteration body is one call into libstb200 (hand-written sm_90a CUDA).

Public surface mirrors /root/reference/style_transfer/style_transfer.py ("ST"): `StyleTransfer(devices, pooling)`
(ST:310), attributes (ST:311-324), `get_image_tensor` / `get_image` (ST:335-347), `stylize(...)` with the same
keyword-only signature, defaults and annotations (ST:349-363; the CLI scrapes them, cli.py:150-153), `STIterate`
(ST:298-306) and the synchronous per-iteration callback (ST:487-493).  Host-side work that is per *scale*, not per
iteration (the random init modes, the per-scale bookkeeping) stays in PyTorch; everything inside the iteration loop
(ST:472-486) runs in the native library, and so do the per-scale resizes of the source images (SourceImage) and the
warm start.  There is no CPU or autograd fallback.
"""
from __future__ import annotations

import contextlib
import ctypes
import gc
import os
import signal
import threading
import time
import warnings
from dataclasses import dataclass

import numpy as np
import torch
from PIL import Image

from . import _lib
from . import distributed as D

CONV_CHANNELS = [(3, 64), (64, 64), (64, 128), (128, 128), (128, 256), (256, 256), (256, 256), (256, 256),
                 (256, 512), (512, 512), (512, 512), (512, 512), (512, 512)]
VGG19_CONV_INDICES = [0, 2, 5, 7, 10, 12, 14, 16, 19, 21, 23, 25, 28]
STYLE_CHANNELS = [64, 128, 256, 512, 512]
# the ReLU taps of the reference model, VGGFeatures(style_layers + content_layers) with its default lists (ST:324), and
# their channel counts: content_layers and style_layers may name any of them
TAP_CHANNELS = {1: 64, 6: 128, 11: 256, 20: 512, 22: 512, 29: 512}
TAP_LEVEL = D.TAP_LEVEL


def check_layers(content_layers, style_layers):
    """Validate StyleTransfer.content_layers / style_layers: KeyError(layer) for a tap the reference model does not
    have (its LayerApply raises the same, ST:234), ValueError for a tap listed twice in one list (the reference would
    count a repeated style layer's target statistics twice, ST:442-450).  An empty content list raises
    ZeroDivisionError earlier, where the content weight is divided by its length (ST:366)."""
    for name, layers in (('content_layers', content_layers), ('style_layers', style_layers)):
        for layer in layers:
            if layer not in TAP_CHANNELS:
                raise KeyError(layer)
        if len(set(layers)) != len(layers):
            raise ValueError(f'{name} lists a layer twice: {list(layers)}')


@dataclass
class STIterate:
    w: int
    h: int
    i: int
    i_max: int
    loss: float
    time: float
    gpu_ram: int


def size_to_fit(size, max_dim, scale_up=False):
    """Aspect-preserving (w, h) whose longer side is max_dim (ST:256-265)."""
    w, h = size
    if max(w, h) <= max_dim and not scale_up:
        return w, h
    if h > w:
        return round(max_dim * w / h), max_dim
    return max_dim, round(max_dim * h / w)


def gen_scales(start, end):
    """Pyramid of scales end / 2^(i/2) down to start, ascending (ST:268-276)."""
    out = set()
    i, scale = 0, end
    while scale >= start:
        out.add(scale)
        i += 1
        scale = round(end / pow(2, i / 2))
    return sorted(out)


def _pil_to_tensor(img, device=None):
    """TF.to_tensor semantics ([1,3,H,W] fp32 in [0,1], contiguous).  With a CUDA `device` the uint8 pixels are
    uploaded (3 bytes/pixel instead of 12) and converted there."""
    if img.mode != 'RGB':
        img = img.convert('RGB')
    t = torch.from_numpy(np.array(img, dtype=np.uint8))
    if device is not None:
        t = t.to(device, non_blocking=True)
    return t.permute(2, 0, 1).to(torch.float32).div_(255).unsqueeze(0).contiguous()


def resample_coeffs(in_size, out_size):
    """Fixed-point tables of one axis of `Image.resize(..., Image.BICUBIC)` on 8-bit pixels, from `in_size` to `out_size`
    samples: (k int32 [out_size, ksize], bounds int32 [out_size, 2]).  Output sample x is
    clip8((2^21 + sum_j source[first + j] * k[x, j]) >> 22) over j < count, with (first, count) = bounds[x]; taps
    beyond count are zero.  Pillow forms the weights in double: the Keys kernel (a = -0.5) stretched by
    max(in / out, 1), divided by their sum accumulated in tap order, rounded half away from zero to 22 fractional
    bits.  The loop below runs over the taps so that every sum is taken in that order (np.sum adds pairwise)."""
    scale = in_size / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    ksize = 2 * int(np.ceil(support)) + 1
    center = (np.arange(out_size, dtype=np.float64) + 0.5) * scale
    first = np.maximum((center - support + 0.5).astype(np.int64), 0)       # astype truncates, as C's (int)
    count = np.minimum((center + support + 0.5).astype(np.int64), in_size) - first
    inv = 1.0 / filterscale
    w = np.zeros((out_size, ksize), dtype=np.float64)
    total = np.zeros(out_size, dtype=np.float64)
    for j in range(ksize):
        t = np.abs((j + first - center + 0.5) * inv)
        near = ((-0.5 + 2.0) * t - (-0.5 + 3.0)) * t * t + 1
        far = (((t - 5) * t + 8) * t - 4) * -0.5
        w[:, j] = np.where(j < count, np.where(t < 1.0, near, np.where(t < 2.0, far, 0.0)), 0.0)
        total += w[:, j]
    total[total == 0.0] = 1.0
    w /= total[:, None]
    k = (w * float(1 << 22) + np.where(w < 0, -0.5, 0.5)).astype(np.int32)
    return k, np.stack([first, count], axis=1).astype(np.int32)


class SourceImage:
    """One content or style image of a stylize() call, resampled to every scale on the device.

    An RGB image is uploaded once, as interleaved uint8 [Hs][Ws][3]; resized() then produces what
    `_pil_to_tensor(img.resize((w, h), Image.BICUBIC), device)` produces, bit for bit, by stb_resample_rgb8.  Pillow
    resamples every other mode (RGBA, P, I;16, F, ...) by other rules, so such an image keeps that expression: it is
    resized in its own mode on the host and converted afterwards."""

    def __init__(self, img, device):
        self.img, self.device = img, device
        self.data = None
        if img.mode == 'RGB':
            self.data = torch.from_numpy(np.array(img, dtype=np.uint8)).to(device, non_blocking=True)

    def resized(self, w, h, row0=0, rows=None):
        """Rows [row0, row0 + rows) (default: all) of the image at w x h: [1,3,rows,w] fp32 in [0,1] on the device."""
        rows = h - row0 if rows is None else rows
        if self.data is None:
            full = _pil_to_tensor(self.img.resize((w, h), Image.BICUBIC), self.device)
            return full[:, :, row0:row0 + rows].contiguous()
        hs, ws, _ = self.data.shape
        lib = _lib.load()
        need = ctypes.c_size_t()
        _lib.check(lib.stb_resample_tmp_bytes(hs, ws, h, w, row0, rows, ctypes.byref(need)))   # validates the window
        # an axis that keeps its size is not filtered (Pillow skips that pass) and has no tables
        axes = [resample_coeffs(n_in, n_out) if n_in != n_out else None for n_in, n_out in ((ws, w), (hs, h))]
        flat = [t.ravel() for axis in axes if axis is not None for t in axis]
        with torch.cuda.device(self.device):
            tab = torch.from_numpy(np.concatenate(flat)).to(self.device) if flat else None   # one upload for all four
            tmp = torch.empty(need.value, dtype=torch.uint8, device=self.device)
            out = torch.empty(1, 3, rows, w, dtype=torch.float32, device=self.device)
            args, off = [], 0
            for axis in axes:
                if axis is None:
                    args += [None, None, 0]
                    continue
                k, bounds = axis
                args += [ctypes.c_void_p(tab.data_ptr() + 4 * off), ctypes.c_void_p(tab.data_ptr() + 4 * (off + k.size)),
                         k.shape[1]]
                off += k.size + bounds.size
            _lib.check(lib.stb_resample_rgb8(_lib.ptr(self.data), hs, ws, h, w, row0, rows, *args,
                                             _lib.ptr(tmp), need.value, _lib.ptr(out), _lib.cur_stream()))
        return out


def load_vgg19_conv_weights():
    """The thirteen conv (weight, bias) pairs of torchvision vgg19 IMAGENET1K_V1 features[:30] (as ST:35)."""
    from torchvision import models
    feats = models.vgg19(weights=models.VGG19_Weights.IMAGENET1K_V1).features
    return [(feats[i].weight.detach().clone(), feats[i].bias.detach().clone()) for i in VGG19_CONV_INDICES]


class EMA:
    """Bias-corrected exponential moving average of the iterate (ST:237-253); `value` is updated in place by the
    native iteration, only the scalar `accum` lives on the host."""

    def __init__(self, input, decay):
        self.decay = float(decay)
        self.accum = self.decay
        self.value = input.detach() * (1 - self.decay)

    @classmethod
    def from_state(cls, value, accum, decay):
        self = cls.__new__(cls)
        self.decay, self.accum, self.value = float(decay), float(accum), value
        return self

    def get(self):
        return self.value / (1 - self.accum)

    def note_update(self):
        self.accum *= self.decay


class NativeVGG:
    """Holder of the frozen VGG-19 conv stack and the native context built from it (replaces VGGFeatures, ST:20-90)."""

    def __init__(self, conv_weights, pooling, device):
        if pooling not in _lib.POOLING:
            raise KeyError(pooling)
        if len(conv_weights) != 13:
            raise ValueError('expected 13 (weight, bias) pairs for vgg19.features[:30]')
        self.pooling = pooling
        self.device = device
        self.weights = []
        for (w, b), (cin, cout) in zip(conv_weights, CONV_CHANNELS):
            if tuple(w.shape) != (cout, cin, 3, 3) or tuple(b.shape) != (cout,):
                raise ValueError(f'bad conv parameter shape {tuple(w.shape)} / {tuple(b.shape)}')
            self.weights.append((w.detach().to(device, torch.float32).contiguous(),
                                 b.detach().to(device, torch.float32).contiguous()))
        self.lib = _lib.load()
        self.ctx = ctypes.c_void_p()
        with torch.cuda.device(device):
            wp, _k1 = _lib.ptr_array([w for w, _ in self.weights])
            bp, _k2 = _lib.ptr_array([b for _, b in self.weights])
            _lib.check(self.lib.stb_ctx_create(device.index or 0, _lib.POOLING[pooling], wp, bp, _lib.cur_stream(),
                                               ctypes.byref(self.ctx)))
        self._ws = None
        self._ws_bound = 0
        self._ws_shared = False

    def __del__(self):
        try:
            if getattr(self, 'ctx', None) and self.ctx.value:
                self.lib.stb_ctx_destroy(self.ctx)
                self.ctx = ctypes.c_void_p()
        except Exception:
            pass

    # ------------------------------------------------------------------ workspace
    def workspace_bytes(self, h, w):
        n = ctypes.c_size_t()
        _lib.check(self.lib.stb_workspace_bytes(self.ctx, h, w, ctypes.byref(n)))
        return n.value

    def ensure_workspace(self, sizes):
        """Bind a torch-owned workspace large enough for every (h, w) in sizes.  Returns True if (re)bound."""
        need = max(self.workspace_bytes(h, w) for h, w in sizes)
        if (self._ws is not None or self._ws_shared) and need <= self._ws_bound:   # what the context was actually given
            return False
        if self._ws_shared:
            raise _lib.NativeError('the library-owned (peer-mapped) workspace of this tiled run is too small: '
                                   f'{need} > {self._ws_bound} bytes')
        self._ws = None
        torch.cuda.empty_cache()  # hand the old block back before asking for the bigger one
        self._ws = torch.empty(need + 2048, dtype=torch.uint8, device=self.device)
        base = self._ws.data_ptr()
        aligned = (base + 1023) // 1024 * 1024
        self._ws_bound = self._ws.numel() - (aligned - base)    # bind everything usable, not just `need`
        _lib.check(self.lib.stb_bind_workspace(self.ctx, ctypes.c_void_p(aligned), self._ws_bound, _lib.cur_stream()))
        return True

    def release_workspace(self):
        self._ws = None
        self._ws_bound = 0

    def alloc_shared_workspace(self, sizes):
        """Per-layer-halo mode of a tiled run: the workspace is allocated (cudaMalloc), zeroed and bound by the library so
        that the neighbouring ranks can map it; returns (64-byte CUDA IPC handle, device pointer)."""
        need = max(self.workspace_bytes(h, w) for h, w in sizes) + 4096
        handle = ctypes.create_string_buffer(64)
        p = ctypes.c_void_p()
        self._ws = None
        torch.cuda.empty_cache()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.stb_comm_alloc_workspace(self.ctx, need, handle, ctypes.byref(p), _lib.cur_stream()))
        self._ws_bound, self._ws_shared = need, True
        return handle.raw, p.value

    def connect_shared_workspaces(self, items, ipc):
        if ipc:
            _lib.check(self.lib.stb_comm_connect_ws_ipc(self.ctx, b''.join(items)))
        else:
            arr = (ctypes.c_void_p * len(items))(*items)
            _lib.check(self.lib.stb_comm_connect_ws_local(self.ctx, ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p))))

    def release_shared_workspace(self, unmap_only):
        _lib.check(self.lib.stb_comm_release_workspace(self.ctx, int(unmap_only)))
        if not unmap_only:
            self._ws_bound, self._ws_shared = 0, False

    # ------------------------------------------------------------------ target extraction
    def _check_image(self, image):
        if image.dim() != 4 or image.shape[0] != 1 or image.shape[1] != 3:
            raise ValueError(f'expected a [1,3,H,W] image, got {tuple(image.shape)}')
        return image.detach().to(self.device, torch.float32).contiguous()

    def set_layers(self, content_layers, style_layers):
        """The context's layer table (stb_set_layers): content and style taps, in list order."""
        content_layers, style_layers = [int(t) for t in content_layers], [int(t) for t in style_layers]
        check_layers(content_layers, style_layers)
        ca = (ctypes.c_int * max(len(content_layers), 1))(*content_layers)
        sa = (ctypes.c_int * max(len(style_layers), 1))(*style_layers)
        _lib.check(self.lib.stb_set_layers(self.ctx, len(content_layers), ca, len(style_layers), sa))
        self.content_layers, self.style_layers = content_layers, style_layers

    content_layers = [22]               # the table of a context that never called set_layers
    style_layers = [1, 6, 11, 20, 29]

    @property
    def n_terms(self):
        """Length of the loss-term vector [total, content terms, style terms, tv] under the layer table."""
        return 2 + len(self.content_layers) + len(self.style_layers)

    def style_stats(self, image):
        """(means, second raw moments) of one image, one pair per style tap of the layer table."""
        image = self._check_image(image)
        _, _, h, w = image.shape
        chans = [TAP_CHANNELS[t] for t in self.style_layers]
        means = [torch.empty(c, device=self.device) for c in chans]
        srms = [torch.empty(c, c, device=self.device) for c in chans]
        mp, _k1 = _lib.ptr_array(means)
        sp, _k2 = _lib.ptr_array(srms)
        _lib.check(self.lib.stb_style_stats(self.ctx, _lib.ptr(image), h, w, mp, sp, _lib.cur_stream()))
        return means, srms

    def content_features(self, image):
        """The content target of the default layer table (tap 22, bf16 NHWC [H/8][W/8][512])."""
        image = self._check_image(image)
        _, _, h, w = image.shape
        out = torch.empty(h // 8, w // 8, 512, dtype=torch.bfloat16, device=self.device)
        _lib.check(self.lib.stb_content_features(self.ctx, _lib.ptr(image), h, w, _lib.ptr(out), _lib.cur_stream()))
        return out

    def content_features_list(self, image):
        """One bf16 NHWC target per content tap of the layer table."""
        image = self._check_image(image)
        _, _, h, w = image.shape
        out = [torch.empty(h >> TAP_LEVEL[t], w >> TAP_LEVEL[t], TAP_CHANNELS[t], dtype=torch.bfloat16,
                           device=self.device) for t in self.content_layers]
        op, _k = _lib.ptr_array(out)
        _lib.check(self.lib.stb_content_features_ex(self.ctx, _lib.ptr(image), h, w, op, _lib.cur_stream()))
        return out

    # ------------------------------------------------------------------ spatial tiling (multi-GPU) plumbing
    def set_band(self, enabled, h_global=0, own_row0=0, own_rows=0):
        _lib.check(self.lib.stb_set_band(self.ctx, int(enabled), h_global, own_row0, own_rows))

    def iterate_fwd(self, image):
        _lib.check(self.lib.stb_iterate_fwd(self.ctx, _lib.ptr(image), _lib.cur_stream()))

    def iterate_bwd(self, image, grad, loss_host):
        _lib.check(self.lib.stb_iterate_bwd(self.ctx, _lib.ptr(image), _lib.ptr(grad), _lib.ptr(loss_host),
                                            _lib.cur_stream()))

    # ------------------------------------------------------------------ peer-memory exchange (csrc/comm.cu)
    def comm_create(self, rank, world, max_h_local, max_w):
        """Allocate this rank's mailbox; returns (64-byte CUDA IPC handle, device pointer)."""
        handle = ctypes.create_string_buffer(64)
        p = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(self.lib.stb_comm_create(self.ctx, rank, world, max_h_local, max_w, handle, ctypes.byref(p)))
        return handle.raw, p.value

    def comm_connect_ipc(self, handles):
        blob = b''.join(handles)
        _lib.check(self.lib.stb_comm_connect_ipc(self.ctx, blob))

    def comm_connect_local(self, pointers):
        arr = (ctypes.c_void_p * len(pointers))(*pointers)
        _lib.check(self.lib.stb_comm_connect_local(self.ctx, ctypes.cast(arr, ctypes.POINTER(ctypes.c_void_p))))

    def comm_disconnect(self):
        _lib.check(self.lib.stb_comm_disconnect(self.ctx))

    def comm_set_geometry(self, w, band, up, down, halo_rows):
        _lib.check(self.lib.stb_comm_set_geometry(self.ctx, w, band.h_local, band.own0, band.own_rows,
                                                  up.h_local if up else 0, up.own0 + up.own_rows if up else 0,
                                                  down.h_local if down else 0, int(halo_rows)))

    def comm_reset(self):
        _lib.check(self.lib.stb_comm_reset(self.ctx, _lib.cur_stream()))

    def iterate_banded(self, image, exp_avg, exp_avg_sq, ema, step, lr, avg_decay, loss_host):
        _lib.check(self.lib.stb_iterate_banded(self.ctx, _lib.ptr(image), _lib.ptr(exp_avg), _lib.ptr(exp_avg_sq),
                                               _lib.ptr(ema), step, lr, 0.9, 0.99, 1e-8, avg_decay,
                                               _lib.ptr(loss_host), _lib.cur_stream()))

    def graph_status(self):
        note = ctypes.create_string_buffer(512)
        return self.lib.stb_graph_status(self.ctx, note, 512), note.value.decode(errors='replace')

    def resize(self, x, hw, mode, post=None):
        """F.interpolate(x, hw, mode=mode, align_corners=False) on the device by the library's own kernel
        (stb_resize): the warm start of a scale, ST:285-295 / ST:420.  post: None | 'relu' | 'clamp'."""
        x = x.detach().to(self.device, torch.float32).contiguous()
        n, c, h, w = x.shape
        out = torch.empty(n, c, hw[0], hw[1], dtype=torch.float32, device=self.device)
        _lib.check(self.lib.stb_resize(_lib.ptr(x), n * c, h, w, _lib.ptr(out), hw[0], hw[1],
                                       {'bilinear': 0, 'bicubic': 1}[mode], {None: 0, 'relu': 1, 'clamp': 2}[post],
                                       _lib.cur_stream()))
        return out

    def launch_count(self):
        """(graph replays, kernels launched by them, kernel nodes per graph slot) -- counted from the captured graphs."""
        a, b, per = ctypes.c_int64(), ctypes.c_int64(), (ctypes.c_int * 4)()
        _lib.check(self.lib.stb_launch_count(self.ctx, ctypes.byref(a), ctypes.byref(b), per))
        return a.value, b.value, list(per)

    def set_targets(self, h, w, content_target, content_weight, means, srms, layer_weights, tv_weight, eps=1e-4):
        """Targets of the default layer table: one content target, five style taps."""
        mp, _k1 = _lib.ptr_array(means)
        sp, _k2 = _lib.ptr_array(srms)
        lw = (ctypes.c_float * 5)(*layer_weights)
        _lib.check(self.lib.stb_set_targets(self.ctx, h, w, _lib.ptr(content_target), content_weight, mp, sp, lw,
                                            tv_weight, eps, _lib.cur_stream()))

    def set_targets_list(self, h, w, content_targets, content_weights, means, srms, layer_weights, tv_weight,
                         eps=1e-4):
        """Per-layer lists in layer-table order: content targets and weights, style moments and layer weights."""
        cp, _k0 = _lib.ptr_array(content_targets)
        cw = (ctypes.c_float * len(content_weights))(*content_weights)
        mp, _k1 = _lib.ptr_array(means)
        sp, _k2 = _lib.ptr_array(srms)
        lw = (ctypes.c_float * max(len(layer_weights), 1))(*layer_weights)
        _lib.check(self.lib.stb_set_targets_ex(self.ctx, h, w, cp, cw, mp, sp, lw, tv_weight, eps, _lib.cur_stream()))

    def loss_terms(self):
        """[total, content terms, style terms, tv] of the last iteration (synchronises the current stream)."""
        out = torch.zeros(_lib.MAX_LOSS_TERMS, dtype=torch.float32)
        n = ctypes.c_int()
        _lib.check(self.lib.stb_loss_terms(self.ctx, _lib.ptr(out), out.numel(), ctypes.byref(n), _lib.cur_stream()))
        torch.cuda.current_stream().synchronize()
        return out[:n.value].clone()


class _Stopped(Exception):
    """The other in-process rank stopped (its error is the one stylize() raises)."""


class _PeerUnavailable(Exception):
    """The in-process ranks could not map each other's memory: the job runs untiled on the first device instead."""


class _Lockstep:
    """Host-side handshake of the two in-process ranks of StyleTransfer(devices=[a, b]), one per stylize() call.

    A banded iteration waits on the device for its peer's stamps, so an iteration launched by one rank and never by the
    other traps after the exchange timeout.  Both ranks must therefore launch the same steps however either one stops:
      * rank 1 announces step s (ready1) only once nothing but its launch is left before it: rank 0's callback of step
        s-1 is over, and with it every gather that callback asked rank 1 to serve;
      * rank 0 launches step s only once rank 1 has announced it and has not stopped since;
      * rank 1 launches step s only after rank 0 has published its launch (launched0).
    Rank 0 raises nothing between its launch and that publication: a launch call that fails has launched nothing, and
    SIGINT is held back (_deferred_sigint) and turned into KeyboardInterrupt at rank 0's next gate.

    get_image() inside rank 0's callback is collective on a banded scale (gather_rows): rank 1 serves the gathers rank 0
    requests while it waits for that callback to end (at its next gate or at the end of the scale).  It has launched the
    step rank 0 is reporting and launches nothing more until rank 0 does, so its rows are that step's."""

    def __init__(self):
        self.cond = threading.Condition()
        self.ready1 = self.launched0 = self.done0 = 0
        self.requested = self.served = 0
        self.stopped = False
        self.interrupt = None    # (handler, signum) of a SIGINT held back until rank 0's next gate

    def deliver_interrupt(self):
        """Rank 0: run the SIGINT handler held back since the signal arrived (it raises KeyboardInterrupt)."""
        if self.interrupt is not None:
            handler, signum = self.interrupt
            self.interrupt = None
            handler(signum, None)

    def stop(self):
        with self.cond:
            self.stopped = True
            self.cond.notify_all()

    def _set(self, **kw):
        with self.cond:
            for k, v in kw.items():
                setattr(self, k, v)
            self.cond.notify_all()

    def request_gather(self):
        with self.cond:
            self.requested += 1
            self.cond.notify_all()

    def _serve_until(self, st, done):
        """Rank 1: serve rank 0's gathers until done() (checked first) or the stop."""
        with self.cond:
            while not done():
                if self.served < self.requested:
                    self.served += 1
                    self.cond.release()
                    try:
                        st.get_image_tensor()
                    finally:
                        self.cond.acquire()
                elif self.stopped:
                    raise _Stopped()
                else:
                    self.cond.wait()

    def before_launch(self, st, step):
        if st._rank == 0:
            with self.cond:
                while True:
                    self.deliver_interrupt()
                    if self.stopped:
                        raise _Stopped()
                    if self.ready1 >= step:
                        return
                    self.cond.wait(0.05)    # a held-back SIGINT does not notify
        else:
            self._serve_until(st, lambda: self.done0 >= step - 1)
            self._set(ready1=step)
            with self.cond:
                while self.launched0 < step:
                    if self.stopped:
                        raise _Stopped()
                    self.cond.wait()

    def after_launch(self, st, step):
        if st._rank == 0:
            self._set(launched0=step)

    def after_iteration(self, st, step):
        if st._rank == 0:
            self._set(done0=step)

    def end_of_scale(self, st, step):
        if st._rank != 0:
            self._serve_until(st, lambda: self.done0 >= step)


@contextlib.contextmanager
def _deferred_sigint(sync):
    """While a two-device stylize() runs on the main thread, SIGINT only records itself; rank 0 runs the handler at its
    next launch gate (_Lockstep.deliver_interrupt).  A KeyboardInterrupt raised wherever the signal lands could fall
    between rank 0's launch and its publication, and rank 1 would stop one launch short of it."""
    prev = signal.getsignal(signal.SIGINT)
    install = threading.current_thread() is threading.main_thread() and callable(prev)
    if install:
        def hold(signum, frame):
            sync.interrupt = (prev, signum)
        signal.signal(signal.SIGINT, hold)
    try:
        yield
    finally:
        if install:
            signal.signal(signal.SIGINT, prev)


class StyleTransfer:
    RING_SLOTS = 8

    def __init__(self, devices=['cpu'], pooling='max', *, vgg_weights=None, distributed=None):
        self.devices = [torch.device(device) for device in devices]
        self.image = None
        self.average = None

        self.content_layers = [22]
        self.style_layers = [1, 6, 11, 20, 29]
        raw = [256, 64, 16, 4, 1]
        total = sum(abs(w) for w in raw)
        self.style_weights = [w / total for w in raw]

        if len(self.devices) not in (1, 2):
            raise ValueError('Only 1 or 2 devices are supported.')
        if not torch.cuda.is_available():
            raise RuntimeError('CUDA is not available; the H100-native hot path cannot run (there is no CPU '
                               'fallback).')
        if any(d.type != 'cuda' for d in self.devices):
            # the reference's default argument is devices=['cpu'] (ST:310): call sites that rely on it keep working,
            # on the GPU this implementation exists for -- loudly, never on a CPU path
            warnings.warn('style-transfer-pytorch_b200 runs its hot path only on CUDA (sm_90a) devices; '
                          f'devices={[str(d) for d in self.devices]} -> using cuda:{torch.cuda.current_device()} '
                          '(there is no CPU fallback)')
            self.devices = [torch.device('cuda', torch.cuda.current_device())]
        # two devices in one process (ST:326-333): one rank per listed device, the large scales tiled across them as
        # under torchrun.  An explicit group, or a torch.distributed job (one process per GPU already), keeps one
        # device per process.
        shared = None
        if len(self.devices) == 2:
            if distributed is None and D.default_group() is None:
                shared = D.ThreadGroup.Shared(2)
            else:
                warnings.warn('the reference\'s 2-device layer split (ST:326-333) is superseded; running on '
                              f'{self.devices[0]} only')
        dev = self.devices[0]
        if dev.index is None:
            dev = torch.device('cuda', torch.cuda.current_device())
        self._dev = dev
        if vgg_weights is None:
            vgg_weights = load_vgg19_conv_weights()
        self.model = NativeVGG(vgg_weights, pooling, dev)
        self._loss_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        # sync-free loss read-back (stb_set_loss_ring): the loss kernel itself writes the terms + an iteration stamp
        # into this pinned ring before the backward pass starts; the callback path polls the stamp
        self._ring = torch.zeros(self.RING_SLOTS, 16, dtype=torch.float32).pin_memory()
        self._ring_f32 = self._ring.numpy()
        self._ring_i32 = self._ring_f32.view(np.int32)
        with torch.cuda.device(dev):
            _lib.check(self.model.lib.stb_set_loss_ring(self.model.ctx, _lib.ptr(self._ring), self.RING_SLOTS))
        # iterations run on a dedicated (non-legacy) stream so that the library can replay them as a CUDA graph
        self._stream = torch.cuda.Stream(device=dev)
        self.last_loss_terms = None
        # one process per GPU under torch.distributed: large scales are tiled spatially over the ranks.
        # `distributed`: None = the torch.distributed default group if initialised, False = never tile, or a group
        # object (distributed.TorchGroup / ThreadGroup).
        if shared is not None:
            self._group = D.ThreadGroup(shared, 0)
        elif distributed is None or distributed is True:
            self._group = D.default_group()
        elif distributed is False:
            self._group = None
        else:
            self._group = distributed
        self._dist = self._group is not None and self._group.world > 1
        self._rank = self._group.rank if self._dist else 0
        self._world = self._group.world if self._dist else 1
        # 'peer': tiled scales iterate with the exchanges inside the library; 'off': the ranks could not map each
        # other's memory, so every scale runs replicated
        self._comm_mode = 'peer'
        # 'halo': a band computes its own rows only and pulls one boundary row per layer from its neighbours (their
        # workspaces are mapped); 'apron': it recomputes 80-row aprons instead (no per-layer exchange); 'auto' (default):
        # per scale, halo rows when the image is at least HALO_MIN_WIDTH wide.  Measured (DESIGN.md section 6): the ~28
        # exchanges of an iteration cost ~0.36 ms whatever the size, the aprons 160 rows x W of convolution work
        # (~1.7e-4 ms per pixel of width): 0.34 ms at W = 2048 (aprons win), 0.69 ms at W = 4096 (halo rows win).
        self._tile_mode = os.environ.get('STB_TILE', 'auto')
        self._halo_now = False
        self._comm_cap = None
        self._shared_cap = 0
        self._band = None
        self._verbose = True
        self._sync = None    # _Lockstep of the in-process ranks while stylize() runs
        # rank 1 of StyleTransfer(devices=[a, b]): the same single-device machinery on the second device, driven by
        # stylize() on a thread of its own
        self._peer = None
        if shared is not None:
            self._peer = StyleTransfer([self.devices[1]], pooling, vgg_weights=vgg_weights,
                                       distributed=D.ThreadGroup(shared, 1))
            self._peer._verbose = False

    # ------------------------------------------------------------------ results
    def get_image_tensor(self):
        self._stream.synchronize()   # iterations run on the library's stream; the EMA must be complete before it is read
        value = self.average.get().detach()
        if self._band is not None:   # tiled scale in flight: the average holds this rank's rows only (collective call)
            if self._sync is not None and self._rank == 0:
                self._sync.request_gather()   # the in-process rank 1 joins the gather (_Lockstep)
            value = D.gather_rows(value, self._band, self._group)
        return value[0].clamp(0, 1)

    def _snapshot(self, kind, gathered=None):
        """The averaged image quantised on the device by stb_snapshot, as an [H, W, 3] tensor ready on the current
        stream: kind 0 uint8 (to_pil_image's mul(255).byte()), kind 1 uint16 (np.uint16(np.round(x * 65535))).

        Untiled, the kernel reads the EMA's storage on the iteration stream, ordered after the iterations, with no host
        synchronisation and no fp32 temporary.  On a banded scale the image is first gathered by get_image_tensor()
        (collective), and the gathered image, already bias-corrected, is quantised with denom = 1.  `gathered`: an
        image get_image_tensor() has already returned at this iteration, quantised instead of gathering again."""
        if gathered is not None:
            src, denom = gathered, 1.0
        elif self._band is not None:
            src, denom = self.get_image_tensor(), 1.0
        else:
            src, denom = self.average.value, 1 - self.average.accum
        h, w = src.shape[-2:]
        cur = torch.cuda.current_stream(self._dev)
        with torch.cuda.device(self._dev), torch.cuda.stream(self._stream):
            self._stream.wait_stream(cur)
            out = torch.empty(h, w, 3, dtype=(torch.uint8, torch.uint16)[kind], device=self._dev)
            _lib.check(self.model.lib.stb_snapshot(_lib.ptr(src), h, w, denom, kind, _lib.ptr(out),
                                                   _lib.cur_stream()))
        cur.wait_stream(self._stream)
        return out

    def get_image(self, image_type='pil'):
        if self.average is None:
            return None
        kind = image_type.lower()
        if kind == 'pil':
            return Image.fromarray(self._snapshot(0).cpu().numpy())
        if kind == 'np_uint16':
            return self._snapshot(1).cpu().numpy()
        raise ValueError("image_type must be 'pil' or 'np_uint16'")

    # ------------------------------------------------------------------ helpers
    def _initial_image(self, init, content_image, style_images, style_weights, cw, ch):
        if init == 'gray':
            return torch.rand([1, 3, ch, cw]) / 255 + 0.5
        if init == 'uniform':
            return torch.rand([1, 3, ch, cw])
        if init == 'normal':
            image = torch.empty([1, 3, ch, cw])
            torch.nn.init.trunc_normal_(image, mean=0.5, std=0.25, a=0, b=1)
            return image
        if init == 'style_stats':
            means, variances = 0, 0
            for weight, simg in zip(style_weights, style_images):
                t = _pil_to_tensor(simg)[0]
                means = means + t.mean(dim=(1, 2)) * weight
                variances = variances + t.var(dim=(1, 2)) * weight
            planes = []
            for mean, variance in zip(means, variances):
                plane = torch.empty([1, 1, ch, cw])
                torch.nn.init.trunc_normal_(plane, mean=mean, std=variance.sqrt(), a=0, b=1)
                planes.append(plane)
            return torch.cat(planes, dim=1)
        raise ValueError("init must be one of 'content', 'gray', 'uniform', 'style_mean'")

    def _iterate(self, exp_avg, exp_avg_sq, step, lr, avg_decay, want_loss):
        m = self.model
        _lib.check(m.lib.stb_iterate(m.ctx, _lib.ptr(self.image), _lib.ptr(exp_avg), _lib.ptr(exp_avg_sq),
                                     _lib.ptr(self.average.value), step, lr, 0.9, 0.99, 1e-8, avg_decay,
                                     _lib.ptr(self._loss_host) if want_loss else None, _lib.cur_stream()))
        self.average.note_update()

    def _iterate_banded(self, band, stats, grad, exp_avg, exp_avg_sq, step, lr, avg_decay):
        """One iteration of a spatially tiled scale: one library call = one CUDA graph holding the compute AND the
        three exchanges (kernels reading the peers' mailboxes over NVLink, csrc/comm.cu)."""
        # band, stats and grad are unused: the library holds the band geometry, the statistics block and the gradient.
        # They stay in the signature because bench.py calls this positionally.
        self.model.iterate_banded(self.image, exp_avg, exp_avg_sq, self.average.value, step, lr, avg_decay,
                                  self._loss_host)
        self.average.note_update()

    def _ensure_peer_memory(self, ws_sizes, cap_h, cap_w):
        """Collective over the ranks, before the first tiled scale touches the workspace: the mailboxes (bands up to
        cap_h x cap_w) and, in halo mode, the library-owned workspace (every (h, w) of ws_sizes fits) exist and are
        mapped by the peers."""
        g, m = self._group, self.model
        if self._comm_mode == 'peer' and (self._comm_cap is None or self._comm_cap[0] < cap_h or self._comm_cap[1] < cap_w):
            ok, mine, err = True, None, None
            try:
                if self._comm_cap is not None:
                    m.comm_disconnect()          # nobody may still map a mailbox that is about to be freed
            except _lib.NativeError as e:
                ok, err = False, e
            g.barrier()
            try:
                handle, pointer = m.comm_create(self._rank, self._world, cap_h, cap_w)
                mine = handle if g.peer_kind == 'ipc' else pointer
            except _lib.NativeError as e:
                ok, err = False, e
            infos = g.all_gather_object((ok, mine))       # every rank takes the same branch from here on
            if all(i[0] for i in infos):
                try:
                    if g.peer_kind == 'ipc':
                        m.comm_connect_ipc([i[1] for i in infos])
                    else:
                        m.comm_connect_local([i[1] for i in infos])
                except _lib.NativeError as e:
                    ok, err = False, e
            else:
                ok = False
            if all(g.all_gather_object(ok)):
                self._comm_cap = (cap_h, cap_w)
            elif self._sync is not None:    # in-process ranks have no NCCL: the driver runs the job untiled
                raise _PeerUnavailable(err)
            else:
                warnings.warn(f'peer-memory exchange unavailable on some rank ({err}); running the tiled scales '
                              'replicated')
                self._comm_mode = 'off'
        if self._comm_mode != 'peer' or self._tile_mode == 'apron' or not self._wants_halo(cap_w):
            return
        need = max(m.workspace_bytes(h, w) for h, w in ws_sizes) + 4096
        grow = need > self._shared_cap
        if any(g.all_gather_object(grow)):      # all ranks re-create together (a neighbour may map what is freed)
            ok, mine, err = True, None, None
            try:
                if self._shared_cap:
                    m.release_shared_workspace(unmap_only=True)
                g.barrier()
                if self._shared_cap:
                    m.release_shared_workspace(unmap_only=False)
                handle, pointer = m.alloc_shared_workspace(ws_sizes)
                mine = handle if g.peer_kind == 'ipc' else pointer
            except _lib.NativeError as e:
                ok, err = False, e
            infos = g.all_gather_object((ok, mine))
            if all(i[0] for i in infos):
                try:
                    m.connect_shared_workspaces([i[1] for i in infos], g.peer_kind == 'ipc')
                except _lib.NativeError as e:
                    ok, err = False, e
            else:
                ok = False
            if all(g.all_gather_object(ok)):
                self._shared_cap = max(need, m._ws_bound)
            else:
                warnings.warn(f'peer-mapped workspace unavailable on some rank ({err}); tiling with recomputed aprons')
                self._tile_mode = 'apron'
                self._shared_cap = 0
                if m._ws_shared:
                    g.barrier()
                    m.release_shared_workspace(unmap_only=False)

    HALO_MIN_WIDTH = 2400

    def _wants_halo(self, w):
        return self._tile_mode == 'halo' or (self._tile_mode == 'auto' and w >= self.HALO_MIN_WIDTH)

    def _setup_comm(self, band, w):
        """Per tiled scale (collective): zero the iteration stamps between two barriers, hand the band geometry to the
        library."""
        g, m = self._group, self.model
        bands = D.all_bands(band.H, self._world)
        g.barrier()
        m.comm_reset()
        g.barrier()
        up = bands[self._rank - 1] if self._rank > 0 else None
        down = bands[self._rank + 1] if self._rank + 1 < self._world else None
        self._halo_now = bool(self._wants_halo(w) and m._ws_shared and self._shared_cap)
        m.comm_set_geometry(w, band, up, down, self._halo_now)

    def _style_stats(self, simg, sh, sw):
        """(means, second raw moments) of one style image (ST:440-443) at sw x sh: a [1,3,sh,sw] tensor, or a
        SourceImage, of which only the rows that are needed are resampled.  Under torch.distributed a large style image
        is tiled like the iterate: every rank runs its band, the raw sums are all-reduced once (per scale, not per
        iteration), and the global pixel counts normalise them."""
        m = self.model
        band = D.make_band(sh, self._rank, self._world) if self._dist else None
        if band is None:
            m.set_band(False)
            return m.style_stats(simg.resized(sw, sh) if isinstance(simg, SourceImage) else simg)
        m.set_band(True, sh, band.own0, band.own_rows)
        if isinstance(simg, SourceImage):
            local = simg.resized(sw, sh, band.loc_begin, band.h_local)
        else:
            local = D.local_slice(simg, band)
        means, srms = m.style_stats(local)      # RAW sums over this band's own rows
        m.set_band(False)
        if not means:
            return means, srms
        flat = torch.cat([t.flatten() for t in means + srms])
        self._group.all_reduce_sum(flat)
        counts = D.tap_pixel_counts(sh, sw, m.style_layers)
        out, off = [], 0
        for t in means + srms:
            out.append(flat[off:off + t.numel()].view_as(t))
            off += t.numel()
        n = len(means)
        means = [t / c for t, c in zip(out[:n], counts)]
        srms = [t / c for t, c in zip(out[n:], counts)]
        return means, srms

    def _wait_loss(self, step):
        """Loss terms of iteration `step` as soon as the device has published them (before its backward pass): polls the
        stamp of the ring slot in pinned host memory -- no stream synchronisation, the rest of the iteration and the
        launch of the next one overlap the callback."""
        slot = step % self.RING_SLOTS
        stamp = self._ring_i32[slot]
        t0 = None
        while stamp[8] != step:
            if t0 is None:
                t0 = time.perf_counter()
            elif time.perf_counter() - t0 > float(os.environ.get('STB_LOSS_TIMEOUT_S', '120')):
                raise _lib.NativeError(f'iteration {step}: the device never published its loss (stamp {int(stamp[8])})')
        # term k sits in word k below the stamp (word 8) and in word k + 1 above it
        n = self.model.n_terms
        words = self._ring_f32[slot, :8] if n <= 8 else np.concatenate([self._ring_f32[slot, :8],
                                                                         self._ring_f32[slot, 9:n + 1]])
        return torch.from_numpy(words[:n].copy())

    def loss_and_grad(self):
        """Closure of ST:472-476 evaluated natively on the current image: returns (host tensor of the loss terms
        [total, content terms, style terms, tv] of the layer table, grad)."""
        m = self.model
        grad = torch.empty_like(self.image)
        _lib.check(m.lib.stb_iterate_ex(m.ctx, _lib.ptr(self.image), None, None, None, 0, 0.0, 0.9, 0.99, 1e-8, 0.0, 0,
                                        _lib.ptr(grad), _lib.ptr(self._loss_host), _lib.cur_stream()))
        torch.cuda.current_stream().synchronize()
        if m.n_terms <= 8:
            return self._loss_host[:m.n_terms].clone(), grad
        return m.loss_terms(), grad

    # ------------------------------------------------------------------ the driver
    def stylize(self, content_image, style_images, *,
                style_weights=None,
                content_weight: float = 0.015,
                tv_weight: float = 2.,
                optimizer: str = 'adam',
                min_scale: int = 128,
                end_scale: int = 512,
                iterations: int = 500,
                initial_iterations: int = 1000,
                step_size: float = 0.02,
                avg_decay: float = 0.99,
                init: str = 'content',
                style_scale_fac: float = 1.,
                style_size: int = None,
                callback=None):
        """ST:349-493.  With two devices (StyleTransfer(devices=[a, b])) the second rank runs on a thread of its own
        for the duration of the call, during which cyclic garbage collection is switched off (gc.disable) and, on the
        main thread, Ctrl-C takes effect at the next iteration boundary rather than at once."""
        kw = dict(style_weights=style_weights, content_weight=content_weight, tv_weight=tv_weight,
                  optimizer=optimizer, min_scale=min_scale, end_scale=end_scale, iterations=iterations,
                  initial_iterations=initial_iterations, step_size=step_size, avg_decay=avg_decay, init=init,
                  style_scale_fac=style_scale_fac, style_size=style_size)
        if self._peer is not None:
            return self._stylize_devices(content_image, style_images, callback, kw)
        return self._stylize(content_image, style_images, callback=callback, **kw)

    def _stylize_devices(self, content_image, style_images, callback, kw):
        """stylize() of StyleTransfer(devices=[a, b]): rank 0 runs on the caller's thread (the user's callback runs
        there, with the whole image), rank 1 (self._peer) on a thread of its own; both run _stylize in lockstep
        (_Lockstep).  The first error of either rank stops both and is raised here, after rank 1's thread is joined and
        the whole image of the stopped iteration is back in self.average."""
        peer, shared = self._peer, self._group.shared
        # rank 1 is an object of its own: it runs the layers set on this one
        peer.content_layers = list(self.content_layers)
        peer.style_layers = list(self.style_layers)
        peer.style_weights = list(self.style_weights)
        if self._dev != peer._dev and not torch.cuda.can_device_access_peer(self._dev, peer._dev):
            return self._stylize_untiled(f'{self._dev} cannot access {peer._dev} peer to peer', content_image,
                                         style_images, callback, kw)
        sync = _Lockstep()
        errors, lock = [], threading.Lock()

        def fail(e):
            with lock:
                errors.append(e)
            sync.stop()
            shared.bar.abort()    # releases a rank waiting in a per-scale collective

        def rank1():
            try:
                torch.cuda.set_device(peer._dev)
                # no callback: rank 1's loss is read by nobody (the images do not depend on it)
                peer._stylize(content_image, style_images, callback=None, **kw)
            except BaseException as e:  # noqa: BLE001 -- re-raised on the caller's thread
                fail(e)

        result = None
        thread = threading.Thread(target=rank1, name='stb-rank1')
        gc_enabled = gc.isenabled()
        with _deferred_sigint(sync):
            try:
                shared.bar.reset()
                self._sync = peer._sync = sync
                # no cyclic garbage collection while the ranks run: a finalizer that frees device memory synchronises
                # the device, and run on one rank's thread while an iteration of the other waits for this rank it
                # would stall both
                gc.collect()
                gc.disable()
                thread.start()
                result = self._stylize(content_image, style_images, callback=callback, **kw)
            except BaseException as e:  # noqa: BLE001 -- re-raised below, once rank 1 has stopped
                fail(e)
            finally:
                if thread.ident is not None:
                    thread.join()
                self._sync = peer._sync = None
                if gc_enabled:
                    gc.enable()
            if errors:
                try:
                    self._stitch_stopped_bands()
                except BaseException as e:  # noqa: BLE001 -- the first error is the one to report
                    errors.append(e)
            else:
                sync.deliver_interrupt()    # a SIGINT that came after rank 0's last gate
        if errors and isinstance(errors[0], _PeerUnavailable):
            return self._stylize_untiled(str(errors[0]), content_image, style_images, callback, kw)
        if errors:
            raise errors[0]
        return result

    def _stitch_stopped_bands(self):
        """After a two-device run stopped on a banded scale: rank 0's EMA becomes the whole image again, rank 1's own
        rows copied in directly.  Both threads have returned and both streams are drained, so nothing changes those rows
        any more, and both ranks launched the same iterations, so they are of the same step as rank 0's."""
        peer, band, pband = self._peer, self._band, self._peer._band
        self._band = peer._band = None
        if band is None:
            return
        with torch.cuda.device(self._dev):
            self._stream.synchronize()
            peer._stream.synchronize()
            self.model.set_band(False)
            if pband is None or pband.H != band.H:   # rank 1 stopped before it held rows of this scale
                self.average = None
                return
            own = [self.average.value[:, :, band.own0:band.own0 + band.own_rows],
                   peer.average.value[:, :, pband.own0:pband.own0 + pband.own_rows].to(self._dev)]
            self.average = EMA.from_state(torch.cat(own, dim=2), self.average.accum, self.average.decay)
            self.image = self.average.get()

    def _stylize_untiled(self, why, content_image, style_images, callback, kw):
        """The job on the first device alone, rank 1 idle: the in-process ranks cannot map each other's memory, and they
        have no NCCL to fall back on.  When the mapping failed only at the first banded scale, the job restarts: the
        callback sees the iterations of the smaller scales again."""
        warnings.warn(f'peer-memory exchange between {self._dev} and {self._peer._dev} unavailable ({why}); '
                      f'running untiled on {self._dev}')
        group = self._group
        self._group, self._dist, self._world = None, False, 1
        try:
            return self._stylize(content_image, style_images, callback=callback, **kw)
        finally:
            self._group, self._dist, self._world = group, True, 2

    def _stylize(self, content_image, style_images, *, style_weights, content_weight, tv_weight, optimizer, min_scale,
                 end_scale, iterations, initial_iterations, step_size, avg_decay, init, style_scale_fac, style_size,
                 callback):
        dev = self._dev
        min_scale = min(min_scale, end_scale)
        if style_weights is None:
            style_weights = [1 / len(style_images)] * len(style_images)
        else:
            norm = sum(abs(w) for w in style_weights)
            style_weights = [w / norm for w in style_weights]
        if len(style_images) != len(style_weights):
            raise ValueError('style_images and style_weights must have the same length')
        if optimizer not in ('adam', 'lbfgs'):
            raise ValueError("optimizer must be one of 'adam', 'lbfgs'")
        per_content_weight = content_weight / len(self.content_layers)
        # the layer attributes are read once per call (the reference re-reads them per scale): loss terms are
        # zip(content_layers, content_weights) and zip(style_layers, style_weights) (ST:427, 451), so entries of
        # style_layers without a weight, or weights without a layer, drop out
        content_layers, style_layers = list(self.content_layers), list(self.style_layers)
        check_layers(content_layers, style_layers)
        layer_weights = [float(w) for w in self.style_weights][:len(style_layers)]
        style_layers = style_layers[:len(layer_weights)]
        content_weights = [per_content_weight] * len(content_layers)
        self.model.set_layers(content_layers, style_layers)

        scales = gen_scales(min_scale, end_scale)
        cw, ch = size_to_fit(content_image.size, scales[0], scale_up=True)
        # the full-size images go to the device once; every scale resamples them there
        content_src = SourceImage(content_image, dev)
        style_srcs = [SourceImage(simg, dev) for simg in style_images]
        if init == 'content':
            self.image = content_src.resized(cw, ch)
        else:
            self.image = self._initial_image(init, content_image, style_images, style_weights, cw, ch).to(dev)
            if self._dist:  # random inits are drawn per process: every rank continues from rank 0's draw
                self._group.broadcast(self.image, 0)

        exp_avg = exp_avg_sq = None
        step = 0
        lbfgs_state = None
        self._stream.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.device(dev), torch.cuda.stream(self._stream), torch.no_grad():
            for scale in scales:
                torch.cuda.empty_cache()

                cw, ch = size_to_fit(content_image.size, scale, scale_up=True)
                styles = []
                for simg, src in zip(style_images, style_srcs):
                    if style_size is None:
                        sw, sh = size_to_fit(simg.size, round(scale * style_scale_fac))
                    else:
                        sw, sh = size_to_fit(simg.size, style_size)
                    styles.append((sw, sh, src))
                # multi-GPU: tile this scale into horizontal bands (None: too small, or the ranks cannot map each
                # other's memory: every rank runs the whole image)
                tiled = self._dist and self._comm_mode == 'peer'
                band = D.make_band(ch, self._rank, self._world) if tiled else None
                h_loc = band.h_local if band is not None else ch
                self.model.set_band(False)
                self._band = None
                style_sizes = []
                for sw, sh, _ in styles:   # a tiled style image needs room for its band only
                    sb = D.make_band(sh, self._rank, self._world) if self._dist else None
                    style_sizes.append((sb.h_local if sb is not None else sh, sw))
                if band is not None:
                    # mailboxes / peer-mapped workspace are sized once, for the largest scale of this call (the last)
                    ew, eh = size_to_fit(content_image.size, scales[-1], scale_up=True)
                    eb = D.make_band(eh, self._rank, self._world)
                    cap_h = max(b.h_local for b in D.all_bands(eh, self._world))
                    end_sizes = [(eb.h_local if eb is not None else eh, ew)]
                    for simg in style_images:   # style sizes of the last scale (they grow with the scale)
                        if style_size is None:
                            lw, lh = size_to_fit(simg.size, round(scales[-1] * style_scale_fac))
                        else:
                            lw, lh = size_to_fit(simg.size, style_size)
                        lb = D.make_band(lh, self._rank, self._world)
                        end_sizes.append((lb.h_local if lb is not None else lh, lw))
                    self._ensure_peer_memory([(h_loc, cw)] + style_sizes + end_sizes, max(cap_h, h_loc), max(ew, cw))
                    if self._comm_mode != 'peer':   # the peer mapping failed on some rank
                        band, h_loc = None, ch
                self.model.ensure_workspace([(h_loc, cw)] + style_sizes)

                self.image = self.model.resize(self.image, (ch, cw), 'bicubic', 'clamp')          # ST:420
                if band is not None:   # the band's rows only: the full-height content tensor is never formed
                    self.image = D.local_slice(self.image, band)
                    content = content_src.resized(cw, ch, band.loc_begin, band.h_local)
                else:
                    content = content_src.resized(cw, ch)
                self.average = EMA(self.image, avg_decay)
                self._band = band   # from here on the average holds the band's rows only

                if self._verbose:
                    print(f'Processing content image ({cw}x{ch})...')
                content_targets = self.model.content_features_list(content)
                means = srms = None
                for weight, (sw, sh, simg) in zip(style_weights, styles):
                    if self._verbose:
                        print(f'Processing style image ({sw}x{sh})...')
                    m_i, s_i = self._style_stats(simg, sh, sw)
                    if means is None:
                        means = [m * weight for m in m_i]
                        srms = [s * weight for s in s_i]
                    else:
                        for acc, m in zip(means, m_i):
                            acc.add_(m * weight)
                        for acc, s in zip(srms, s_i):
                            acc.add_(s * weight)
                if band is not None:
                    self.model.set_band(True, ch, band.own0, band.own_rows)
                self.model.set_targets_list(h_loc, cw, content_targets, content_weights, means, srms, layer_weights,
                                            tv_weight)
                if band is not None:
                    self._setup_comm(band, cw)

                if optimizer == 'adam':
                    if exp_avg is None:
                        exp_avg = torch.zeros_like(self.image)
                        exp_avg_sq = torch.zeros_like(self.image)
                    else:  # warm start at the new size, step counter carried over (ST:285-295, 460-462)
                        exp_avg = self.model.resize(exp_avg, (ch, cw), 'bicubic')
                        exp_avg_sq = self.model.resize(exp_avg_sq, (ch, cw), 'bilinear', 'relu')
                    if band is not None and exp_avg.shape[2] != h_loc:
                        exp_avg, exp_avg_sq = D.local_slice(exp_avg, band), D.local_slice(exp_avg_sq, band)
                else:
                    lbfgs_state = None   # hand the previous scale's block back before the new one is allocated
                    lbfgs_state = self._lbfgs_state(band.own_rows if band is not None else ch, cw)
                torch.cuda.empty_cache()

                actual_its = initial_iterations if scale == scales[0] else iterations
                sync = self._sync
                for i in range(1, actual_its + 1):
                    if sync is not None:
                        sync.before_launch(self, step + 1)
                    if optimizer == 'adam' and band is not None:
                        step += 1
                        self._iterate_banded(band, None, None, exp_avg, exp_avg_sq, step, step_size, avg_decay)
                    elif optimizer == 'adam':
                        step += 1
                        self._iterate(exp_avg, exp_avg_sq, step, step_size, avg_decay, callback is not None)
                    elif band is not None:
                        step += 1
                        self._iterate_lbfgs_banded(lbfgs_state, step, avg_decay)
                    else:
                        step += 1
                        self._iterate_lbfgs(lbfgs_state, step, avg_decay)
                    if sync is not None:
                        sync.after_launch(self, step)
                    if callback is not None:
                        # host-side bookkeeping first: it overlaps the iteration still running on the device (the
                        # native path allocates nothing, so the high-water mark cannot move before the sync)
                        gpu_ram = 0
                        for device in self.devices:
                            if device.type == 'cuda':
                                gpu_ram = max(gpu_ram, torch.cuda.max_memory_allocated(device))
                        # the reference syncs here (loss.item()); this waits for the loss only
                        self.last_loss_terms = self._wait_loss(step)
                        loss_value = float(self.last_loss_terms[0])
                        callback(STIterate(w=cw, h=ch, i=i, i_max=actual_its, loss=loss_value, time=time.time(),
                                           gpu_ram=gpu_ram))
                    if sync is not None:
                        sync.after_iteration(self, step)
                if sync is not None:
                    sync.end_of_scale(self, step)

                if band is not None:  # stitch the bands back together (identical full tensors on every rank)
                    g = self._group
                    self.average = EMA.from_state(D.gather_rows(self.average.value, band, g), self.average.accum,
                                                  avg_decay)
                    self._band = None
                    if optimizer == 'adam':   # L-BFGS starts afresh every scale: it has no state to carry
                        exp_avg, exp_avg_sq = D.gather_rows(exp_avg, band, g), D.gather_rows(exp_avg_sq, band, g)
                    self.image = self.average.get()
                    self.model.set_band(False)
                else:
                    self.image.copy_(self.average.get())
            self._stream.synchronize()

        return self.get_image()

    # ------------------------------------------------------------------ L-BFGS (ST:464-465): closure, torch's
    # LBFGS.step (max_iter=1, history_size=10) and the EMA run natively as one CUDA graph per iteration (csrc/lbfgs.cu)
    def _lbfgs_state(self, h, w):
        """Fresh optimizer state for one scale (the reference builds a new optim.LBFGS per scale): a torch-owned block
        of ~25 x 3HW floats (history ring, g, g_prev, d), so that max_memory_allocated stays truthful.  On a tiled
        scale h is the band's own rows: each rank keeps the vectors of its own rows only."""
        lib = self.model.lib
        n = ctypes.c_size_t()
        _lib.check(lib.stb_lbfgs_state_bytes(h, w, ctypes.byref(n)))
        state = torch.empty(n.value, dtype=torch.uint8, device=self._dev)
        _lib.check(lib.stb_lbfgs_reset(_lib.ptr(state), h, w, _lib.cur_stream()))
        return state

    def _iterate_lbfgs(self, state, step, avg_decay):
        """One L-BFGS iteration with no host sync; its loss is published to the loss ring under stamp `step`."""
        m = self.model
        _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(self.image), _lib.ptr(self.average.value), _lib.ptr(state),
                                           state.numel(), step, avg_decay, None, _lib.cur_stream()))
        self.average.note_update()

    def _iterate_lbfgs_banded(self, state, step, avg_decay):
        """One L-BFGS iteration of a tiled scale ('peer' mode): one CUDA graph with the compute, the exchanges and the
        cross-rank reductions of the step; the loss goes to the loss ring like the untiled one's."""
        m = self.model
        _lib.check(m.lib.stb_iterate_lbfgs_banded(m.ctx, _lib.ptr(self.image), _lib.ptr(self.average.value),
                                                  _lib.ptr(state), state.numel(), step, avg_decay, None,
                                                  _lib.cur_stream()))
        self.average.note_update()
