"""Cost of bringing the content and style images to a scale: the device resampler (stb_resample_rgb8) against the host
path it replaces (Image.resize, upload, convert), per call and over whole stylize() runs.

  python tools/setup_bench.py [--reps 20] [--pairs 3] [--skip-e2e] [--out DIR]

Seeded synthetic sources (block noise enlarged, as BASELINE.md section 3 builds its inputs), one style image.
  * per call, a 6000x4000 source to 128, 512, 2048 and 4096 wide: time of the two kernels from CUDA events over `reps`
    launches with the tables already on the device, the bytes they must move (the source rows read once, the horizontal
    result written and read, 12 B per output pixel) over that time, the wall time of SourceImage.resized() (tables built
    and uploaded, kernels, synchronise), and the wall time of the host expression on this machine's CPU;
  * end to end, a 4000x3000 content and a 6000x4000 style: stylize() with the CLI defaults (128 -> 512, 1000 + 4 x 500
    iterations) and with end_scale=2048, iterations=100, initial_iterations=200, callback=None, wall clock with a final
    synchronise, device path and host path alternated `pairs` times; the host path is the holder built without its
    device copy, which is the path images of other modes take;
  * per-scale setup time of both paths, from the end of a scale's last iteration (synchronised) to the point where the
    next scale's first iteration can be launched with all set-up work on the device finished, in one short run each.
The card's name, power limit and maximum SM clock are read in the same run.  One GPU only.  Prints one JSON line.
"""
import argparse
import contextlib
import ctypes
import io
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch
from PIL import Image

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200 import _lib  # noqa: E402
from style_transfer_b200 import style_transfer as ST  # noqa: E402
from oracle import st_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'nvidia-smi unavailable ({e})'


def stats(xs):
    return dict(median=float(np.median(xs)), min=float(min(xs)), max=float(max(xs)))


def bench_call(img, w, reps):
    ws, hs = img.size
    w, h = ST.size_to_fit(img.size, w, scale_up=True)
    holder = ST.SourceImage(img, DEV)
    lib = _lib.load()
    kx, bx = (torch.from_numpy(t).to(DEV) for t in ST.resample_coeffs(ws, w))
    ky, by = (torch.from_numpy(t).to(DEV) for t in ST.resample_coeffs(hs, h))
    need = ctypes.c_size_t()
    _lib.check(lib.stb_resample_tmp_bytes(hs, ws, h, w, 0, h, ctypes.byref(need)))
    tmp = torch.empty(need.value, dtype=torch.uint8, device=DEV)
    out = torch.empty(1, 3, h, w, device=DEV)

    def launch():
        _lib.check(lib.stb_resample_rgb8(_lib.ptr(holder.data), hs, ws, h, w, 0, h, _lib.ptr(kx), _lib.ptr(bx),
                                         kx.shape[1], _lib.ptr(ky), _lib.ptr(by), ky.shape[1], _lib.ptr(tmp),
                                         need.value, _lib.ptr(out), _lib.cur_stream()))

    for _ in range(3):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / reps
    ref = ST._pil_to_tensor(img.resize((w, h), Image.BICUBIC), DEV)
    assert torch.equal(out, ref), 'the device result differs from Pillow'
    moved = hs * ws * 3 + 2 * need.value + 12 * h * w

    device_ms, host_ms = [], []
    for _ in range(5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        holder.resized(w, h)
        torch.cuda.synchronize()
        device_ms.append(1e3 * (time.perf_counter() - t0))
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ST._pil_to_tensor(img.resize((w, h), Image.BICUBIC), DEV)
        torch.cuda.synchronize()
        host_ms.append(1e3 * (time.perf_counter() - t0))
    return dict(source=[ws, hs], to=[w, h], kernels_us=us, modelled_bytes=moved, GB_per_s=moved / us / 1e3,
                resized_call_ms=stats(device_ms), host_resize_upload_convert_ms=stats(host_ms))


def host_init(self, img, device):
    """SourceImage without its device copy: resized() then takes the host path (Image.resize, upload, convert)."""
    self.img, self.device, self.data = img, device, None


@contextlib.contextmanager
def path(kind):
    init = ST.SourceImage.__init__
    if kind == 'host':
        ST.SourceImage.__init__ = host_init
    try:
        yield
    finally:
        ST.SourceImage.__init__ = init


def run(st, content, style, kw, callback=None):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(content, [style], callback=callback, **kw)
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def setup_times(st, content, style, kw):
    """Seconds between the end of a scale and the first iteration of the next, per scale boundary."""
    ends, starts, state = [], [], dict(fresh=False)
    inner = st._iterate

    def iterate(*a):
        if state['fresh']:
            st._stream.synchronize()
            starts.append(time.perf_counter())
            state['fresh'] = False
        return inner(*a)

    def cb(it):
        if it.i == it.i_max:
            st._stream.synchronize()
            ends.append(time.perf_counter())
            state['fresh'] = True

    st._iterate = iterate
    try:
        run(st, content, style, dict(kw, iterations=10, initial_iterations=10), cb)
    finally:
        del st._iterate
    return [s - e for s, e in zip(starts, ends)]


def bench_e2e(name, kw, pairs, wts, content, style):
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    res = dict(config=name, scales=ST.gen_scales(kw['min_scale'], kw['end_scale']))
    with path('device'):
        run(st, content, style, dict(kw, iterations=3, initial_iterations=3))     # loads kernels, captures graphs
    wall = dict(device=[], host=[])
    for _ in range(pairs):
        for kind in ('device', 'host'):
            with path(kind):
                wall[kind].append(run(st, content, style, kw))
    res['wall_s'] = {k: stats(v) for k, v in wall.items()}
    for kind in ('device', 'host'):
        with path(kind):
            res[f'setup_ms_per_scale_boundary_{kind}'] = [round(1e3 * t, 2) for t in setup_times(st, content, style, kw)]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--pairs', type=int, default=3)
    ap.add_argument('--skip-e2e', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('setup_bench: no CUDA device (timings exist only on the GPU)')
    content, style = O.synth_image(1, 64, 4000, 3000), O.synth_image(2, 64, 6000, 4000)
    line = dict(card=card(), per_call=[bench_call(style, w, args.reps) for w in (128, 512, 2048, 4096)])
    if not args.skip_e2e:
        wts = O.make_vgg_weights(1234)
        line['end_to_end'] = [
            bench_e2e('cli defaults', dict(min_scale=128, end_scale=512, iterations=500, initial_iterations=1000),
                      args.pairs, wts, content, style),
            bench_e2e('end_scale=2048', dict(min_scale=128, end_scale=2048, iterations=100, initial_iterations=200),
                      args.pairs, wts, content, style)]
    print(json.dumps(line), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'setup_bench.json').write_text(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
