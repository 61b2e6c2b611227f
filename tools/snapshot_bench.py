"""Cost of saving the averaged image: the stb_snapshot kernel, get_image('np_uint16') and a `.tif` periodic save.

  python tools/snapshot_bench.py [--sizes 2048 4096] [--reps 20] [--out DIR]

Per size (square, single scale, synthetic images):
  * kernel time of stb_snapshot, uint8 and uint16, from CUDA events over `reps` launches, with the bytes it moves
    (12 B read + 3 / 6 B written per pixel) over that time;
  * wall time of get_image('np_uint16') against the expression it replaced (a full fp32 device-to-host copy, then
    multiply, round and cast in numpy), alternated, medians;
  * host time spent inside AsyncImageWriter.submit_snapshot for a `.tif` path, called from the callback of a running
    stylize() every other iteration.
The card's name and power limit are read in the same run.  Prints one JSON line.
"""
import argparse
import contextlib
import io
import json
import subprocess
import sys
import tempfile
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200 import _lib  # noqa: E402
from style_transfer_b200.image_io import AsyncImageWriter  # noqa: E402
from oracle import st_oracle as O  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'nvidia-smi unavailable ({e})'


def old_np_uint16(st):
    st._stream.synchronize()
    image = st.average.get().detach()[0].clamp(0, 1)
    return np.uint16(np.round(image.cpu().movedim(0, 2).numpy() * 65535))


def bench_size(size, reps, wts):
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    writer = AsyncImageWriter()
    submit_ms = []
    with tempfile.TemporaryDirectory() as tmp:
        path = Path(tmp) / 'snap.tif'

        def cb(it):
            if it.i % 2 == 0:
                t0 = time.perf_counter()
                writer.submit_snapshot(st, path)
                submit_ms.append(1e3 * (time.perf_counter() - t0))

        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=reps + 4,
                       callback=cb)
        writer.close()
    submit_ms = submit_ms[2:]   # the first calls allocate the pinned buffers

    h, w = st.average.value.shape[-2:]
    res = dict(size=size, submit_snapshot_tif_host_ms=dict(median=float(np.median(submit_ms)),
                                                           max=float(max(submit_ms)), calls=len(submit_ms)))
    lib, stream = st.model.lib, st._stream
    denom = 1 - st.average.accum
    for kind, name, out_b in ((0, 'uint8', 3), (1, 'uint16', 6)):
        out = torch.empty(h, w, 3, dtype=(torch.uint8, torch.uint16)[kind], device='cuda')
        with torch.cuda.stream(stream):
            for _ in range(3):
                _lib.check(lib.stb_snapshot(_lib.ptr(st.average.value), h, w, denom, kind, _lib.ptr(out),
                                            _lib.cur_stream()))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(reps):
                _lib.check(lib.stb_snapshot(_lib.ptr(st.average.value), h, w, denom, kind, _lib.ptr(out),
                                            _lib.cur_stream()))
            e1.record(stream)
        e1.synchronize()
        us = 1e3 * e0.elapsed_time(e1) / reps
        res[f'kernel_{name}_us'] = us
        res[f'kernel_{name}_GB_per_s'] = h * w * (12 + out_b) / us / 1e3

    assert np.array_equal(old_np_uint16(st), st.get_image('np_uint16'))
    old, new = [], []
    for _ in range(reps):
        for fn, acc in ((old_np_uint16, old), (lambda s: s.get_image('np_uint16'), new)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn(st)
            acc.append(1e3 * (time.perf_counter() - t0))
    res['get_image_np_uint16_ms'] = dict(old=float(np.median(old)), new=float(np.median(new)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[2048, 4096])
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('snapshot_bench: no CUDA device (timings exist only on the GPU)')
    wts = O.make_vgg_weights(1234)
    line = dict(card=card(), results=[bench_size(s, args.reps, wts) for s in args.sizes])
    print(json.dumps(line), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'snapshot_bench.json').write_text(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
