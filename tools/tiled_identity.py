"""Writes what the tiled iterations compute, so that two builds can be compared byte for byte.

Runs stylize() with 2 and 3 thread-ranks on ONE GPU (distributed.ThreadGroup, the peer-memory exchange), for Adam and
L-BFGS, in apron and halo tile mode, at a width that is a multiple of 4 (the float4 row kernels) and one that is not
(the scalar ones), 20 iterations each.  Per job and rank it writes the final image, the EMA and the loss trace as .npy
files under OUT/<job>/.  Every job is seeded, so the same build writes the same bytes; `diff -r` of the OUT directories
of two builds then shows whether a change moved any bit of the tiled paths.
  python tools/tiled_identity.py --out DIR [--its 20]"""
import argparse
import contextlib
import gc
import io
import json
import os
import sys
import threading
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200 import distributed as D  # noqa: E402
from oracle import st_oracle as O  # noqa: E402  (fixture generator only)

# (W, H): 320 rows split into bands of at least distributed.MIN_BAND_ROWS rows for 2 and for 3 ranks
SIZES = [(184, 320), (181, 320)]


def run(world, W, H, optimizer, its, wts):
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
    kw = dict(min_scale=max(W, H), end_scale=max(W, H), initial_iterations=its, optimizer=optimizer)
    shared = D.ThreadGroup.Shared(world)
    results, errors = [None] * world, []

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts,
                                   distributed=D.ThreadGroup(shared, rank))
            trace = []
            st.stylize(content, [style], callback=lambda it: trace.append(it.loss), **kw)
            st._stream.synchronize()
            results[rank] = dict(image=st.image.detach().cpu().numpy(), ema=st.average.get().cpu().numpy(),
                                 loss=np.array(trace, dtype=np.float64),
                                 mode=[st._comm_mode, 'halo' if st._halo_now else 'apron'])
        except BaseException as e:  # noqa: BLE001 -- report and release the other ranks
            errors.append((rank, repr(e)))
            shared.bar.abort()

    # gc is off: a finalizer that frees device memory synchronises the device, and run on one rank's thread while a
    # peer's kernel waits for that rank it would stall both.  stdout is process-wide, so stylize's progress output is
    # dropped around all ranks at once.
    gc.collect()
    gc.disable()
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
            for t in threads:
                t.start()
            for t in threads:
                t.join()
    finally:
        gc.enable()
    if errors:
        raise RuntimeError(errors)
    return results


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--its', type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA GPU')
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '60')
    wts = O.make_vgg_weights(1234)
    out = Path(a.out)
    summary = {}
    for optimizer in ('adam', 'lbfgs'):
        for tile in ('apron', 'halo'):
            os.environ['STB_TILE'] = tile   # read when a StyleTransfer is created
            for W, H in SIZES:
                for world in (2, 3):
                    job = f'{optimizer}_{tile}_{W}x{H}_world{world}'
                    res = run(world, W, H, optimizer, a.its, wts)
                    for r in res:
                        if r['mode'] != ['peer', tile] or len(r['loss']) != a.its:
                            raise RuntimeError(f'{job}: not a tiled run ({r["mode"]}, {len(r["loss"])} iterations)')
                    (out / job).mkdir(parents=True, exist_ok=True)
                    for rank, r in enumerate(res):
                        for key in ('image', 'ema', 'loss'):
                            np.save(out / job / f'rank{rank}_{key}.npy', r[key])
                    summary[job] = [float(r['loss'][-1]) for r in res]
                    print(job, 'final loss per rank', summary[job], flush=True)
    (out / 'summary.json').write_text(json.dumps(summary, indent=1) + '\n')


if __name__ == '__main__':
    main()
