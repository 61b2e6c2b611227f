"""Banded L-BFGS (stb_iterate_lbfgs_banded) with N thread-ranks on ONE GPU against the untiled stb_iterate_lbfgs at the
same image size, and the device time of the cross-rank reduction kernels (lbfgs_xreduce_kernel, 22 per iteration).

The ranks share one GPU, so the banded figure is a one-GPU latency, not a multi-GPU scaling figure: it shows what the
exchanges and the 22 extra one-block kernels cost, with N ranks' kernels interleaved on the same SMs.
  python tools/lbfgs_tiled_bench.py [--size 1024] [--world 2] [--its 40] [--warmup 10] [--out DIR]
Iteration time = wall time between the loss callbacks of iterations warmup and its (each callback waits for the loss
that iteration publishes before its backward pass), over its - warmup.  Kernel times come from torch.profiler in a
second, shorter run (profiling slows the host)."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200 import distributed as D  # noqa: E402
from oracle import st_oracle as O  # noqa: E402  (fixture generator only)


def run(world, size, its, wts, profile=False):
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size // 2, size // 2)
    kw = dict(min_scale=size, end_scale=size, initial_iterations=its, optimizer='lbfgs')
    stamps = [[] for _ in range(max(world, 1))]
    errors = []

    def one(rank, group):
        torch.cuda.set_device(0)
        st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts, distributed=group)
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], callback=lambda it: stamps[rank].append(time.perf_counter()), **kw)
        return st

    if world <= 1:
        one(0, False)
    else:
        shared = D.ThreadGroup.Shared(world)

        def worker(rank):
            try:
                one(rank, D.ThreadGroup(shared, rank))
            except BaseException as e:  # noqa: BLE001
                errors.append(repr(e))
                shared.bar.abort()

        threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
    torch.cuda.synchronize()
    if errors:
        raise RuntimeError(errors)
    return stamps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--world', type=int, default=2)
    ap.add_argument('--its', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA GPU')
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '60')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    wts = O.make_vgg_weights(1234)
    res = dict(gpu=gpu, size=a.size, world=a.world, iterations=a.its, warmup=a.warmup)
    for name, world in (('untiled', 1), ('banded', a.world), ('untiled_again', 1), ('banded_again', a.world)):
        st = run(world, a.size, a.its, wts)
        per = [(s[a.its - 1] - s[a.warmup - 1]) / (a.its - a.warmup) * 1e3 for s in st]
        res[f'{name}_ms_per_iteration'] = max(per)
    prof_its = 12
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        run(a.world, a.size, prof_its, wts)
    xr = [e for e in prof.events() if 'lbfgs_xreduce_kernel' in e.name]
    step_kernels = [e for e in prof.events() if 'lbfgs_' in e.name]
    n_iter = prof_its * a.world
    res['xreduce_kernels_seen'] = len(xr)
    res['xreduce_kernels_expected'] = 22 * n_iter
    if xr:
        res['xreduce_ms_per_rank_iteration'] = sum(e.device_time_total for e in xr) / 1e3 / n_iter
        res['xreduce_us_mean'] = sum(e.device_time_total for e in xr) / len(xr)
        res['lbfgs_step_kernels_ms_per_rank_iteration'] = sum(e.device_time_total for e in step_kernels) / 1e3 / n_iter
    line = json.dumps(res)
    print(line)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / 'lbfgs_tiled_bench.json').write_text(line + '\n')


if __name__ == '__main__':
    main()
