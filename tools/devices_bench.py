"""stylize() on one GPU against StyleTransfer(devices=['cuda:0', 'cuda:1']), single scale at 2048^2 and 4096^2.

  python tools/devices_bench.py [--sizes 2048 4096] [--its 50] [--warmup 5] [--out DIR]

Iteration rate = (its - warmup) / wall time from the callback of iteration `warmup` (after synchronising every device
of the run) to the return of stylize() (which ends in a synchronise of the ranks' streams; the final gather of the
bands is inside the window).  Per GPU: torch's peak allocation and the drop in free device memory from before the
StyleTransfer is built to iteration `warmup` (it also counts the library-owned workspace, mailboxes and the CUDA
context).  The two-device runs need two GPUs; with fewer they are reported as not measured.  GPU name, power limit
and SM clocks are read in the same call."""
import argparse
import contextlib
import io
import json
import subprocess
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import style_transfer_b200 as stb  # noqa: E402
from oracle import st_oracle as O  # noqa: E402  (synthetic images and weights only)

MIB = 1024 * 1024


def run(devices, size, its, warmup, wts):
    ids = sorted({torch.device(d).index for d in devices})
    for i in ids:
        torch.cuda.synchronize(i)
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(i)
    free0 = {i: torch.cuda.mem_get_info(i)[0] for i in ids}
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    st = stb.StyleTransfer(devices=devices, pooling='max', vgg_weights=wts)
    mark = {}

    def cb(it):
        if it.i == warmup:
            for i in ids:
                torch.cuda.synchronize(i)
                mark[i] = torch.cuda.mem_get_info(i)[0]
            mark['t0'] = time.perf_counter()

    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=its, callback=cb)
    dt = time.perf_counter() - mark['t0']
    out = dict(devices=devices, size=size, its_per_s=round((its - warmup) / dt, 2),
               ms_per_iteration=round(dt / (its - warmup) * 1e3, 3),
               tile_mode=('halo' if st._halo_now else 'apron') if st._peer is not None else None)
    for i in ids:
        out[f'cuda{i}_torch_peak_mib'] = round(torch.cuda.max_memory_allocated(i) / MIB)
        out[f'cuda{i}_device_used_mib'] = round((free0[i] - mark[i]) / MIB)
    del st
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[2048, 4096])
    ap.add_argument('--its', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('needs a CUDA GPU')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=index,name,power.limit,clocks.sm,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip().splitlines()
    wts = O.make_vgg_weights(1234)
    lines = [dict(gpus=gpu, device_count=torch.cuda.device_count(), its=a.its, warmup=a.warmup)]
    for size in a.sizes:
        lines.append(run(['cuda:0'], size, a.its, a.warmup, wts))
        if torch.cuda.device_count() >= 2:
            lines.append(run(['cuda:0', 'cuda:1'], size, a.its, a.warmup, wts))
        else:
            lines.append(dict(devices=['cuda:0', 'cuda:1'], size=size, its_per_s='not measured (one GPU)'))
    text = '\n'.join(json.dumps(x) for x in lines)
    print(text)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / 'devices_bench.jsonl').write_text(text + '\n')


if __name__ == '__main__':
    main()
