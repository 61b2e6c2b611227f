"""Iterations/sec of the native Adam iteration for several layer tables at one size (default 2048^2, single scale).

  python tools/layers_bench.py [--size 2048] [--steps 40] [--rounds 5] [--out DIR]

Configurations: the default table (content [22], style [1, 6, 11, 20, 29]), A (content [11], style [1, 6, 11]) and
B (content [22], style [1, 6, 11, 20, 22, 29]).  Each has a context of its own, set up once; the timed windows
alternate between them (`rounds` windows of `steps` graphed iterations each, CUDA events on the iteration stream), so
that clock and neighbour drift spread over all of them.  The card's name and power limit are read in the same run.
Prints one JSON line: median / min / max it/s per configuration.
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200.style_transfer import EMA  # noqa: E402
from oracle import st_oracle as O  # noqa: E402

CONFIGS = {
    'default': ([22], [1, 6, 11, 20, 29], [256, 64, 16, 4, 1]),
    'A': ([11], [1, 6, 11], [256, 64, 16]),
    'B': ([22], [1, 6, 11, 20, 22, 29], [256, 64, 16, 4, 4, 1]),
}


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'nvidia-smi unavailable ({e})'


def setup(name, size, wts):
    content_layers, style_layers, raw = CONFIGS[name]
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    m = st.model
    m.set_layers(content_layers, style_layers)
    cimg = O.to_tensor(O.synth_image(1, 16, size, size)).cuda()
    simg = O.to_tensor(O.synth_image(2, 32, size, size)).cuda()
    lw = [w / sum(raw) for w in raw]
    with torch.cuda.stream(st._stream):
        m.ensure_workspace([(size, size)])
        cts = m.content_features_list(cimg)
        means, srms = m.style_stats(simg)
        m.set_targets_list(size, size, cts, [0.015 / len(content_layers)] * len(content_layers), means, srms, lw, 2.0)
        st.image = cimg.clone()
        st.average = EMA(st.image, 0.99)
        state = dict(st=st, ea=torch.zeros_like(cimg), eas=torch.zeros_like(cimg), step=0)
    return state


def run(state, n):
    st = state['st']
    with torch.cuda.stream(st._stream):
        for _ in range(n):
            state['step'] += 1
            st._iterate(state['ea'], state['eas'], state['step'], 0.02, 0.99, False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=2048)
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('layers_bench: no CUDA device (timings exist only on the GPU)')
    wts = O.make_vgg_weights(1234)
    states = {name: setup(name, args.size, wts) for name in CONFIGS}
    for s in states.values():   # eager runs, graph capture, one warm window
        run(s, 10)
        s['st']._stream.synchronize()
    rates = {name: [] for name in CONFIGS}
    for _ in range(args.rounds):
        for name, s in states.items():
            stream = s['st']._stream
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            run(s, args.steps)
            e1.record(stream)
            e1.synchronize()
            rates[name].append(1000.0 * args.steps / e0.elapsed_time(e1))
    line = dict(card=card(), size=args.size, steps=args.steps, rounds=args.rounds,
                kernels_per_iteration={n: s['st'].model.launch_count()[2][0] for n, s in states.items()},
                it_per_s={n: dict(median=float(np.median(r)), min=float(min(r)), max=float(max(r)))
                          for n, r in rates.items()})
    print(json.dumps(line), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / 'layers_bench.json').write_text(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
