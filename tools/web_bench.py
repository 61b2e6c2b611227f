"""Cost of the live web monitor (--web) to the optimisation loop, with a browser-like client connected.

  python tools/web_bench.py [--sizes 2048 4096] [--warmup 10] [--steps 60] [--rounds 3] [--out DIR]

Per size (one square scale, synthetic images and weights), `rounds` times alternately: a run without the monitor, then
a run whose callback calls put_iterate(it, st) every iteration while a loopback client, in a process of its own as a
browser is, holds the websocket and fetches /image back to back.  Each run is `warmup` + `steps` iterations; it/s is
taken over the `steps` timed ones from the callbacks' clock.  Reported: it/s off and on (median over the rounds, and
every round), their ratio, snapshots per second, the median JPEG encode time and the median /image latency seen by the
client.  The card's name and power limit are read in the same run.  Prints one JSON line.

--breakdown splits the cost of the monitor at each size into parts, alternating these runs `rounds` times:
  off         no monitor
  full        the monitor with a client fetching /image back to back
  no_encode   the same, with the JPEG encode replaced by a constant (so a snapshot is taken about every iteration)
  ws_only     the monitor with a client that holds the websocket and fetches nothing (one snapshot, at the end)
  snap_every  no client: a snapshot (kernel, side-stream copy, event) forced at every iteration, nothing encoded
  switch_5ms  full, with the switch interval put back to Python's default 5 ms (the monitor lowers it to 0.5 ms)
and reports, per run kind, it/s and the host time per timed iteration spent inside put_iterate and polling the loss
ring (_wait_loss).
"""
import argparse
import asyncio
import contextlib
import io
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

import style_transfer_b200 as stb  # noqa: E402
from oracle import st_oracle as O  # noqa: E402


def card():
    try:
        return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f'nvidia-smi unavailable ({e})'


class Client:
    """A browser stand-in in a process of its own (as a browser is): holds the websocket and fetches /image back to back
    until the run's WIDone, then reports the latency of every image it received."""

    def __init__(self, url, fetch=True):
        self.proc = subprocess.Popen([sys.executable, __file__, '--client', url] + ([] if fetch else ['--no-fetch']),
                                     stdout=subprocess.PIPE, text=True)
        assert self.proc.stdout.readline().strip() == 'connected'

    def join(self):
        out, _ = self.proc.communicate(timeout=120)
        return json.loads(out)


def client_main(url, fetch_images):
    import aiohttp
    latency = []

    async def fetch(s, done):
        while fetch_images and not done.is_set():
            t0 = time.perf_counter()
            async with s.get(url + 'image') as r:
                await r.read()
                if r.status == 200:
                    latency.append(time.perf_counter() - t0)
                else:
                    await asyncio.sleep(0.002)

    async def main():
        async with aiohttp.ClientSession() as s:
            async with s.ws_connect(url + 'websocket') as ws:
                print('connected', flush=True)
                done = asyncio.Event()
                fetcher = asyncio.ensure_future(fetch(s, done))
                async for msg in ws:
                    if json.loads(msg.data)['_type'] == 'WIDone':
                        break
                done.set()
                await fetcher

    asyncio.run(main())
    print(json.dumps(latency), flush=True)


def run(st, content, style, size, warmup, steps, web, force_snapshots=False, host=None):
    """it/s and snapshots/s over the timed iterations.  `host`: a dict that receives the host seconds per timed
    iteration spent inside put_iterate ('put_iterate_ms') and inside _wait_loss ('wait_loss_ms')."""
    stamps, put_s, wait_s = [], [], []
    wait_loss = st._wait_loss

    def timed_wait(step):
        t0 = time.perf_counter()
        try:
            return wait_loss(step)
        finally:
            wait_s.append(time.perf_counter() - t0)

    def cb(it):
        stamps.append(time.perf_counter())
        if web is not None and len(stamps) == warmup:
            snaps0[0] = web.snapshots
        if web is not None:
            if force_snapshots:
                web._wanted = True
            t0 = time.perf_counter()
            web.put_iterate(it, st)
            put_s.append(time.perf_counter() - t0)
            if it.i == it.i_max:
                web.put_done()

    snaps0 = [0]
    if host is not None:
        st._wait_loss = timed_wait
    try:
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=warmup + steps,
                       callback=cb)
    finally:
        st.__dict__.pop('_wait_loss', None)
    span = stamps[-1] - stamps[warmup - 1]
    snaps = (web.snapshots - snaps0[0]) if web is not None else 0
    if host is not None:
        host['put_iterate_ms'] = 1e3 * sum(put_s[warmup:]) / steps if put_s else 0.0
        host['wait_loss_ms'] = 1e3 * sum(wait_s[warmup:]) / steps
    return steps / span, snaps / span


def _constant_jpeg(_pixels, _body=[]):
    if not _body:
        buf = io.BytesIO()
        from PIL import Image
        Image.new('RGB', (8, 8)).save(buf, format='jpeg')
        _body.append(buf.getvalue())
    return _body[0]


def breakdown_size(size, args, wts):
    from style_transfer_b200 import web as W
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    kinds = ['off', 'full', 'no_encode', 'ws_only', 'snap_every', 'switch_5ms']
    res = {k: dict(its_per_s=[], snapshots_per_s=[], put_iterate_ms=[], wait_loss_ms=[]) for k in kinds}
    encode = W.encode_jpeg
    interval = sys.getswitchinterval()
    for _ in range(args.rounds):
        for kind in kinds:
            host = {}
            web = client = None
            try:
                if kind != 'off':
                    with contextlib.redirect_stdout(io.StringIO()):
                        web = stb.WebInterface('127.0.0.1', 0)
                    if kind in ('full', 'no_encode', 'switch_5ms', 'ws_only'):
                        client = Client(web.url, fetch=kind != 'ws_only')
                if kind == 'no_encode':
                    W.encode_jpeg = _constant_jpeg
                if kind == 'switch_5ms':
                    sys.setswitchinterval(5e-3)
                ips, sps = run(st, content, style, size, args.warmup, args.steps, web,
                               force_snapshots=kind == 'snap_every', host=host)
            finally:
                W.encode_jpeg = encode
                if web is not None:
                    web.close()
                sys.setswitchinterval(interval)
                if client is not None:
                    client.join()
            r = res[kind]
            r['its_per_s'].append(ips)
            r['snapshots_per_s'].append(sps)
            r['put_iterate_ms'].append(host['put_iterate_ms'])
            r['wait_loss_ms'].append(host['wait_loss_ms'])
    out = dict(size=size)
    for kind, r in res.items():
        out[kind] = {k: float(np.median(v)) for k, v in r.items()}
        out[kind]['its_per_s_rounds'] = r['its_per_s']
        out[kind]['vs_off'] = out[kind]['its_per_s'] / float(np.median(res['off']['its_per_s']))
    return out


def bench_size(size, args, wts):
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    off, on, refresh, encode, latency = [], [], [], [], []
    for _ in range(args.rounds):
        off.append(run(st, content, style, size, args.warmup, args.steps, None)[0])
        with contextlib.redirect_stdout(io.StringIO()):
            web = stb.WebInterface('127.0.0.1', 0)
        try:
            client = Client(web.url)
            ips, rps = run(st, content, style, size, args.warmup, args.steps, web)
        finally:
            web.close()
        latency += client.join()
        on.append(ips)
        refresh.append(rps)
        encode += web.encode_times
    med = lambda v: float(np.median(v)) if v else None   # noqa: E731
    return dict(size=size, its_per_s_off=med(off), its_per_s_on=med(on), ratio=med(on) / med(off),
                rounds_off=off, rounds_on=on, refreshes_per_s=med(refresh),
                jpeg_encode_ms=1e3 * med(encode) if encode else None,
                image_latency_ms=1e3 * med(latency) if latency else None, images_fetched=len(latency))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[2048, 4096])
    ap.add_argument('--warmup', type=int, default=10)
    ap.add_argument('--steps', type=int, default=60)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    ap.add_argument('--breakdown', action='store_true', help='split the cost into parts (see the module docstring)')
    ap.add_argument('--client', default=None, help=argparse.SUPPRESS)
    ap.add_argument('--no-fetch', action='store_true', help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.client:
        return client_main(args.client, not args.no_fetch)
    if args.warmup < 1 or args.steps < 1:
        raise SystemExit('web_bench: --warmup and --steps must be at least 1 (it/s is timed from the last warm-up '
                         'iteration)')
    if not torch.cuda.is_available():
        raise SystemExit('web_bench: no CUDA device (timings exist only on the GPU)')
    wts = O.make_vgg_weights(1234)
    fn = breakdown_size if args.breakdown else bench_size
    line = dict(card=card(), results=[fn(s, args, wts) for s in args.sizes])
    print(json.dumps(line), flush=True)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / ('web_breakdown.json' if args.breakdown else 'web_bench.json')).write_text(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
