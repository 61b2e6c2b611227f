"""`style_transfer` console entry point for the H100-native build.

Same flags as the reference CLI (/root/reference/style_transfer/cli.py:155-203): positional content + styles,
`-o/--output`, `-sw/--style-weights`, `-d/--devices`, `-r/--random-seed`, `-p/--pooling`, `--save-every`, and one
option per keyword of `StyleTransfer.stylize` whose default and type are read from the method's signature (as
CLI:150-153 does).  Image I/O follows the reference too: inputs with an embedded ICC profile are converted to sRGB,
`--proof PROFILE` soft-proofs the content and style images through a CMYK profile, and a `.tif`/`.tiff` output is
written with 16 bits per channel and an sRGB profile (image_io.py).

`--web` serves the live monitor (web.py) at http://HOST:PORT/ (`--host`, default 0.0.0.0; `--port`, default 8080, 0 for
any free port; `--browser [NAME]` opens it).  Rank 0 feeds it every iteration; its image is a device snapshot taken when
a browser has fetched the previous one and at the end of every scale.  Under torchrun only rank 0 serves, and on a scale
tiled across the ranks its image refreshes only where every rank gathers anyway: at the saves and the scale ends.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from dataclasses import asdict
from pathlib import Path

import torch

from .image_io import TIFF_SUFFIXES, AsyncImageWriter, load_image, srgb_profile, write_tiff16
from .style_transfer import StyleTransfer

_SHORT = {'content_weight': 'cw', 'tv_weight': 'tw', 'optimizer': None, 'min_scale': 'ms', 'end_scale': 's',
          'iterations': 'i', 'initial_iterations': 'ii', 'step_size': 'ss', 'avg_decay': 'ad', 'init': None,
          'style_scale_fac': 'ssf', 'style_size': 'sz'}
_CHOICES = {'optimizer': ['adam', 'lbfgs'], 'init': ['content', 'gray', 'uniform', 'normal', 'style_stats']}


def build_parser():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('content', type=str, help='the content image')
    ap.add_argument('styles', type=str, nargs='+', metavar='style', help='the style images')
    ap.add_argument('--output', '-o', type=str, default='out.png', help='the output image')
    ap.add_argument('--style-weights', '-sw', type=float, nargs='+', default=None, metavar='STYLE_WEIGHT',
                    help='relative weights of the style images')
    ap.add_argument('--devices', '-d', type=str, default=[], nargs='+', help='the CUDA device name(s)')
    ap.add_argument('--random-seed', '-r', type=int, default=0, help='the random seed')
    ap.add_argument('--pooling', '-p', type=str, default='max', choices=['max', 'average', 'l2'],
                    help="the model's pooling mode")
    ap.add_argument('--save-every', type=int, default=0, help='save the image every SAVE_EVERY iterations')
    ap.add_argument('--web', default=False, action='store_true', help='enable the live web monitor')
    ap.add_argument('--host', type=str, default='0.0.0.0', help='the host the web monitor binds to')
    ap.add_argument('--port', type=int, default=8080, help='the port the web monitor binds to (0: any free port)')
    ap.add_argument('--browser', type=str, default='', nargs='?',
                    help='open a web browser (name one if not the system default)')
    ap.add_argument('--proof', type=str, default=None, metavar='PROFILE',
                    help='soft-proof the content and style images through this CMYK ICC profile')
    defaults = StyleTransfer.stylize.__kwdefaults__
    types = StyleTransfer.stylize.__annotations__
    for name, short in _SHORT.items():
        flags = ['--' + name.replace('_', '-')] + ([f'-{short}'] if short else [])
        kind = types[name]
        kind = {'float': float, 'int': int, 'str': str}.get(kind, kind) if isinstance(kind, str) else kind
        if name == 'end_scale':
            kind = str  # accepts "N+" like the reference (CLI:84-87, 233-236)
        ap.add_argument(*flags, type=kind, default=defaults[name], choices=_CHOICES.get(name), dest=name)
    return ap


def main(argv=None):
    args = build_parser().parse_args(argv)
    out_path = Path(args.output)
    tiff = out_path.suffix.lower() in TIFF_SUFFIXES   # 16 bits per channel, sRGB-tagged (reference CLI:63-81)
    content = load_image(args.content, args.proof)
    styles = [load_image(p, args.proof) for p in args.styles]

    # one process per GPU under torchrun: the ranks tile the large scales between them (distributed.py); rank 0 talks
    # and writes, every rank takes part in the collective gathers behind get_image()
    world, rank, local = (int(os.environ.get(k, d)) for k, d in (('WORLD_SIZE', 1), ('RANK', 0), ('LOCAL_RANK', 0)))
    devices = [torch.device(d) for d in args.devices]
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(local)
        devices = [torch.device('cuda', local)]
        if not dist.is_initialized():
            dist.init_process_group('nccl', device_id=devices[0])
    if not devices:
        if not torch.cuda.is_available():
            sys.exit('no CUDA device: this build has no CPU path')
        devices = [torch.device('cuda:0')]
    if len(set(d.type for d in devices)) != 1 or devices[0].type != 'cuda':
        sys.exit('devices must all be CUDA devices')
    # two devices in one process: StyleTransfer runs one rank per device and tiles the large scales across them
    for i, device in enumerate(devices):
        props = torch.cuda.get_device_properties(device)
        print(f'GPU {i} type: {props.name} (compute {props.major}.{props.minor})')
        print(f'GPU {i} RAM:', round(props.total_memory / 1024 / 1024), 'MB')

    end_scale = str(args.end_scale)
    if end_scale.endswith('+'):  # "N+": a safe scale for a non-square image given that N x N fits (CLI:84-87)
        dim = int(end_scale.rstrip('+'))
        w, h = content.size
        args.end_scale = int(pow(w / h if w > h else h / w, 1 / 2) * dim)
    else:
        args.end_scale = int(end_scale)

    web = None
    if args.web and rank == 0:   # only rank 0 serves: the other ranks cannot see the browser's requests
        from .web import WebInterface
        web = WebInterface(args.host, args.port)
    try:
        _run(args, content, styles, devices, rank, out_path, tiff, web)
    finally:
        if web is not None:
            web.close()


def _run(args, content, styles, devices, rank, out_path, tiff, web):
    for device in devices:
        torch.tensor(0).to(device)
    torch.manual_seed(args.random_seed)
    st = StyleTransfer(devices=[str(d) for d in devices], pooling=args.pooling)
    trace = []
    writer = AsyncImageWriter()  # periodic saves are encoded off the loop's critical path (image_io.py)
    if web is not None:
        import webbrowser
        if args.browser:
            webbrowser.get(args.browser).open(web.url)
        elif args.browser is None:
            webbrowser.open(web.url)
    done_after_run = []

    def on_iterate(it):
        trace.append(asdict(it))
        if rank == 0:
            print(f'Size: {it.w}x{it.h}, iteration: {it.i}, loss: {it.loss:g}')
        last_of_scale = it.i == it.i_max
        end = max(it.w, it.h) == args.end_scale
        # a scale tiled across processes: a gather takes every rank, so the monitor's image comes from the saves' gathers
        tiled_apart = web is not None and st._band is not None and st._sync is None
        gathered = None
        if (args.save_every and it.i % args.save_every == 0) or (last_of_scale and not end):
            if rank == 0:
                if tiled_apart:
                    gathered = st.get_image_tensor()
                writer.submit_snapshot(st, out_path, gathered)
            else:
                st.get_image_tensor()   # the gather of a tiled scale is collective
        if web is not None:
            web.put_iterate(it, st, gathered=gathered)
            if last_of_scale and end:
                if tiled_apart:
                    done_after_run.append(True)   # the final image is whole once stylize() has stitched the bands
                else:
                    web.put_done()

    kwargs = {k: getattr(args, k) for k in _SHORT}
    try:
        st.stylize(content, styles, style_weights=args.style_weights, callback=on_iterate, **kwargs)
        if done_after_run:
            web.put_done(st)
    except KeyboardInterrupt:
        pass
    writer.close()
    image = st.get_image('np_uint16' if tiff else 'pil')
    if rank != 0:
        return
    if image is not None:
        print(f'Writing image to {out_path}.')
        if tiff:
            write_tiff16(out_path, image, srgb_profile)
        else:
            image.save(out_path)
    with open('trace.json', 'w') as fp:
        json.dump(dict(args={k: (str(v) if isinstance(v, Path) else v) for k, v in vars(args).items()},
                       iterates=trace), fp, indent=4)


if __name__ == '__main__':
    main()
