#!/usr/bin/env python
"""Per-launch times of the 3x3 conv kernel (pixel_gemm_kernel) in the 2048^2 iteration that bench.py measures.

  python tools/conv_launch_times.py [--size 2048] [--iters 5] [--warmup 5] [--out DIR] [--root TREE]

Sets the iteration up as bench.py does for one GPU (same seeds, weights, style statistics and set_targets), warms
up, then records --iters iterations under torch.profiler with CUDA activities (trace written to DIR).  Prints the
GPU's name, power limit and max SM clock, then one row per launch of an iteration, mapped to its layer by launch
order: mode (0 fwd + bias/ReLU, 1 dgrad + mask/content, 2 dgrad before a pool), BN, tiles, tiles per CTA,
algorithmic FLOP (incl. the tap-gradient GEMM of the C2 operand), modelled HBM bytes (each operand read once: A, the
mask unless the staged tap operand serves as it, A2, the content target, out, pooled out), the median time over
the recorded iterations and the rates these give.  --root imports the package from another checkout (to time two
versions with the same script).
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent

KCIN = [3, 64, 64, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512]
KCOUT = [64, 64, 128, 128, 256, 256, 256, 256, 512, 512, 512, 512, 512]
POOL_AFTER = [False, True, False, True, False, False, False, True, False, False, False, True, False]
STYLE_CONV = {0: 64, 2: 128, 4: 256, 8: 512, 12: 512}   # conv index -> channels of its style tap
CONTENT_CONV = 9
NAMES = ['conv1_1', 'conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_2', 'conv3_3', 'conv3_4', 'conv4_1', 'conv4_2',
         'conv4_3', 'conv4_4', 'conv5_1']
TILE_H, TILE_W = 16, 8


def launches(size):
    """The pixel_gemm launches of one iteration in issue order (api.cu: forward convs 1..12, the relu5_1 tap, then
    the dgrad of convs 12..1), as dicts of the launch arguments."""
    h = []
    s = size
    for i in range(13):
        h.append(s)
        if POOL_AFTER[i]:
            s //= 2
    out = []
    for i in range(1, 13):
        out.append(dict(layer=f'{NAMES[i]} fwd', mode=0, H=h[i], Cin=KCIN[i], Cout=KCOUT[i], C2=0,
                        pool=POOL_AFTER[i] and i < 12, ctarget=False, a2_is_mask=False))
    out.append(dict(layer='relu5_1 tap', mode=1, H=h[12], Cin=0, Cout=512, C2=512, pool=False, ctarget=False,
                    a2_is_mask=True))
    for i in range(12, 0, -1):
        if POOL_AFTER[i - 1]:
            out.append(dict(layer=f'{NAMES[i]} dgrad', mode=2, H=h[i], Cin=KCOUT[i], Cout=KCIN[i], C2=0, pool=False,
                            ctarget=False, a2_is_mask=False))
        else:
            c2 = STYLE_CONV.get(i - 1, 0)
            out.append(dict(layer=f'{NAMES[i]} dgrad', mode=1, H=h[i], Cin=KCOUT[i], Cout=KCIN[i], C2=c2, pool=False,
                            ctarget=i - 1 == CONTENT_CONV, a2_is_mask=c2 > 0))
    return out


def model(L, sms):
    bn = 256 if L['Cout'] >= 256 else L['Cout']
    mt = 1 if bn == 256 else 2
    H = W = L['H']
    tiles = -(-H // TILE_H) * -(-W // (TILE_W * mt)) * (L['Cout'] // bn)
    px = H * W
    flop = 2.0 * px * L['Cout'] * (9 * L['Cin'] + L['C2'])
    # the staged tap operand serves as the mask on the 64- and 128-channel taps (C2 = Cout = BN <= 128, untiled)
    mask_from_a2 = L['mode'] == 1 and L['a2_is_mask'] and L['C2'] == L['Cout'] == bn <= 128
    b = dict(A=2 * px * L['Cin'],
             mask=2 * px * L['Cout'] if L['mode'] == 1 and not mask_from_a2 else 0,
             A2=2 * px * L['C2'],
             ctarget=2 * px * L['Cout'] if L['ctarget'] else 0,
             out=2 * px * L['Cout'],
             pool=2 * px * L['Cout'] // 4 if L['pool'] else 0)
    return dict(BN=bn, tiles=tiles, tiles_per_cta=tiles / min(tiles, sms), flop=flop, bytes=b,
                mask_src='A2' if mask_from_a2 else ('HBM' if L['mode'] == 1 else '-'))


def gpu_info():
    r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else 'nvidia-smi unavailable'


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--size', type=int, default=2048)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--out', default='conv_launch_times')
    ap.add_argument('--root', default=str(ROOT), help='checkout whose package is timed')
    args = ap.parse_args()
    sys.path.insert(0, str(Path(args.root).resolve()))
    import torch
    import style_transfer_b200 as stb
    from oracle import st_oracle as O
    from torch.profiler import ProfilerActivity, profile

    assert torch.cuda.is_available(), 'needs a GPU'
    out_dir = Path(args.out)
    out_dir.mkdir(parents=True, exist_ok=True)
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    size = args.size
    # ---- the setup of bench.py (one GPU)
    wts = O.make_vgg_weights(1234)
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    st = stb.StyleTransfer(devices=[str(dev)], pooling='max', vgg_weights=wts)
    m = st.model
    cimg = O.to_tensor(content).to(dev)
    simg = O.to_tensor(style).to(dev)
    m.ensure_workspace([(size, size), (size, size)])
    means, srms = st._style_stats(simg, size, size)
    ct = m.content_features(cimg)
    m.set_targets(size, size, ct, 0.015, means, srms, st.style_weights, 2.0)
    st.image = cimg.clone()
    st.average = stb.style_transfer.EMA(st.image, 0.99)
    ea, eas = torch.zeros_like(st.image), torch.zeros_like(st.image)
    step = 0

    def one_iteration():
        nonlocal step
        step += 1
        st._iterate(ea, eas, step, 0.02, 0.99, True)

    side = torch.cuda.Stream(device=dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    torch.cuda.set_stream(side)
    for _ in range(max(args.warmup, 3)):
        one_iteration()
    torch.cuda.synchronize()

    L = launches(size)
    per_iter = len(L)

    def record(tag):
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                one_iteration()
            torch.cuda.synchronize()
        trace = out_dir / f'trace_{tag}.json'
        prof.export_chrome_trace(str(trace))
        ev = [e for e in json.loads(trace.read_text())['traceEvents']
              if e.get('cat') == 'kernel' and 'pixel_gemm_kernel' in e.get('name', '')]
        return sorted(ev, key=lambda e: e['ts'])

    ev = record('graph')
    how = 'CUDA graph replay'
    if len(ev) != per_iter * args.iters:
        # graph-launched kernels not reported: time the same launches issued one by one (library profiling mode)
        from style_transfer_b200 import _lib
        _lib.check(m.lib.stb_profile_enable(m.ctx, 1))
        ev = record('eager')
        _lib.check(m.lib.stb_profile_enable(m.ctx, 0))
        how = 'launches issued one by one (library profiling mode; graph kernels were not reported)'
    assert len(ev) == per_iter * args.iters, f'{len(ev)} pixel_gemm launches recorded, expected {per_iter} x {args.iters}'

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    print(f'GPU: {gpu_info()}  (name, power limit, max SM clock); {sms} SMs; root {Path(args.root).resolve()}')
    print(f'{size}x{size}, {args.iters} iterations recorded ({how}); median per launch')
    hdr = (f'{"#":>2} {"layer":<14} {"mode":>4} {"BN":>3} {"tiles":>6} {"t/CTA":>6} {"mask":>4} {"GFLOP":>8} '
           f'{"MB A":>7} {"mask":>6} {"A2":>6} {"ctgt":>6} {"out":>6} {"pool":>6} {"us":>8} {"TFLOP/s":>8} '
           f'{"GB/s":>7}')
    print(hdr)
    rows = []
    tot = {0: 0.0, 1: 0.0, 2: 0.0}
    for k, l in enumerate(L):
        d = sorted(ev[it * per_iter + k]['dur'] for it in range(args.iters))
        us = d[len(d) // 2]
        mo = model(l, sms)
        nbytes = sum(mo['bytes'].values())
        mb = {n: v / 1e6 for n, v in mo['bytes'].items()}
        tot[l['mode']] += us
        rows.append(dict(layer=l['layer'], mode=l['mode'], us=us, us_all=d, **mo))
        print(f'{k:>2} {l["layer"]:<14} {l["mode"]:>4} {mo["BN"]:>3} {mo["tiles"]:>6} {mo["tiles_per_cta"]:>6.1f} '
              f'{mo["mask_src"]:>4} {mo["flop"] / 1e9:>8.1f} {mb["A"]:>7.0f} {mb["mask"]:>6.0f} {mb["A2"]:>6.0f} '
              f'{mb["ctarget"]:>6.0f} {mb["out"]:>6.0f} {mb["pool"]:>6.0f} {us:>8.1f} '
              f'{mo["flop"] / us / 1e6:>8.1f} {nbytes / us / 1e3:>7.0f}')
    print(f'sum per iteration: mode 0 {tot[0] / 1e3:.3f} ms, mode 1 {tot[1] / 1e3:.3f} ms, mode 2 {tot[2] / 1e3:.3f} ms, '
          f'all {sum(tot.values()) / 1e3:.3f} ms')
    (out_dir / 'launches.json').write_text(json.dumps(dict(gpu=gpu_info(), how=how, rows=rows), indent=1))


if __name__ == '__main__':
    main()
