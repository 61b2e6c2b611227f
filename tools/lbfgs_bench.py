"""optimizer='lbfgs': native iterations (stb_iterate_lbfgs, one CUDA graph, no host sync) against the torch-driven loop
(torch.optim.LBFGS on the host over the native closure st.loss_and_grad(), EMA after each step), at 512^2 and 2048^2,
with the Adam iteration rate of the same run as context.  Both loops are timed with CUDA events, alternately, 3 times,
each time from the content image with a fresh optimizer given 10 pairs before the timed window (see bench_size).
The L-BFGS kernels alone are timed around stb_test_lbfgs_step at the 2048^2 vector length with a full history and
reported as achieved bandwidth against the traffic model of csrc/lbfgs.cu.  Prints one JSON line.
Usage: python tools/lbfgs_bench.py [--sizes 512,2048] [--iters 20] [--natural-its 30]"""
import argparse
import ctypes
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
import style_transfer_b200 as stb  # noqa: E402
from style_transfer_b200 import _lib  # noqa: E402
from oracle import st_oracle as O  # noqa: E402  (fixture generator only)

DEV = torch.device('cuda:0')
DECAY = 0.99
HIST = 10


def card():
    info = dict(name=torch.cuda.get_device_name(DEV))
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info['power_limit'], info['max_sm_clock'] = [v.strip() for v in q.split(',')]
    except Exception as e:   # the number is still reported, without the limit
        info['power_limit'] = f'unavailable ({e})'
    return info


def setup(st, size):
    m = st.model
    cimg = O.to_tensor(O.synth_image(1, 16, size, size)).to(DEV)
    simg = O.to_tensor(O.synth_image(2, 32, size, size)).to(DEV)
    m.ensure_workspace([(size, size)])
    ct = m.content_features(cimg)
    means, srms = m.style_stats(simg)
    m.set_targets(size, size, ct, 0.015, means, srms, st.style_weights, 2.0)
    return cimg.contiguous()


def timed(stream, fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(iters):
        fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / iters


def lbfgs_header(state):
    """n_iter, count, head, skip, took_step: the leading int32 fields of the state block (LbHeader, csrc/lbfgs.cu)."""
    h = state[:20].view(torch.int32).tolist()
    return dict(n_iter=h[0], pairs=h[1], skip=h[3], took_step=h[4])


def bench_size(wts, size, iters, natural_its):
    """Both L-BFGS loops are timed only over iterations that do the full work (10 pairs held, all 21 two-loop rounds).
    On its own trajectory this problem may store no pair at all: at 2048^2 every y.s stays <= 1e-10, in torch as on the
    device, so a plain run times the 0-pair step.  `natural_pairs` reports what each loop holds after `natural_its`
    iterations from the content image.  For the timing, every repetition restarts from the content image with a fresh
    optimizer, gives it 10 pairs with 11 untimed steps on a diagonal quadratic (so every pair is accepted), and then
    times `iters` real iterations.  Later pairs may be accepted or rejected; either way 10 stay held.  Afterwards it
    checks that 10 pairs are still held, that n_iter advanced once per iteration (no opt_cond exit) and that the
    iterate and the loss are finite.  Adam runs on a context of its own, whose device step counter is never re-seeded
    inside a timed window."""
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    sa = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts)
    m, ma = st.model, sa.model
    img = setup(st, size)
    setup(sa, size)
    stream = torch.cuda.Stream(device=DEV)   # graphs need a non-legacy stream
    stream.wait_stream(torch.cuda.current_stream())
    res = {'native_ms': [], 'torch_driven_ms': [], 'adam_ms': [], 'native_check': [], 'torch_check': []}
    with torch.cuda.stream(stream):
        n = ctypes.c_size_t()
        _lib.check(m.lib.stb_lbfgs_state_bytes(size, size, ctypes.byref(n)))
        state = torch.empty(n.value, dtype=torch.uint8, device=DEV)
        x_n, ema_n = img.clone(), img * (1 - DECAY)
        step_n = [0]

        def native():
            step_n[0] += 1
            _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(x_n), _lib.ptr(ema_n), _lib.ptr(state), state.numel(),
                                               step_n[0], DECAY, None, _lib.cur_stream()))

        # the torch-driven loop: what optimizer='lbfgs' ran before the step moved onto the device
        x_t, ema_t = img.clone(), img * (1 - DECAY)
        param = torch.nn.Parameter(x_t, requires_grad=True)
        box = {}

        def torch_driven():
            st.image = x_t

            def closure():
                terms, grad = st.loss_and_grad()
                box['loss'] = float(terms[0])
                param.grad = grad
                return terms[0].to(DEV)

            with torch.enable_grad():
                box['opt'].step(closure)
            ema_t.mul_(DECAY).add_(x_t, alpha=1 - DECAY)

        def torch_pairs():
            return len(box['opt'].state[param].get('old_dirs', []))

        x_a, m1, m2, ema_a = img.clone(), torch.zeros_like(img), torch.zeros_like(img), img * (1 - DECAY)
        step_a = [0]

        def adam():
            step_a[0] += 1
            _lib.check(ma.lib.stb_iterate(ma.ctx, _lib.ptr(x_a), _lib.ptr(m1), _lib.ptr(m2), _lib.ptr(ema_a),
                                          step_a[0], 0.02, 0.9, 0.99, 1e-8, DECAY, None, _lib.cur_stream()))

        gen = torch.Generator(device=DEV).manual_seed(0)
        qa = torch.rand(img.numel(), device=DEV, generator=gen) * 9.9 + 0.1   # diagonal quadratic of the prefill
        qb = torch.randn(img.numel(), device=DEV, generator=gen) * 0.1
        tlib = _lib.load_test()

        def native_prefill():
            for _ in range(HIST + 1):
                g = (qa * x_n.flatten() + qb).contiguous()
                _lib.check(tlib.stb_test_lbfgs_step(_lib.ptr(state), state.numel(), size, size, _lib.ptr(x_n),
                                                    _lib.ptr(g), _lib.ptr(ema_n), DECAY, None, None,
                                                    _lib.cur_stream()), test_lib=True)

        def torch_prefill():
            def closure():
                param.grad = (qa * x_t.flatten() + qb).view_as(x_t)
                return torch.zeros((), device=DEV)

            for _ in range(HIST + 1):
                box['opt'].step(closure)

        def restart():
            x_n.copy_(img)
            ema_n.copy_(img * (1 - DECAY))
            _lib.check(m.lib.stb_lbfgs_reset(_lib.ptr(state), size, size, _lib.cur_stream()))
            x_t.copy_(img)
            ema_t.copy_(img * (1 - DECAY))
            box['opt'] = torch.optim.LBFGS([param], max_iter=1, history_size=HIST)

        restart()   # the natural trajectory, untimed
        for _ in range(natural_its):
            native()
            torch_driven()
        natural = dict(iterations=natural_its, native=lbfgs_header(state)['pairs'], torch_driven=torch_pairs())
        timed(stream, adam, 5)
        for _ in range(3):
            restart()
            native_prefill()
            h0 = lbfgs_header(state)
            res['native_ms'].append(timed(stream, native, iters))
            h1 = lbfgs_header(state)
            loss = float(st._wait_loss(step_n[0])[0])
            res['native_check'].append(dict(pairs_before=h0['pairs'], **h1,
                                            steps_in_window=h1['n_iter'] - h0['n_iter'], last_loss=loss,
                                            finite=bool(torch.isfinite(x_n).all()) and loss == loss and abs(loss) < 1e30))
            torch_prefill()
            p0, it0 = torch_pairs(), box['opt'].state[param]['n_iter']
            res['torch_driven_ms'].append(timed(stream, torch_driven, iters))
            loss = box['loss']
            res['torch_check'].append(dict(pairs_before=p0, pairs=torch_pairs(),
                                           steps_in_window=box['opt'].state[param]['n_iter'] - it0, last_loss=loss,
                                           finite=bool(torch.isfinite(x_t).all()) and loss == loss and abs(loss) < 1e30))
            res['adam_ms'].append(timed(stream, adam, iters))
    stream.synchronize()
    full = all(c['pairs_before'] == HIST and c['pairs'] == HIST and c['steps_in_window'] == iters and c['finite']
               for c in res['native_check'] + res['torch_check'])
    out = {k: ([round(v, 4) for v in vs] if k.endswith('_ms') else vs) for k, vs in res.items()}
    nat, td = statistics.median(res['native_ms']), statistics.median(res['torch_driven_ms'])
    out.update(natural_pairs=natural, full_history_and_finite=full, native_ms_median=round(nat, 4),
               torch_driven_ms_median=round(td, 4), speedup=round(td / nat, 3), adam_it_s=round(1000 / statistics.median(res['adam_ms']), 2),
               graph_status=m.graph_status()[0], lbfgs_state_bytes=n.value)
    del state, param, box, st, sa
    torch.cuda.empty_cache()
    return out


def bench_kernels(size, iters):
    """The step alone at n = 3 size^2 with 10 pairs held.  Traffic model of the launch sequence (floats moved per
    element, m pairs): pass 0 reads g, g_prev, d and writes y, s (5); the 2m + 1 rounds of the two-loop read and write d
    and read one or two history vectors (3 + 4(m - 1) + 3 + 4(m - 1) + 4); the final pass reads x, d, ema, g and writes
    x, ema, g_prev (7): (8 m + 14) n floats."""
    tlib = _lib.load_test()
    lib = _lib.load()
    nb = ctypes.c_size_t()
    _lib.check(lib.stb_lbfgs_state_bytes(size, size, ctypes.byref(nb)))
    n = 3 * size * size
    state = torch.empty(nb.value, dtype=torch.uint8, device=DEV)
    _lib.check(lib.stb_lbfgs_reset(_lib.ptr(state), size, size, _lib.cur_stream()))
    gen = torch.Generator(device=DEV).manual_seed(0)
    a = torch.rand(n, device=DEV, generator=gen) * 9.9 + 0.1      # diagonal quadratic: every pair is accepted
    b = torch.randn(n, device=DEV, generator=gen) * 0.1
    x = torch.rand(n, device=DEV, generator=gen)
    ema = x * (1 - DECAY)
    pairs, t = ctypes.c_int(), ctypes.c_float()

    def step(grad, info=False):
        _lib.check(tlib.stb_test_lbfgs_step(_lib.ptr(state), nb.value, size, size, _lib.ptr(x), _lib.ptr(grad),
                                            _lib.ptr(ema), DECAY, ctypes.byref(pairs) if info else None,
                                            ctypes.byref(t) if info else None, _lib.cur_stream()), test_lib=True)

    for _ in range(HIST + 2):
        step(a * x + b, info=True)
    assert pairs.value == HIST, pairs.value
    # from here the gradient held by the state is reused: y = 0 is rejected, the history stays full, every round runs
    for _ in range(5):
        step(None)
    ms = statistics.median(timed(torch.cuda.current_stream(), lambda: step(None), iters) for _ in range(3))
    step(None, info=True)
    assert pairs.value == HIST
    model_bytes = (8 * HIST + 14) * n * 4
    return dict(n=n, pairs=pairs.value, ms=round(ms, 4), model_bytes=model_bytes,
                achieved_gb_s=round(model_bytes / ms / 1e6, 1), launches=2 * HIST + 4)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', default='512,2048')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--natural-its', type=int, default=30, help='untimed iterations of the pair-count diagnostic')
    args = ap.parse_args()
    out = dict(card=card())
    wts = O.make_vgg_weights(1234)
    for size in (int(s) for s in args.sizes.split(',')):
        out[f'iter_{size}'] = bench_size(wts, size, args.iters, args.natural_its)
    out['lbfgs_step_2048'] = bench_kernels(2048, 50)
    out['card_after'] = card()
    print(json.dumps(out))
    # a timing of loops that did not both hold a full history with finite iterates does not measure the same work
    if not all(out[k]['full_history_and_finite'] for k in out if k.startswith('iter_')):
        sys.exit('some timed window was not full-history / finite: see native_check / torch_check')


if __name__ == '__main__':
    main()
