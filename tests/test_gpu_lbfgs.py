"""-m gpu: optimizer='lbfgs' on the device (csrc/lbfgs.cu, stb_iterate_lbfgs).

The oracle of the optimizer step is torch.optim.LBFGS itself (max_iter=1, history_size=10, no line search) fed the same
gradients.  The native step keeps torch's fp32 arithmetic order but accumulates its dot products in fp64, so the bars
are self-calibrating: the native iterate may be at most twice as far from an fp64 torch run as an fp32 torch run is.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

import style_transfer_b200 as stb
from style_transfer_b200 import _lib
from oracle import st_oracle as O

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
H, W = 37, 53                        # n = 3 * 37 * 53 = 5883: not a multiple of 4 (the scalar tail runs too)
N = 3 * H * W
DECAY = float(np.float32(0.99))      # the EMA decay as the library holds it


def _tlib():
    return _lib.load_test()


def _rel(a, ref):
    a, ref = a.double().cpu().flatten(), ref.double().cpu().flatten()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


class TorchReplay:
    """torch.optim.LBFGS driven by scripted gradients, with the EMA of the iterate (value * d + (1 - d) * x)."""

    def __init__(self, x0, dtype):
        self.x = torch.nn.Parameter(x0.detach().clone().to(dtype))
        self.ema = (x0.double() * (1 - DECAY)).to(dtype)
        self.opt = torch.optim.LBFGS([self.x], max_iter=1, history_size=10)

    def step(self, g):
        def closure():
            self.x.grad = g.detach().clone().to(self.x.dtype)
            return torch.zeros((), dtype=self.x.dtype)

        self.opt.step(closure)
        self.ema.mul_(DECAY).add_(self.x.detach(), alpha=1 - DECAY)

    @property
    def state(self):
        return self.opt.state[self.x]

    @property
    def pairs(self):
        return len(self.state.get('old_dirs', []))

    @property
    def t(self):
        return float(self.state['t'])


class Native:
    """The launch sequence of stb_iterate_lbfgs' optimizer step (stb_test_lbfgs_step) on scripted gradients."""

    def __init__(self, x0):
        n = ctypes.c_size_t()
        _lib.check(_lib.load().stb_lbfgs_state_bytes(H, W, ctypes.byref(n)))
        self.bytes = n.value
        self.state = torch.empty(self.bytes, dtype=torch.uint8, device=DEV)
        self.x = x0.float().to(DEV).contiguous()
        self.ema = (x0.double() * (1 - DECAY)).float().to(DEV).contiguous()
        self.pairs, self.t = None, None
        self.reset()

    def reset(self):
        _lib.check(_lib.load().stb_lbfgs_reset(_lib.ptr(self.state), H, W, _lib.cur_stream()))

    def step(self, g):
        g = g.float().to(DEV).contiguous()
        pairs, t = ctypes.c_int(), ctypes.c_float()
        _lib.check(_tlib().stb_test_lbfgs_step(_lib.ptr(self.state), self.bytes, H, W, _lib.ptr(self.x), _lib.ptr(g),
                                               _lib.ptr(self.ema), DECAY, ctypes.byref(pairs), ctypes.byref(t),
                                               _lib.cur_stream()), test_lib=True)
        self.pairs, self.t = pairs.value, t.value


def _objectives():
    gen = torch.Generator().manual_seed(0)
    a = torch.logspace(-1, 1, N, dtype=torch.float64)[torch.randperm(N, generator=gen)]   # condition number 100
    b = torch.randn(N, dtype=torch.float64, generator=gen) * 0.1
    c = torch.randn(N, dtype=torch.float64, generator=gen)
    quad = lambda x: a * x + b                                          # grad of 0.5 a x^2 + b x
    nonconvex = lambda x: -0.3 * c * torch.sin(3 * x) + 0.1 * x         # grad of 0.1 sum c cos(3x) + 0.05 |x|^2
    return {'quadratic': quad, 'nonconvex': nonconvex}


def _record(grad_fn, steps, seed=1):
    """Gradients of a float64 torch L-BFGS run (evaluated along its own trajectory) and its start point."""
    x0 = torch.rand(N, dtype=torch.float64, generator=torch.Generator().manual_seed(seed))
    x = torch.nn.Parameter(x0.clone())
    opt = torch.optim.LBFGS([x], max_iter=1, history_size=10)
    gs = []

    def closure():
        g = grad_fn(x.detach())
        x.grad = g.clone()
        gs.append(g.clone())
        return torch.zeros((), dtype=torch.float64)

    for _ in range(steps):
        opt.step(closure)
    return x0, gs


def _run_script(x0, script):
    """Feeds the script (gradients, or 'reset') to native, fp64 and fp32 torch; checks x and the EMA at every step
    against the self-calibrating bar, the pair count and t against the fp64 run.  Returns per-step records."""
    nat, r64, r32 = Native(x0), TorchReplay(x0, torch.float64), TorchReplay(x0, torch.float32)
    recs = []
    for k, g in enumerate(script):
        if isinstance(g, str):
            assert g == 'reset'
            nat.reset()
            r64.opt = torch.optim.LBFGS([r64.x], max_iter=1, history_size=10)
            r32.opt = torch.optim.LBFGS([r32.x], max_iter=1, history_size=10)
            continue
        x_before = nat.x.clone()
        nat.step(g)
        r64.step(g)
        r32.step(g)
        torch.cuda.synchronize()
        e_nat, e32 = _rel(nat.x, r64.x.detach()), _rel(r32.x.detach(), r64.x.detach())
        ee_nat, ee32 = _rel(nat.ema, r64.ema), _rel(r32.ema, r64.ema)
        assert e_nat <= 2 * e32 + 1e-6, (k, e_nat, e32)
        assert ee_nat <= 2 * ee32 + 1e-6, (k, ee_nat, ee32)
        assert nat.pairs == r64.pairs, (k, nat.pairs, r64.pairs)
        if 't' in r64.state:
            assert abs(nat.t - r64.t) <= 1e-5 * abs(r64.t), (k, nat.t, r64.t)
        recs.append(dict(step=k, moved=not torch.equal(nat.x, x_before), pairs=nat.pairs, e_nat=e_nat, e32=e32,
                         n_iter=r64.state.get('n_iter', 0)))
    return recs


@pytest.mark.parametrize('name', ['quadratic', 'nonconvex'])
def test_scripted_gradients_match_torch(name):
    """30 steps (the 11-slot history ring wraps twice) on gradients recorded from a float64 torch run."""
    x0, gs = _record(_objectives()[name], 30)
    recs = _run_script(x0, gs)
    print(name, 'max native err', max(r['e_nat'] for r in recs), 'max fp32 torch err', max(r['e32'] for r in recs))
    assert recs[-1]['pairs'] == 10


def test_branch_opt_cond_leaves_everything_unchanged():
    """An all-zero gradient (max|g| <= 1e-7) returns before n_iter advances: a zero gradient FIRST must leave the next
    step a first iteration (t = min(1, 1/sum|g|)); one in the middle changes neither x nor the history."""
    x0, gs = _record(_objectives()['quadratic'], 8)
    zero = torch.zeros(N, dtype=torch.float64)
    recs = _run_script(x0, [zero] + gs[:4] + [zero] + gs[4:])
    assert not recs[0]['moved'] and recs[0]['n_iter'] == 0 and recs[0]['pairs'] == 0
    assert not recs[5]['moved'] and recs[5]['pairs'] == recs[4]['pairs'] and recs[5]['n_iter'] == recs[4]['n_iter']
    assert all(r['moved'] for i, r in enumerate(recs) if i not in (0, 5))


def test_branch_repeated_gradient_skips_the_pair():
    """The same gradient twice: y = 0, so y.s = 0 fails the 1e-10 test, the pair is not stored and H_diag is kept."""
    x0, gs = _record(_objectives()['nonconvex'], 8)
    recs = _run_script(x0, gs[:4] + [gs[3]] + gs[4:])
    assert recs[4]['pairs'] == recs[3]['pairs']


def test_branch_tiny_gradient_takes_no_step():
    """max|g| just above 1e-7 on a few entries: g.d > -1e-9, so x does not move -- but d and t are kept, and the next
    step's s = d * t uses them (torch's quirk).  Both as a first iteration and with a history."""
    x0, gs = _record(_objectives()['quadratic'], 8)
    tiny = torch.zeros(N, dtype=torch.float64)
    tiny[[5, 700, 4000]] = torch.tensor([2e-7, -3e-7, 1.5e-7], dtype=torch.float64)
    script = [tiny] + gs[:5] + [tiny] + gs[5:]
    recs = _run_script(x0, script)
    # the fp64 torch run took the break branch: n_iter advanced, x stayed (asserted against torch itself)
    r = TorchReplay(x0, torch.float64)
    r.step(tiny)
    assert r.state['n_iter'] == 1 and torch.equal(r.x.detach(), x0)
    assert not recs[0]['moved'] and recs[0]['n_iter'] == 1
    assert not recs[6]['moved'] and recs[6]['n_iter'] == recs[5]['n_iter'] + 1
    assert all(rc['moved'] for i, rc in enumerate(recs) if i not in (0, 6))


def test_branch_reset_starts_a_new_first_iteration():
    """stb_lbfgs_reset (a new scale): the next step is a first iteration again, as with a fresh optim.LBFGS."""
    x0, gs = _record(_objectives()['nonconvex'], 14)
    recs = _run_script(x0, gs[:7] + ['reset'] + gs[7:])
    assert recs[7]['n_iter'] == 1 and recs[7]['pairs'] == 0 and recs[6]['pairs'] > 0


# ---------------------------------------------------------------------------------------------- end to end
class TorchDrivenLBFGS(stb.StyleTransfer):
    """Reference runner: torch.optim.LBFGS on the host over the native closure st.loss_and_grad(), EMA after each
    step, no clamp -- what optimizer='lbfgs' computed before the step moved onto the device."""

    def _lbfgs_state(self, h, w):
        self._param = torch.nn.Parameter(self.image, requires_grad=True)
        self._opt = torch.optim.LBFGS([self._param], max_iter=1, history_size=10)
        self._terms = {}
        return None

    def _iterate_lbfgs(self, state, step, avg_decay):
        def closure():
            terms, grad = self.loss_and_grad()
            self._terms[step] = terms
            self._param.grad = grad
            return terms[0].to(self._dev)

        with torch.enable_grad():
            self._opt.step(closure)
        self.average.value.mul_(avg_decay).add_(self.image, alpha=1 - avg_decay)
        self.average.note_update()

    def _wait_loss(self, step):
        return self._terms[step]


class TorchDrivenLBFGS64(TorchDrivenLBFGS):
    """The same loop with the optimizer arithmetic in float64: the parameter is a float64 copy of the image, the native
    closure is evaluated at its fp32 rounding and hands its gradient back as float64.  This is the yardstick both fp32
    optimizers (torch's and the device's) are measured against."""

    def _lbfgs_state(self, h, w):
        self._param = torch.nn.Parameter(self.image.double(), requires_grad=True)
        self._opt = torch.optim.LBFGS([self._param], max_iter=1, history_size=10)
        self._terms = {}
        return None

    def _iterate_lbfgs(self, state, step, avg_decay):
        def closure():
            self.image.copy_(self._param.detach())
            terms, grad = self.loss_and_grad()
            self._terms[step] = terms
            self._param.grad = grad.double()
            return terms[0].double().to(self._dev)

        with torch.enable_grad():
            self._opt.step(closure)
        self.image.copy_(self._param.detach())
        self.average.value.mul_(avg_decay).add_(self.image, alpha=1 - avg_decay)
        self.average.note_update()


@pytest.mark.parametrize('kw', [dict(min_scale=64, end_scale=64, initial_iterations=8),
                                dict(min_scale=64, end_scale=91, initial_iterations=7, iterations=5)],
                         ids=['64x48_8its', 'pyramid_64_91'])
def test_stylize_lbfgs_matches_the_torch_driven_loop(vgg_weights, kw):
    """Native stylize(optimizer='lbfgs') against the torch-driven loop (fp32, what the option ran before), with the
    same loop on a float64 optimizer as the yardstick of how far rounding alone moves this trajectory.

    L-BFGS with t = 1 and no clamp amplifies rounding.  After the tiny first step (t = 1 / sum|g|), y = g1 - g0 is
    small against the closure's own bf16 rounding, and from the first stored pair on H_diag = y.s / y.y scales the
    whole direction.  Measured on an H100, per-iteration loss, 64 -> 91 pyramid, scale 2, iteration 3: native vs torch
    fp32 0.61, native vs fp64 optimizer 0.32, torch fp32 vs fp64 optimizer 2.42.  So the bar is self-calibrating: per
    scale and for the final EMA, native may differ from torch's fp32 run by at most twice what torch's fp32 run differs
    from the float64 one.  Before the first stored pair the two fp32 runs are bit-identical, and on the first scale
    they agree to 5e-4 (measured: 1.2e-4)."""
    content, style = O.synth_image(1, 16, 64, 48), O.synth_image(2, 32, 56, 40)
    runs = []
    for cls in (stb.StyleTransfer, TorchDrivenLBFGS, TorchDrivenLBFGS64):
        st = cls(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights)
        tr = []
        st.stylize(content, [style], optimizer='lbfgs', callback=lambda it: tr.append((it.loss, it.w, it.h)), **kw)
        runs.append((st, tr))
    (nat, tn), (ref, tr), (r64, t64) = runs
    assert [t[1:] for t in tn] == [t[1:] for t in tr] == [t[1:] for t in t64]
    ln, lr, l64 = (np.array([t[0] for t in x]) for x in (tn, tr, t64))
    first = kw['initial_iterations']
    assert len(ln) == first + (kw.get('iterations', 0) if kw['end_scale'] != kw['min_scale'] else 0)
    assert np.isfinite(ln).all()
    drift = np.abs(ln - lr) / np.abs(lr)
    e_nat, e32 = np.abs(ln - l64) / np.abs(l64), np.abs(lr - l64) / np.abs(l64)
    ema64 = r64.average.get()
    ema_nat, ema32 = _rel(nat.average.get(), ema64), _rel(ref.average.get(), ema64)
    print('loss drift native vs torch fp32', drift.tolist())
    print('loss error vs fp64 optimizer: native', e_nat.tolist(), 'torch fp32', e32.tolist())
    ema_drift = _rel(nat.average.get(), ref.average.get())
    print('final EMA error vs fp64 optimizer: native', ema_nat, 'torch fp32', ema32, 'native vs torch fp32', ema_drift)
    assert (drift[:2] == 0).all(), drift
    assert drift[:first].max() < 5e-4, drift
    for sl in (slice(0, first), slice(first, len(ln))):
        if sl.start < sl.stop:
            assert drift[sl].max() <= 2 * e32[sl].max() + 1e-5, (sl, drift[sl], e32[sl])
    assert ema_drift <= 2 * ema32 + 1e-5, (ema_drift, ema32)


def test_nan_gradient_keeps_stepping_like_torch():
    """A NaN in the gradient fails opt_cond in torch (NaN <= 1e-7 is false), so torch steps and the iterate turns NaN.
    The device must do the same rather than take the opt_cond exit and freeze the iterate."""
    x0, gs = _record(_objectives()['quadratic'], 4)
    bad = gs[3].clone()
    bad[17] = float('nan')
    nat, r64 = Native(x0), TorchReplay(x0, torch.float64)
    for g in gs[:3] + [bad]:
        nat.step(g)
        r64.step(g)
    torch.cuda.synchronize()
    assert r64.state['n_iter'] == 4 and torch.isnan(r64.x.detach()).all()
    assert torch.isnan(nat.x).all()


# ---------------------------------------------------------------------------------------------- graphs and errors
def _targets(st, Hi=48, Wi=64):
    m = st.model
    cimg = O.to_tensor(O.synth_image(1, 16, Wi, Hi)).to(DEV)
    simg = O.to_tensor(O.synth_image(2, 32, 56, 40)).to(DEV)
    m.ensure_workspace([(Hi, Wi), (40, 56)])
    ct = m.content_features(cimg)
    means, srms = m.style_stats(simg)
    m.set_targets(Hi, Wi, ct, 0.015, means, srms, st.style_weights, 2.0)
    torch.manual_seed(3)
    return (cimg + 0.05 * torch.randn_like(cimg)).clamp(0, 1).contiguous(), (ct, means, srms)


def _state(m, Hi, Wi):
    n = ctypes.c_size_t()
    _lib.check(m.lib.stb_lbfgs_state_bytes(Hi, Wi, ctypes.byref(n)))
    state = torch.empty(n.value, dtype=torch.uint8, device=DEV)
    _lib.check(m.lib.stb_lbfgs_reset(_lib.ptr(state), Hi, Wi, _lib.cur_stream()))
    return state


def _ten_iterations(vgg_weights, graphs):
    old = os.environ.get('STB_GRAPH')
    if not graphs:
        os.environ['STB_GRAPH'] = '0'    # read when the context is created
    try:
        st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights)
    finally:
        if old is None:
            os.environ.pop('STB_GRAPH', None)
        else:
            os.environ['STB_GRAPH'] = old
    m = st.model
    img, _ = _targets(st)
    x, ema = img.clone(), img * 0.01
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    losses = []
    replays0 = m.launch_count()[0]
    with torch.cuda.stream(side):
        state = _state(m, 48, 64)
        for step in range(1, 11):
            _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(x), _lib.ptr(ema), _lib.ptr(state), state.numel(), step,
                                               DECAY, None, _lib.cur_stream()))
            losses.append(st._wait_loss(step).clone())
    side.synchronize()
    return x.cpu(), ema.cpu(), torch.stack(losses), m.graph_status()[0], m.launch_count()[0] - replays0


def test_graphed_lbfgs_iterations_equal_eager_ones(vgg_weights):
    xg, eg, lg, status_g, replays_g = _ten_iterations(vgg_weights, graphs=True)
    xe, ee, le, status_e, replays_e = _ten_iterations(vgg_weights, graphs=False)
    assert status_g == 1 and status_e == 0
    assert replays_g >= 7 and replays_e == 0
    assert torch.isfinite(lg).all() and lg[-1, 0] < lg[0, 0]
    for a, b in ((xg, xe), (eg, ee), (lg, le)):
        torch.testing.assert_close(a, b, rtol=0, atol=0)


def test_lbfgs_errors_are_reported(vgg_weights):
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights)
    m = st.model
    img, (ct, means, srms) = _targets(st)
    ema = img * 0.01
    small = _state(m, 40, 64)          # sized for another H x W
    with pytest.raises(ValueError, match='too small'):
        _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(img), _lib.ptr(ema), _lib.ptr(small), small.numel(), 1,
                                           DECAY, None, _lib.cur_stream()))
    state = _state(m, 48, 64)
    with pytest.raises(ValueError):    # null image
        _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, None, _lib.ptr(ema), _lib.ptr(state), state.numel(), 1, DECAY, None,
                                           _lib.cur_stream()))
    m.set_band(True, 96, 0, 48)        # a banded context (a tiled Adam scale) cannot run L-BFGS
    m.set_targets(48, 64, ct, 0.015, means, srms, st.style_weights, 2.0)
    with pytest.raises(_lib.NativeError, match='error -4'):
        _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(img), _lib.ptr(ema), _lib.ptr(state), state.numel(), 1,
                                           DECAY, None, _lib.cur_stream()))
    m.set_band(False)                  # ... nor one whose targets are not set
    with pytest.raises(_lib.NativeError, match='error -4'):
        _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(img), _lib.ptr(ema), _lib.ptr(state), state.numel(), 1,
                                           DECAY, None, _lib.cur_stream()))
