"""-m gpu: optimizer='lbfgs' tiled over ranks (stb_iterate_lbfgs_banded), with the ranks as threads on ONE GPU.

Each rank keeps the L-BFGS vectors of its own rows; every dot product of the step is summed over the ranks by a one-block
kernel inside the iteration (ranks combined in rank order), so every rank holds bit-identical scalars.  The ranks run as
threads of this process with their own contexts and streams on cuda:0 (distributed.ThreadGroup, mailboxes connected
with stb_comm_connect_local), as in test_gpu_tiled.py.

The scripted tests feed the banded step (stb_test_lbfgs_step_banded) and the untiled one (stb_test_lbfgs_step) the same
gradients: multiples of 2^-16, and in apron mode split between a row's owner and the neighbour's apron copy so that the
seam sum is exact in fp32.  The end-to-end tests hold stylize(optimizer='lbfgs') tiled against the untiled native run
(see _check_end_to_end for the bars).
"""
import contextlib
import ctypes
import gc
import io
import os
import threading

import numpy as np
import pytest
import torch

import style_transfer_b200 as stb
from style_transfer_b200 import _lib
from style_transfer_b200 import distributed as D
from style_transfer_b200.style_transfer import NativeVGG
from oracle import st_oracle as O
import test_gpu_lbfgs as L

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
DECAY = L.DECAY
Q = 2.0 ** -16
HDR_BYTES = 136          # n_iter, count, head, skip, took_step, pad, t, H_diag, gtd, pad, ro[11], al[11]


def _tlib():
    return _lib.load_test()


def _threads(world, fn):
    """Runs fn(rank, group) on `world` threads; returns the results in rank order.  The garbage collector is off while
    they run: a finalizer that frees device memory synchronises the device, and run on one rank's thread while a peer's
    reduction kernel waits for that rank it would stall both."""
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '20')
    shared = D.ThreadGroup.Shared(world)
    results, errors = [None] * world, []
    gc.collect()
    gc.disable()

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            results[rank] = fn(rank, D.ThreadGroup(shared, rank))
        except BaseException as e:  # noqa: BLE001 -- report and release the other ranks
            errors.append((rank, repr(e)))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    gc.enable()
    assert not errors, errors
    assert all(r is not None for r in results), 'a rank did not finish'
    return results


# ---------------------------------------------------------------------------------------------- scripted steps
def _grad_fns(n):
    gen = torch.Generator().manual_seed(0)
    a = torch.logspace(-1, 1, n, dtype=torch.float64)[torch.randperm(n, generator=gen)]   # condition number 100
    b = torch.randn(n, dtype=torch.float64, generator=gen) * 0.1
    c = torch.randn(n, dtype=torch.float64, generator=gen)
    return {'quadratic': lambda x: a * x + b, 'nonconvex': lambda x: -0.3 * c * torch.sin(3 * x) + 0.1 * x}


def _record(grad_fn, n, steps):
    """Gradients of a float64 torch L-BFGS run along its own trajectory, rounded to multiples of 2^-16 (exact in fp32,
    and so are the seam splits of _local_grad)."""
    x0 = torch.rand(n, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    x = torch.nn.Parameter(x0.clone())
    opt = torch.optim.LBFGS([x], max_iter=1, history_size=10)
    gs = []

    def closure():
        g = grad_fn(x.detach())
        x.grad = g.clone()
        gs.append(torch.round(g / Q) * Q)
        return torch.zeros((), dtype=torch.float64)

    for _ in range(steps):
        opt.step(closure)
    return x0, gs


def _local_grad(g, band, bands, add_seams):
    """This rank's local gradient [3][h_local][W] for the full gradient g [3][H][W].  Apron mode: the first APRON own
    rows of a band below another keep g - a (a = ~g/4 goes to the upper band's bottom apron), the last APRON own rows of
    a band above another keep g - b (b = ~3g/8 goes to the lower band's top apron); all parts are multiples of 2^-16.
    Halo mode: the own rows hold g, the apron rows NaN (the step must not read them)."""
    ap = D.APRON
    if not add_seams:
        out = torch.full((3, band.h_local, g.shape[2]), float('nan'), dtype=torch.float64)
        out[:, band.own0:band.own0 + band.own_rows] = g[:, band.own_begin:band.own_end]
        return out
    a = torch.zeros_like(g)
    b = torch.zeros_like(g)
    for bd in bands:
        if bd.rank > 0:
            a[:, bd.own_begin:bd.own_begin + ap] = torch.round(g[:, bd.own_begin:bd.own_begin + ap] * 0.25 / Q) * Q
        if bd.rank + 1 < bd.world:
            b[:, bd.own_end - ap:bd.own_end] = torch.round(g[:, bd.own_end - ap:bd.own_end] * 0.375 / Q) * Q
    own = g - a - b
    out = torch.zeros((3, band.h_local, g.shape[2]), dtype=torch.float64)
    out[:, band.own0:band.own0 + band.own_rows] = own[:, band.own_begin:band.own_end]
    if band.rank > 0:          # top apron = the upper band's last own rows: their share b
        out[:, :band.own0] = b[:, band.loc_begin:band.own_begin]
    if band.rank + 1 < band.world:   # bottom apron = the lower band's first own rows: their share a
        out[:, band.own0 + band.own_rows:] = a[:, band.own_end:band.loc_end]
    return out


def _untiled(x0, script, H, W):
    n = ctypes.c_size_t()
    _lib.check(_lib.load().stb_lbfgs_state_bytes(H, W, ctypes.byref(n)))
    state = torch.empty(n.value, dtype=torch.uint8, device=DEV)
    _lib.check(_lib.load().stb_lbfgs_reset(_lib.ptr(state), H, W, _lib.cur_stream()))
    x = x0.float().to(DEV).contiguous()
    ema = (x0.double() * (1 - DECAY)).float().to(DEV).contiguous()
    recs = []
    for g in script:
        g = g.float().to(DEV).contiguous()
        pairs, t = ctypes.c_int(), ctypes.c_float()
        _lib.check(_tlib().stb_test_lbfgs_step(_lib.ptr(state), n.value, H, W, _lib.ptr(x), _lib.ptr(g), _lib.ptr(ema),
                                               DECAY, ctypes.byref(pairs), ctypes.byref(t), _lib.cur_stream()),
                   test_lib=True)
        recs.append(dict(pairs=pairs.value, t=t.value, x=x.cpu().clone(), ema=ema.cpu().clone(),
                         hdr=state[:HDR_BYTES].cpu().clone()))
    return recs


def _banded(wts, world, x0, script, H, W, add_seams):
    """The same script on `world` thread-ranks; per rank, per step: pairs, t, header bytes, the local x and ema."""
    bands = D.all_bands(H, world)
    assert all(b is not None for b in bands)
    # every kernel of the test library is loaded before the ranks step (a lazy load at a first launch would synchronise
    # the context while a peer's reduction kernel waits for this rank)
    _lib.check(_tlib().stb_test_preload(), test_lib=True)
    cap_h = max(b.h_local for b in bands)

    def rank_fn(rank, g):
        band = bands[rank]
        stream = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(stream):
            m = NativeVGG(wts, 'max', DEV)
            _, p = m.comm_create(rank, world, cap_h, W)
            m.comm_connect_local(g.all_gather_object(p))
            m.comm_set_geometry(W, band, bands[rank - 1] if rank > 0 else None,
                                bands[rank + 1] if rank + 1 < world else None, False)
            g.barrier()
            m.comm_reset()
            g.barrier()
            n = ctypes.c_size_t()
            _lib.check(m.lib.stb_lbfgs_state_bytes(band.own_rows, W, ctypes.byref(n)))
            state = torch.empty(n.value, dtype=torch.uint8, device=DEV)
            _lib.check(m.lib.stb_lbfgs_reset(_lib.ptr(state), band.own_rows, W, _lib.cur_stream()))
            full = x0.view(3, H, W)
            x = full[:, band.loc_begin:band.loc_end].float().to(DEV).contiguous()
            ema = (full[:, band.loc_begin:band.loc_end].double() * (1 - DECAY)).float().to(DEV).contiguous()
            # everything the steps touch exists before they start: while the ranks step, nothing but stream-ordered
            # work is issued (a device allocation or a synchronous copy could stall a rank a peer's reduction waits for)
            grads = [_local_grad(gf.view(3, H, W), band, bands, add_seams).float().to(DEV).contiguous() for gf in script]
            xs, emas = torch.empty((len(script),) + x.shape, device=DEV), torch.empty((len(script),) + x.shape, device=DEV)
            hdrs = torch.empty(len(script), HDR_BYTES, dtype=torch.uint8, device=DEV)
            stream.synchronize()
            g.barrier()
            for k, gl in enumerate(grads):
                _lib.check(_tlib().stb_test_lbfgs_step_banded(m.ctx, _lib.ptr(state), n.value, _lib.ptr(x),
                                                              _lib.ptr(gl), _lib.ptr(ema), DECAY, add_seams, None,
                                                              None, _lib.cur_stream()), test_lib=True)
                xs[k].copy_(x)
                emas[k].copy_(ema)
                hdrs[k].copy_(state[:HDR_BYTES])
            stream.synchronize()
            g.barrier()            # nobody frees a mailbox a neighbour may still read
            hdrs = hdrs.cpu()
            recs = [dict(pairs=int(h[4:8].view(torch.int32)[0]), t=float(h[32:36].view(torch.float32)[0]),
                         x=xx, ema=ee, hdr=h) for h, xx, ee in zip(hdrs, xs.cpu(), emas.cpu())]
            m.comm_disconnect()
            g.barrier()
            return recs

    return bands, _threads(world, rank_fn)


def _compare(bands, ranks, ref, H, W, check_values=True):
    """Per step: pairs and t equal the untiled run's, the header is bit-identical across ranks, the halo rows hold the
    neighbours' own rows of the previous step, and (check_values) x / ema of the own rows are within 1e-6 of the
    untiled run.  Returns (steps, bit-identical steps)."""
    identical = 0
    for k, r0 in enumerate(ref):
        for band, recs in zip(bands, ranks):
            rec = recs[k]
            assert rec['pairs'] == r0['pairs'] and rec['t'] == r0['t'], (k, band.rank, rec['pairs'], r0['pairs'],
                                                                        rec['t'], r0['t'])
            assert torch.equal(rec['hdr'], ranks[0][k]['hdr']), (k, band.rank)
            if band.rank > 0 and k > 0:
                up, urecs = bands[band.rank - 1], ranks[band.rank - 1]
                np.testing.assert_array_equal(rec['x'][:, :band.own0].numpy(),
                                              urecs[k - 1]['x'][:, up.own0 + up.own_rows - band.own0:
                                                                up.own0 + up.own_rows].numpy())
            if band.rank + 1 < band.world and k > 0:
                dn, drecs = bands[band.rank + 1], ranks[band.rank + 1]
                np.testing.assert_array_equal(rec['x'][:, band.own0 + band.own_rows:].numpy(),
                                              drecs[k - 1]['x'][:, dn.own0:dn.own0 + band.bottom_apron].numpy())
        if not check_values:
            continue
        same = True
        for key in ('x', 'ema'):
            ref_full = r0[key].view(3, H, W)
            got = torch.cat([recs[k][key][:, b.own0:b.own0 + b.own_rows] for b, recs in zip(bands, ranks)], dim=1)
            rel = L._rel(got, ref_full)
            assert rel <= 1e-6, (k, key, rel)
            same = same and torch.equal(got, ref_full)
        identical += same
    return len(ref), identical


GEOMS = [(2, 256, 181), (3, 400, 64), (4, 512, 48)]   # 181: scalar path; 3 ranks: unequal bands (128, 144, 128 rows)


@pytest.mark.parametrize('seams', ['apron', 'halo'])
@pytest.mark.parametrize('name', ['quadratic', 'nonconvex'])
@pytest.mark.parametrize('world,H,W', GEOMS)
def test_scripted_banded_step_equals_untiled(vgg_weights, world, H, W, name, seams):
    """30 steps (the ring wraps) of the banded step against the untiled one on the same gradients."""
    n = 3 * H * W
    x0, gs = _record(_grad_fns(n)[name], n, 30)
    ref = _untiled(x0, gs, H, W)
    bands, ranks = _banded(vgg_weights, world, x0, gs, H, W, int(seams == 'apron'))
    steps, same = _compare(bands, ranks, ref, H, W)
    print(f'world {world} {H}x{W} {name} {seams}: x and EMA bit-identical to the untiled step in {same}/{steps} steps')
    assert ref[-1]['pairs'] == 10


def _branch_run(wts, script, world=2, H=256, W=64):
    x0 = torch.rand(3 * H * W, dtype=torch.float64, generator=torch.Generator().manual_seed(1))
    ref = _untiled(x0, script, H, W)
    bands, ranks = _banded(wts, world, x0, script, H, W, 1)
    return x0, bands, ranks, ref


def _n_iter(rec):
    return int(rec['hdr'][:4].view(torch.int32)[0])


def _moved(recs, k, band):
    own = slice(band.own0, band.own0 + band.own_rows)
    return not torch.equal(recs[k]['x'][:, own], recs[k - 1]['x'][:, own])


def _branch_script(H=256, W=64, steps=8):
    n = 3 * H * W
    _, gs = _record(_grad_fns(n)['quadratic'], n, steps)
    return gs


def test_branch_zero_gradient_on_one_rank_still_steps(vgg_weights):
    """max|g| is global: a gradient that is zero on rank 0's rows only passes opt_cond on every rank, n_iter advances
    everywhere, and rank 0's rows move (the direction mixes in the stored pairs)."""
    H, W = 256, 64
    gs = _branch_script(H, W)
    z = gs[4].clone().view(3, H, W)
    z[:, :D.band_edges(H, 2)[1]] = 0
    script = gs[:4] + [z.flatten()] + gs[4:]
    _, bands, ranks, ref = _branch_run(vgg_weights, script, H=H, W=W)
    _compare(bands, ranks, ref, H, W)
    for b, recs in zip(bands, ranks):
        assert _n_iter(recs[4]) == _n_iter(recs[3]) + 1
        assert _moved(recs, 4, b), b.rank


def test_branch_zero_gradient_everywhere_changes_nothing(vgg_weights):
    H, W = 256, 64
    gs = _branch_script(H, W)
    script = gs[:4] + [torch.zeros_like(gs[0])] + gs[4:]
    _, bands, ranks, ref = _branch_run(vgg_weights, script, H=H, W=W)
    _compare(bands, ranks, ref, H, W)
    for b, recs in zip(bands, ranks):
        assert _n_iter(recs[4]) == _n_iter(recs[3]) and recs[4]['pairs'] == recs[3]['pairs']
        assert not _moved(recs, 4, b)


def test_branch_repeated_gradient_rejects_the_pair(vgg_weights):
    H, W = 256, 64
    gs = _branch_script(H, W)
    script = gs[:4] + [gs[3]] + gs[4:]
    _, bands, ranks, ref = _branch_run(vgg_weights, script, H=H, W=W)
    _compare(bands, ranks, ref, H, W)
    for recs in ranks:
        assert recs[4]['pairs'] == recs[3]['pairs']


def test_branch_tiny_gradient_takes_no_step(vgg_weights):
    """max|g| just above 1e-7 on entries of both bands: g.d > -1e-9, n_iter advances, x stays."""
    H, W = 256, 64
    gs = _branch_script(H, W)
    tiny = torch.zeros(3 * H * W, dtype=torch.float64)
    tiny[[5, 10 * W + 7, 2 * H * W + 200 * W + 3]] = torch.tensor([2e-7, -3e-7, 1.5e-7], dtype=torch.float64)
    script = gs[:5] + [tiny] + gs[5:]
    _, bands, ranks, ref = _branch_run(vgg_weights, script, H=H, W=W)
    _compare(bands, ranks, ref, H, W)
    for b, recs in zip(bands, ranks):
        assert _n_iter(recs[5]) == _n_iter(recs[4]) + 1
        assert not _moved(recs, 5, b)


def test_branch_nan_on_one_rank_steps_every_rank_into_nan(vgg_weights):
    """A NaN fails opt_cond (NaN <= 1e-7 is false) and poisons every dot product: like torch, every rank steps and its
    whole band turns NaN."""
    H, W = 256, 64
    gs = _branch_script(H, W, 4)
    bad = gs[3].clone()
    bad[17] = float('nan')              # rank 0's rows only
    _, bands, ranks, ref = _branch_run(vgg_weights, gs[:3] + [bad], H=H, W=W)
    _compare(bands, ranks, ref[:3], H, W)
    assert torch.isnan(ref[3]['x']).all()
    for b, recs in zip(bands, ranks):
        assert _n_iter(recs[3]) == 4
        assert torch.isnan(recs[3]['x'][:, b.own0:b.own0 + b.own_rows]).all(), b.rank


# ---------------------------------------------------------------------------------------------- end to end
def _stylize_tiled(world, content, style, wts, kw):
    def rank_fn(rank, g):
        st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts, distributed=g)
        trace = []
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], optimizer='lbfgs', callback=lambda it: trace.append((it.loss, it.w, it.h)),
                       **kw)
        return (trace, st.average.get().cpu(), (st._comm_mode, 'halo' if st._halo_now else 'apron'),
                st.model.graph_status())

    return _threads(world, rank_fn)


_REFS = {}


def _untiled_ref(content, style, wts, kw, key):
    """Trace and final EMA of the untiled native run (cached per job)."""
    if key not in _REFS:
        st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts, distributed=False)
        tr = []
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], optimizer='lbfgs', callback=lambda it: tr.append((it.loss, it.w, it.h)), **kw)
        _REFS[key] = (tr, st.average.get().cpu())
    return _REFS[key]


def _check_end_to_end(tiled, ref, mode):
    """Every rank ends with the same bits; graphs replay; before the first stored pair the loss drifts by no more than
    the summation order of the split statistics moves it (5e-4, the tiled Adam bar).  After it, L-BFGS amplifies that
    closure-level difference: H_diag = y.s / y.y rescales the whole direction and there is no clamp.  Measured on an
    H100 over these jobs: up to 6.4e-3 relative in the loss and 2.4e-3 mean |diff| in the final EMA (bars 1e-2 and
    5e-3), against 1e-5 .. 1.3e-4 between torch's fp32 and fp64 optimizers on the untiled closure -- a yardstick of
    optimizer rounding alone, which a changed closure does not meet."""
    tn, en = ref
    trace, ema = tiled[0][0], tiled[0][1]
    for rank, (tr, e, md, (gs_, nt)) in enumerate(tiled):
        assert md == ('peer', mode), (rank, md)
        assert gs_ == 1, f'rank {rank}: iterations did not replay as a CUDA graph ({nt})'
        assert [t[1:] for t in tr] == [t[1:] for t in tn]
        assert tr == trace and torch.equal(e, ema), rank      # bit-identical across ranks
    lt, ln = (np.array([t[0] for t in x]) for x in (trace, tn))
    assert np.isfinite(lt).all()
    drift = np.abs(lt - ln) / np.abs(ln)
    ema_diff = (ema - en).abs().mean().item()
    print(mode, 'loss drift tiled vs untiled', drift.tolist(), 'final EMA mean |diff|', ema_diff)
    assert drift[:2].max() <= 5e-4, drift
    assert drift.max() <= 1e-2, drift
    assert ema_diff < 5e-3, ema_diff


@pytest.mark.parametrize('tile', ['halo', 'apron'])
@pytest.mark.parametrize('world,W,H,its', [(2, 512, 384, 6), (3, 200, 400, 5), (2, 362, 384, 4), (4, 256, 512, 4)])
def test_stylize_lbfgs_tiled_matches_untiled(vgg_weights, monkeypatch, tile, world, W, H, its):
    monkeypatch.setenv('STB_TILE', tile)
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
    scale = max(H, W)
    kw = dict(min_scale=scale, end_scale=scale, initial_iterations=its)
    tiled = _stylize_tiled(world, content, style, vgg_weights, kw)
    ref = _untiled_ref(content, style, vgg_weights, kw, (W, H, its))
    assert len(tiled[0][0]) == its
    _check_end_to_end(tiled, ref, tile)


@pytest.mark.parametrize('tile', ['halo', 'apron'])
def test_stylize_lbfgs_pyramid_mixes_replicated_and_banded_scales(vgg_weights, monkeypatch, tile):
    """128 -> 384 at 2 ranks: the 136-row scale is too small to tile and runs replicated, the others banded."""
    monkeypatch.setenv('STB_TILE', tile)
    W, H = 288, 384
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, 260, 300)
    kw = dict(min_scale=128, end_scale=384, iterations=3, initial_iterations=4)
    tiled = _stylize_tiled(2, content, style, vgg_weights, kw)
    ref = _untiled_ref(content, style, vgg_weights, kw, 'pyramid')
    heights = sorted({t[2] for t in ref[0]})
    assert D.make_band(heights[0], 0, 2) is None and D.make_band(heights[-1], 0, 2) is not None
    assert len(tiled[0][0]) == 4 + 3 * (len(heights) - 1)
    _check_end_to_end(tiled, ref, tile)


def test_graphed_banded_lbfgs_equals_eager(vgg_weights):
    """10 banded iterations at 2 ranks: CUDA-graph replay and eager launches give the same bits."""
    content, style = O.synth_image(1, 16, 256, 256), O.synth_image(2, 32, 168, 152)
    kw = dict(min_scale=256, end_scale=256, initial_iterations=10)
    runs = []
    for graphs in (True, False):
        old = os.environ.get('STB_GRAPH')
        if not graphs:
            os.environ['STB_GRAPH'] = '0'     # read when the contexts are created
        try:
            runs.append(_stylize_tiled(2, content, style, vgg_weights, kw))
        finally:
            if old is None:
                os.environ.pop('STB_GRAPH', None)
            else:
                os.environ['STB_GRAPH'] = old
    graphed, eager = runs
    for g, e in zip(graphed, eager):
        assert g[3][0] == 1 and e[3][0] == 0
        assert len(g[0]) == 10 and g[0] == e[0]
        assert torch.equal(g[1], e[1])


# ---------------------------------------------------------------------------------------------- errors
def test_lbfgs_banded_errors_are_reported_before_any_launch(vgg_weights):
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights, distributed=False)
    m = st.model
    Hl, W = 96, 64
    img, (ct, means, srms) = L._targets(st, Hl, W)
    ema = img * 0.01

    def call(state, nbytes):
        _lib.check(m.lib.stb_iterate_lbfgs_banded(m.ctx, _lib.ptr(img), _lib.ptr(ema), ctypes.c_void_p(state),
                                                  nbytes, 1, DECAY, None, _lib.cur_stream()))

    def sized(rows):
        n = ctypes.c_size_t()
        _lib.check(m.lib.stb_lbfgs_state_bytes(rows, W, ctypes.byref(n)))
        t = torch.zeros(n.value + 512, dtype=torch.uint8, device=DEV)
        return t, (t.data_ptr() + 255) // 256 * 256, n.value

    keep, state, nbytes = sized(Hl)
    with pytest.raises(_lib.NativeError, match='error -4'):     # no band
        call(state, nbytes)
    m.set_band(True, Hl, 0, Hl)
    m.set_targets(Hl, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    with pytest.raises(_lib.NativeError, match='error -4'):     # no comm connection / geometry
        call(state, nbytes)
    _, p = m.comm_create(0, 1, Hl, W)
    m.comm_connect_local([p])
    full = D.Band(0, 1, Hl, 0, Hl - 16, 0, Hl - 16)            # a geometry of 80 own rows: not this band
    m.comm_set_geometry(W, full, None, None, False)
    with pytest.raises(_lib.NativeError, match='error -4'):     # geometry does not match the band
        call(state, nbytes)
    m.comm_set_geometry(W, D.Band(0, 1, Hl, 0, Hl, 0, Hl), None, None, False)
    keep_small, small, small_bytes = sized(Hl - 16)
    with pytest.raises(ValueError, match='too small'):
        call(small, small_bytes)
    with pytest.raises(ValueError, match='aligned'):
        call(state + 16, nbytes)
    torch.cuda.synchronize()
    assert st.model.graph_status()[0] == 2    # nothing was captured (or launched) by the refused calls
