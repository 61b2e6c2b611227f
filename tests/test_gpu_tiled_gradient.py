"""-m gpu: the image gradient of the tiled iteration, row by row, against the untiled closure on the same statistics.

A tiled run and an untiled run of the same job differ by ~1e-5 in the loss, and only because the band-local statistics
are summed in another order.  This file removes that difference and compares the pieces the tiled closure is built from
(own-row restriction of statistics and tap gradients, the seam reduce of apron mode, the per-layer halo rows of halo
mode, floor-mode pooling on a ragged bottom band) against exact expectations:

  R = a context with a one-band band (stb_set_band(ctx, 1, H, 0, H)) and the same targets: its closure is the untiled
      one (asserted in test_reference_is_the_untiled_closure), and its statistics block can be written between
      stb_iterate_fwd and stb_iterate_bwd.
  g_ref = R's gradient with the statistics block the tiled ranks all-reduced injected before its backward pass.

The ranks run as threads on one GPU (distributed.ThreadGroup, mailboxes and halo-mode workspaces connected with plain
device pointers), as in test_gpu_lbfgs_tiled.py.

Measured on an NVIDIA H100 80GB HBM3 (400 W limit) over the 12 cases of test_tiled_iteration_matches_the_untiled_closure
(the whole file runs in ~15 s there):
  - halo mode: every own row of the tiled gradient equals g_ref bit for bit, in all six geometries.
  - apron mode: every own row at least APRON = 80 rows from every seam equals g_ref bit for bit (the backward receptive
    field of relu5_1 is 77.5 rows).  Rows nearer a seam differ only by where the bf16 roundings of the intermediate
    gradients fall (each side's share is rounded on its own, then the two are summed in fp32): per row, max |g - g_ref|
    / max |g_ref| reached 2.57e-3 (3 ranks, 400 x 200), over a whole seam zone 2.06e-3 (4 ranks, 1024^2).  Bars 6e-3
    and 5e-3.
  - the loss terms equal R's on the injected statistics, and every rank holds the same reduced statistics and loss, bit
    for bit; each band's content target equals R's on its own rows, bit for bit.
  - statistics, tiled reduced block vs R's own block, per segment (5 Gram matrices, 5 channel sums, content SSE, TV
    sum): at most 3.8e-7 relative (fp32 summation order).  Bar 1.5e-6.  A row missing from a band is ~1/rows of a
    segment.
  - Adam on a band vs the float64 reference fed the gradient read back from the L-BFGS state: 8.7e-7 (bar 2e-6, as
    tests/test_gpu_iterate.py).
Hand-made mutations (not committed), each of which made this file fail:
  1. no lower-neighbour seam add (has_dn = false in adam_seam_kernel and lbfgs_seam_gather_kernel): the apron-mode seam
     bars fail in all six geometries, per row 0.40 ... 0.48 (bar 6e-3), per zone 0.26 ... 0.34 (bar 5e-3); the
     seam sum restated in torch (case (e)) no longer equals the peer-mode gradient.
  2. the backward pass's halo exchanges publish their stamps but copy no row: the halo-mode bit identity fails in all
     six geometries, max |g - g_ref| / max |g_ref| 0.29 ... 0.52.
  3. band_rows gives a bottom band with own rows below local row 0 one row fewer at the pooled levels: the statistics
     check fails in all 12 cases, first at the level-1 Gram matrix with 3.3e-3 ... 9.1e-3 (bar 1.5e-6), up to 3.5e-2 in
     the level-4 channel sums.
"""
import ctypes
import gc
import os
import threading

import numpy as np
import pytest
import torch

from style_transfer_b200 import _lib
from style_transfer_b200 import distributed as D
from style_transfer_b200.style_transfer import NativeVGG
from oracle import st_oracle as O
from test_gpu_iterate import _adam_reference

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
DECAY = float(np.float32(0.99))     # the EMA decay as the library holds it
CONTENT_WEIGHT, TV_WEIGHT, LR = 0.015, 2.0, 0.02
STYLE_WEIGHTS = [w / 341 for w in (256, 64, 16, 4, 1)]
STYLE_C = [64, 128, 256, 512, 512]
FIRST_STEP = 7                      # Adam starts from a warm state, as after a previous scale

# the reduced statistics block: per style layer the raw Gram sums then the channel sums, then content SSE and TV sum
SEGMENTS = []
_o = 0
for _l, _c in enumerate(STYLE_C):
    SEGMENTS += [(f'gram{_l + 1}', _o, _o + _c * _c), (f'sums{_l + 1}', _o + _c * _c, _o + _c * _c + _c)]
    _o += _c * _c + _c
SEGMENTS += [('content_sse', _o, _o + 1), ('tv_sum', _o + 1, _o + 2)]

# bars (measurements in the module docstring)
STATS_BAR = 1.5e-6      # per segment, tiled reduced block vs R's own block (fp32 summation order)
SEAM_ROW_BAR = 6e-3     # apron mode: max |g - g_ref| / max |g_ref| over one own row within APRON rows of a seam
SEAM_ZONE_BAR = 5e-3    # the same over the whole seam zone of a band
ADAM_BAR = 2e-6         # relative to the largest magnitude, as tests/test_gpu_iterate.py


def _tlib():
    return _lib.load_test()


class _DeviceFloats:
    """A device range of fp32 values torch can alias (through the CUDA array interface) without copying."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {'shape': (n,), 'typestr': '<f4', 'data': (ptr, False), 'version': 2}


def _stats_block(m, h, w):
    """fp32 tensor aliasing the context's statistics block (works for torch-owned and library-owned workspaces)."""
    p, n = ctypes.c_void_p(), ctypes.c_size_t()
    _lib.check(m.lib.stb_stats_block(m.ctx, h, w, ctypes.byref(p), ctypes.byref(n)))
    return torch.as_tensor(_DeviceFloats(p.value, n.value))


def _lbfgs_state(m, h, w):
    n = ctypes.c_size_t()
    _lib.check(m.lib.stb_lbfgs_state_bytes(h, w, ctypes.byref(n)))
    state = torch.empty(n.value, dtype=torch.uint8, device=DEV)
    _lib.check(m.lib.stb_lbfgs_reset(_lib.ptr(state), h, w, _lib.cur_stream()))
    return state


def _lbfgs_gradient(state, h, w, out):
    _lib.check(_tlib().stb_test_lbfgs_gradient(_lib.ptr(state), state.numel(), h, w, _lib.ptr(out),
                                               _lib.cur_stream()), test_lib=True)


def _rel(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _threads(world, fn):
    """fn(rank, group) on `world` threads, results in rank order.  The garbage collector is off while they run: a
    finalizer that frees device memory synchronises the device, and run on one rank's thread while a peer's wait kernel
    waits for that rank it would stall both."""
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


# ---------------------------------------------------------------------------------------------- the job and R
class Job:
    """Content, style moments (computed once, handed to every context), the iterate (content plus noise, clamped), a
    warm Adam state, and the reference context R with a one-band band."""

    def __init__(self, wts, H, W):
        self.wts, self.H, self.W = wts, H, W
        self.content = O.to_tensor(O.synth_image(1, 16, W, H)).to(DEV).contiguous()
        style = O.to_tensor(O.synth_image(2, 32, 200, 152)).to(DEV).contiguous()
        self.R = NativeVGG(wts, 'max', DEV)
        self.R.ensure_workspace([(H, W), tuple(style.shape[2:])])
        self.means, self.srms = self.R.style_stats(style)
        self.ct = self.R.content_features(self.content)
        torch.manual_seed(3)
        self.img = (self.content + 0.05 * torch.randn_like(self.content)).clamp(0, 1).contiguous()
        gen = torch.Generator().manual_seed(FIRST_STEP)
        self.exp_avg = (1e-4 * torch.randn(self.img.shape, generator=gen)).to(DEV)
        self.exp_avg_sq = ((1e-4 * torch.randn(self.img.shape, generator=gen)) ** 2).to(DEV)
        self.loss = torch.zeros(8, dtype=torch.float32).pin_memory()
        self.set_band(True)
        self.stats = _stats_block(self.R, H, W)
        torch.cuda.synchronize()

    def set_band(self, on):
        self.R.set_band(on, self.H, 0, self.H)
        self.R.set_targets(self.H, self.W, self.ct, CONTENT_WEIGHT, self.means, self.srms, STYLE_WEIGHTS, TV_WEIGHT)

    def closure(self, inject=None):
        """R's (gradient, loss terms, own statistics block); `inject` replaces the statistics before the backward."""
        grad = torch.empty_like(self.img)
        self.R.iterate_fwd(self.img)
        own = self.stats.clone()
        if inject is not None:
            self.stats.copy_(inject)
        self.R.iterate_bwd(self.img, grad, self.loss)
        torch.cuda.synchronize()
        return grad[0], self.loss.clone(), own


_JOB = {}


def _job(wts, H, W):
    if (H, W) not in _JOB:
        _JOB.clear()
        torch.cuda.empty_cache()
        _JOB[(H, W)] = Job(wts, H, W)
    return _JOB[(H, W)]


GEOMS = [(2, 384, 512), (3, 400, 200), (4, 512, 256), (2, 362, 181), (3, 453, 362), (4, 1024, 1024)]


@pytest.mark.parametrize('H,W', sorted({(h, w) for _, h, w in GEOMS}))
def test_reference_is_the_untiled_closure(vgg_weights, H, W):
    """R's gradient on its own statistics equals stb_iterate_ex(apply_update=0) on the unbanded context, and the
    gradient stb_iterate_lbfgs consumed (read back from its state) equals both, bit for bit."""
    job = _job(vgg_weights, H, W)
    job.set_band(False)
    m, img = job.R, job.img.clone()
    g_ex, loss_ex = torch.empty_like(img), torch.zeros(8).pin_memory()
    _lib.check(m.lib.stb_iterate_ex(m.ctx, _lib.ptr(img), None, None, None, 0, 0.0, 0.9, 0.99, 1e-8, 0.0, 0,
                                    _lib.ptr(g_ex), _lib.ptr(loss_ex), _lib.cur_stream()))
    state = _lbfgs_state(m, H, W)
    x, ema = img.clone(), img * (1 - DECAY)
    g_lb = torch.empty(3, H, W, device=DEV)
    _lib.check(m.lib.stb_iterate_lbfgs(m.ctx, _lib.ptr(x), _lib.ptr(ema), _lib.ptr(state), state.numel(), 1, DECAY,
                                       None, _lib.cur_stream()))
    _lbfgs_gradient(state, H, W, g_lb)
    torch.cuda.synchronize()
    job.set_band(True)
    g_r, loss_r, _ = job.closure()
    assert torch.equal(g_r, g_ex[0]), _rel(g_r, g_ex[0])
    assert torch.equal(g_lb, g_ex[0]), _rel(g_lb, g_ex[0])
    assert torch.equal(loss_r, loss_ex), (loss_r, loss_ex)
    assert torch.isfinite(g_r).all() and g_r.abs().max() > 0


# ---------------------------------------------------------------------------------------------- the tiled ranks
def _run_ranks(job, world, halo):
    """Per rank: (c) one stb_iterate_lbfgs_banded step from a reset state, its gradient read through the state;
    (d) after a comm reset, two stb_iterate_banded Adam iterations from the warm state on the restored image."""
    H, W = job.H, job.W
    bands = D.all_bands(H, world)
    assert all(b is not None for b in bands)
    cap_h = max(b.h_local for b in bands)
    torch.cuda.synchronize()
    # every kernel of the test library is loaded before the ranks step (a lazy module load synchronises the context)
    _lib.check(_tlib().stb_test_preload(), test_lib=True)

    def rank_fn(rank, g):
        band = bands[rank]
        up = bands[rank - 1] if rank > 0 else None
        dn = bands[rank + 1] if rank + 1 < world else None
        stream = torch.cuda.Stream(device=DEV)
        with torch.cuda.stream(stream):
            m = NativeVGG(job.wts, 'max', DEV)
            _, p = m.comm_create(rank, world, cap_h, W)
            m.comm_connect_local(g.all_gather_object(p))
            if halo:          # as StyleTransfer._ensure_peer_memory: the neighbours map this rank's workspace
                _, wp = m.alloc_shared_workspace([(band.h_local, W)])
                m.connect_shared_workspaces(g.all_gather_object(wp), False)
            else:
                m.ensure_workspace([(band.h_local, W)])
            m.set_band(True, H, band.own0, band.own_rows)
            ct = m.content_features(D.local_slice(job.content, band))      # from the local content slice, as stylize()
            m.set_targets(band.h_local, W, ct, CONTENT_WEIGHT, job.means, job.srms, STYLE_WEIGHTS, TV_WEIGHT)
            g.barrier()
            m.comm_reset()
            g.barrier()
            m.comm_set_geometry(W, band, up, dn, halo)
            # everything the steps touch exists before they start
            x0 = D.local_slice(job.img, band)
            x, ema = x0.clone(), x0 * (1 - DECAY)
            state = _lbfgs_state(m, band.own_rows, W)
            g_own = torch.empty(3, band.own_rows, W, device=DEV)
            loss = torch.zeros(8, dtype=torch.float32).pin_memory()
            stats = _stats_block(m, band.h_local, W)
            stats_c = torch.empty_like(stats)
            adam = [x0.clone(), D.local_slice(job.exp_avg, band), D.local_slice(job.exp_avg_sq, band), x0 * 0.01]
            after1 = [torch.empty_like(t) for t in adam]
            x_after2 = torch.empty_like(x0)
            stream.synchronize()
            g.barrier()
            # (c) the closure gradient through the banded L-BFGS step
            _lib.check(m.lib.stb_iterate_lbfgs_banded(m.ctx, _lib.ptr(x), _lib.ptr(ema), _lib.ptr(state),
                                                      state.numel(), 1, DECAY, _lib.ptr(loss), _lib.cur_stream()))
            _lbfgs_gradient(state, band.own_rows, W, g_own)
            stats_c.copy_(stats)
            stream.synchronize()
            g.barrier()
            m.comm_reset()
            g.barrier()
            # (d) Adam on the band, restored image, warm state
            for k in range(2):
                xa, ea, eas, emaa = adam
                _lib.check(m.lib.stb_iterate_banded(m.ctx, _lib.ptr(xa), _lib.ptr(ea), _lib.ptr(eas), _lib.ptr(emaa),
                                                    FIRST_STEP + k, LR, 0.9, 0.99, 1e-8, 0.99, None,
                                                    _lib.cur_stream()))
                if k == 0:
                    for dst, src in zip(after1, adam):
                        dst.copy_(src)
            x_after2.copy_(adam[0])
            stream.synchronize()
            g.barrier()            # nobody unmaps a mailbox or workspace a neighbour may still read
            out = dict(m=m, ct=ct.cpu(), g=g_own.cpu(), loss=loss.clone(), stats=stats_c.cpu(),
                       after1=[t[0].cpu() for t in after1], x_after2=x_after2[0].cpu(), x0=x0[0].cpu())
            m.comm_disconnect()
            g.barrier()
            return out

    return bands, _threads(world, rank_fn)


def _host_seam_gradients(job, bands, ranks):
    """(e) An independent restatement of the apron-mode seam sum, in one thread and without communication: per band
    stb_iterate_fwd, the statistics blocks summed on the device in rank order (ThreadGroup.all_reduce_sum),
    stb_iterate_bwd, then the seams added in torch (own, upper neighbour's bottom apron, lower neighbour's top apron).
    Returns the full local gradients [1,3,h_local,W]."""
    W = job.W
    x0s = [D.local_slice(job.img, b) for b in bands]
    views = [_stats_block(r['m'], b.h_local, W) for b, r in zip(bands, ranks)]
    for r, x0 in zip(ranks, x0s):
        r['m'].iterate_fwd(x0)
    acc = views[0].clone()
    for v in views[1:]:
        acc += v
    local = []
    for r, x0, v in zip(ranks, x0s, views):
        v.copy_(acc)
        gl = torch.empty_like(x0)
        r['m'].iterate_bwd(x0, gl, None)
        local.append(gl)
    out = []
    for i, b in enumerate(bands):
        gl = local[i].clone()
        end = b.own0 + b.own_rows
        if i > 0:
            u = bands[i - 1]
            ue = u.own0 + u.own_rows
            gl[:, :, b.own0:b.own0 + D.APRON] += local[i - 1][:, :, ue:ue + u.bottom_apron]
        if i + 1 < len(bands):
            gl[:, :, end - D.APRON:end] += local[i + 1][:, :, :bands[i + 1].top_apron]
        out.append(gl)
    torch.cuda.synchronize()
    return out


def _seam_rows(band):
    """Own rows (band-local own index) within APRON rows of a seam."""
    rows = torch.zeros(band.own_rows, dtype=torch.bool)
    if band.rank > 0:
        rows[:D.APRON] = True
    if band.rank + 1 < band.world:
        rows[band.own_rows - D.APRON:] = True
    return rows


def _row_metric(g, ref):
    """per own row: max |g - ref| / max |ref| over the row's 3 x W values"""
    d = (g.double() - ref.double()).abs().amax(dim=(0, 2))
    return d / ref.double().abs().amax(dim=(0, 2)).clamp_min(1e-30)


@pytest.mark.parametrize('mode', ['apron', 'halo'])
@pytest.mark.parametrize('world,H,W', GEOMS)
def test_tiled_iteration_matches_the_untiled_closure(vgg_weights, world, H, W, mode):
    """(b) statistics, (c) closure gradient and loss terms, (d) Adam on a band, (e, apron mode) the seam sum restated
    on the host -- see the module docstring for R and g_ref."""
    halo = mode == 'halo'
    job = _job(vgg_weights, H, W)
    job.set_band(True)
    bands, ranks = _run_ranks(job, world, halo)
    tiled = ranks[0]['stats'].to(DEV)
    g_ref, loss_ref, stats_own = job.closure(inject=tiled)
    g_ref, stats_own = g_ref.cpu(), stats_own.cpu()
    tiled = tiled.cpu()
    metrics = dict(case=f'{world}x{H}x{W}-{mode}')

    # (b) the statistics cover every own row exactly once
    seg = {name: _rel(tiled[a:b], stats_own[a:b]) for name, a, b in SEGMENTS}
    metrics['stats_rel_max'] = max(seg.values())
    metrics['stats_rel'] = seg

    # (c) closure gradient of the banded L-BFGS step
    far_equal, seam_rows, seam_zone = True, [], []
    for b, r in zip(bands, ranks):
        ref = g_ref[:, b.own_begin:b.own_end]
        zone = _seam_rows(b)
        if halo:
            far_equal = far_equal and torch.equal(r['g'], ref)
        else:
            far_equal = far_equal and torch.equal(r['g'][:, ~zone], ref[:, ~zone])
        if zone.any():
            seam_rows.append(_row_metric(r['g'][:, zone], ref[:, zone]).max().item())
            seam_zone.append(_rel(r['g'][:, zone], ref[:, zone]))
    metrics['grad_rel_max'] = max(_rel(r['g'], g_ref[:, b.own_begin:b.own_end]) for b, r in zip(bands, ranks))
    metrics['seam_row_max'], metrics['seam_zone_max'] = max(seam_rows), max(seam_zone)

    # (d) Adam: the float64 reference fed the gradient of (c), on the own rows
    adam_err = 0.0
    for b, r in zip(bands, ranks):
        own = slice(b.own0, b.own0 + b.own_rows)
        start = (r['x0'], D.local_slice(job.exp_avg, b)[0].cpu(), D.local_slice(job.exp_avg_sq, b)[0].cpu(),
                 r['x0'] * 0.01)
        want = _adam_reference(tuple(t[:, own] for t in start), r['g'], FIRST_STEP)
        for got, w in zip(r['after1'], want):
            adam_err = max(adam_err, (got[:, own].double() - w).abs().max().item() / max(w.abs().max().item(), 1e-30))
    metrics['adam_rel_max'] = adam_err

    # (e) apron mode: the seam sum restated on the host gives the peer-mode gradient
    if not halo:
        host = _host_seam_gradients(job, bands, ranks)
        metrics['host_grad_equal'] = all(torch.equal(gl[0, :, b.own0:b.own0 + b.own_rows].cpu(), r['g'])
                                         for b, r, gl in zip(bands, ranks, host))
    print('METRICS', metrics)

    # (b)
    for name, rel in seg.items():
        assert rel <= STATS_BAR, (name, rel, seg)
    # (c) every rank holds the same reduced statistics and loss terms, which equal R's on the injected statistics
    for rank, r in enumerate(ranks):
        assert torch.equal(r['stats'], tiled), rank
        assert torch.equal(r['loss'], ranks[0]['loss']), rank
    assert torch.equal(ranks[0]['loss'], loss_ref), (ranks[0]['loss'], loss_ref)
    assert far_equal, metrics
    if not halo:
        assert metrics['seam_row_max'] <= SEAM_ROW_BAR and metrics['seam_zone_max'] <= SEAM_ZONE_BAR, metrics
    # (c) each band's content target equals R's on its own rows
    ct_full = job.ct.cpu()
    for b, r in zip(bands, ranks):
        o3 = b.own0 >> 3
        n3 = r['ct'].shape[0] - o3 if b.rank + 1 == world else b.own_rows >> 3
        assert torch.equal(r['ct'][o3:o3 + n3], ct_full[b.own_begin >> 3:(b.own_begin >> 3) + n3]), b.rank
    # (d) the update, the untouched halo rows after the first iteration, the pulled ones after the second
    assert adam_err <= ADAM_BAR, metrics
    for i, (b, r) in enumerate(zip(bands, ranks)):
        end = b.own0 + b.own_rows
        start = (r['x0'], D.local_slice(job.exp_avg, b)[0].cpu(), D.local_slice(job.exp_avg_sq, b)[0].cpu(),
                 r['x0'] * 0.01)
        for got, s in zip(r['after1'], start):
            assert torch.equal(got[:, :b.own0], s[:, :b.own0]) and torch.equal(got[:, end:], s[:, end:]), i
        if i > 0:
            u = ranks[i - 1]
            ue = bands[i - 1].own0 + bands[i - 1].own_rows
            assert torch.equal(r['x_after2'][:, :b.own0], u['after1'][0][:, ue - b.own0:ue]), i
        if i + 1 < world:
            d, db = ranks[i + 1], bands[i + 1]
            assert torch.equal(r['x_after2'][:, end:], d['after1'][0][:, db.own0:db.own0 + b.bottom_apron]), i
    # (e)
    if not halo:
        assert metrics['host_grad_equal'], metrics
