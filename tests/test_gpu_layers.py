"""StyleTransfer.content_layers / style_layers / style_weights over the six taps of the reference model.

Configurations (content, style, layer weights):
  A  content [11], style [1, 6, 11]: a forward truncated at conv 4, whose tap has both roles
  B  content [22], style [1, 6, 11, 20, 22, 29] with six weights: six W2 layers, tap 22 in both roles
  C  content [1, 29], style [20]: two content layers, one at full resolution, a content-only deepest tap (seed kernel)
  D  content [22], style []: no W2 chain
  E  content [22], style [1, 6] with the default five weights: zip() keeps the first two (ST:451)
Tests without the gpu mark run on the CPU: validation, pixel counts and the layer-aware oracle below.
"""
import contextlib
import ctypes
import importlib.util
import io
import threading
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import st_oracle as O

gpu = pytest.mark.gpu

GOLD = Path(__file__).resolve().parent / 'golden'
_spec = importlib.util.spec_from_file_location('make_layers_golden', GOLD / 'make_layers_golden.py')
MLG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MLG)

DEFAULT_W = [w / 341 for w in (256, 64, 16, 4, 1)]
SIX_W = [w / 345 for w in (256, 64, 16, 4, 4, 1)]
CONFIGS = {
    'A': ([11], [1, 6, 11], DEFAULT_W),
    'B': ([22], [1, 6, 11, 20, 22, 29], SIX_W),
    'C': ([1, 29], [20], DEFAULT_W),
    'D': ([22], [], DEFAULT_W),
    'E': ([22], [1, 6], DEFAULT_W),
}
TERM_RTOL = {False: 5e-3, True: 2e-3}   # as tests/test_gpu_iterate.py
# Bars against the oracle (fp32: False, modelling the bf16 storage points: True), as tests/test_gpu_iterate.py.
TOTAL_RTOL = {False: 1e-3, True: 1e-3}
COS = {False: 0.995, True: 0.9995}
# Content MSE: a small difference of two independently rounded bf16 feature maps.  At tap 29 these images have 1 to 35
# pixels of it, and the MSE is ~1e-4 (measured on an H100: 6.6e-2 from the fp32 oracle, 1.5e-2 from the bf16 model).
CONTENT_RTOL = {29: {False: 1e-1, True: 3e-2}}
CONTENT_RTOL_OTHER = {False: 3e-2, True: 1e-2}
# C's one style term is tap 20 with weight 256/341; the default table gives that tap 4/341, which hides how closely the
# W2 engine follows the oracle there.  Measured on an H100 (the same with the default table and its weights moved to put
# 256/341 on tap 20, so these follow the weight, not the layer table):
#  * the tap-20 W2 term on the bf16-stored features is 1.4e-3 from its value on fp32 features at these sizes (fp32 oracle
#    against the oracle modelling the storage points): the total is held to 1e-3 against the latter, 2e-3 against fp32;
#  * the gradient's cosine is 0.978-0.998 to the fp32 oracle and 0.991-0.9994 to the bf16 model at 48x64 .. 72x72,
#    with or without either content layer (content [1, 29] with style [1] or none: >= 0.9999).  Forming the mean term of
#    the tap gradient from the bf16 Gs / N of the tap GEMM instead of the fp32 Gs changed it by less than 1e-5, so it is
#    the W2 backward on that covariance, not the rounding of the tap GEMM's operand;
#  * the loss at the native iterate of a 32 -> 64 run is up to 2.1e-3 from the fp32 oracle; a tiled run's loss is up to
#    5.4e-4 and its image 0.62 / 255 from the untiled one (the full-resolution content SSE summed per band).
TOTAL_RTOL_C = {False: 2e-3, True: 1e-3}
COS_C = {False: 0.97, True: 0.985}
ITERATE_RTOL_C = 3e-3
TILED_DRIFT_C = 1e-3
TILED_IMG_C = 1.0


# ------------------------------------------------------------------------------------- the oracle over layer lists
# oracle/st_oracle.py evaluates the reference's default layers; these restate ST:365-455 for any lists on its
# building blocks (vgg_forward / vgg_backward take any taps).
def oracle_targets(content, style, wts, pooling, content_layers, style_layers, sim=False):
    """Targets of ST:425-450 for one content and one style tensor: (content targets, [StyleTarget])."""
    a_c = O.vgg_forward(content, wts, pooling, max(content_layers), sim)
    style_t = []
    if style_layers:
        a_s = O.vgg_forward(style, wts, pooling, max(style_layers), sim)
        style_t = [O.StyleTarget.build(*O.style_stats(a_s[t])) for t in style_layers]
    return [a_c[t] for t in content_layers], style_t


def oracle_loss_and_grad(image, wts, targets, pooling, content_layers, style_layers, layer_weights,
                         content_weight=0.015, tv_weight=2.0, sim=False, detail=None):
    """closure() of ST:472-476 over the given lists: terms in SumLoss order (content, style, TV; ST:455)."""
    ctargets, style_t = targets
    acts = O.vgg_forward(image, wts, pooling, 29, sim)   # the closure's model holds all six taps (ST:324)
    cw = content_weight / len(content_layers)
    terms, tap_grads = [], {}
    for t, target in zip(content_layers, ctargets):
        cl, cg = O.content_loss_and_grad(acts[t], target)
        terms.append(cl * cw)
        tap_grads[t] = cg * cw   # added in fp32 inside the dgrad epilogue
    for t, lw, tgt in zip(style_layers, layer_weights, style_t):
        sl, sg, _ = O.w2_loss_and_grad(acts[t], tgt)
        terms.append(sl * lw)
        sg = O._q(sg * lw, sim) if t not in content_layers else sg * lw
        tap_grads[t] = tap_grads[t] + sg if t in tap_grads else sg
    tvl, tvg = O.tv_loss_and_grad(image)
    terms.append(tvl * tv_weight)
    g = O.vgg_backward(tap_grads, acts, wts, pooling, sim) + tvg * tv_weight
    loss = terms[0]
    for t in terms[1:]:
        loss = loss + t
    if detail is not None:
        detail['terms'] = [float(t) for t in terms]
    return loss, g


def oracle_scale_targets(content_pil, style_pil, scale, wts, content_layers, style_layers):
    from PIL import Image
    cw, ch = O.size_to_fit(content_pil.size, scale, scale_up=True)
    sw, sh = O.size_to_fit(style_pil.size, scale)
    content = O.to_tensor(content_pil.resize((cw, ch), Image.BICUBIC))
    style = O.to_tensor(style_pil.resize((sw, sh), Image.BICUBIC))
    return oracle_targets(content, style, wts, 'max', content_layers, style_layers), (cw, ch)


def oracle_stylize_trace(content_pil, style_pil, wts, content_layers, style_layers, layer_weights, min_scale,
                         end_scale, initial_iterations, iterations=500):
    """Loss trace and result of ST:349-499 (init='content', Adam, one style image, max pooling) over the given
    lists."""
    from PIL import Image
    scales = O.gen_scales(min(min_scale, end_scale), end_scale)
    cw, ch = O.size_to_fit(content_pil.size, scales[0], scale_up=True)
    image = O.to_tensor(content_pil.resize((cw, ch), Image.BICUBIC))
    st, trace = None, []
    for si, scale in enumerate(scales):
        tg, (cw, ch) = oracle_scale_targets(content_pil, style_pil, scale, wts, content_layers, style_layers)
        image = O._interp(image, (ch, cw), 'bicubic').clamp(0, 1)
        new = O.IterState.fresh(image)
        if st is not None:
            new.exp_avg = O._interp(st.exp_avg, (ch, cw), 'bicubic')
            new.exp_avg_sq = O._interp(st.exp_avg_sq, (ch, cw), 'bilinear').relu_()
            new.step = st.step
        st = new
        for _ in range(initial_iterations if si == 0 else iterations):
            loss, g = oracle_loss_and_grad(st.image, wts, tg, 'max', content_layers, style_layers, layer_weights)
            trace.append(float(loss))
            st.step += 1
            st.exp_avg = st.exp_avg + (g - st.exp_avg) * (1 - 0.9)
            st.exp_avg_sq = st.exp_avg_sq * 0.99 + (1 - 0.99) * g * g
            denom = st.exp_avg_sq.sqrt() / (1 - 0.99 ** st.step) ** 0.5 + 1e-8
            st.image = (st.image - (0.02 / (1 - 0.9 ** st.step)) * st.exp_avg / denom).clamp(0, 1)
            st.ema_update(0.99)
        image = st.ema_get()
        st.image = image
    return trace, st.ema_get()[0].clamp(0, 1)


def _pkg():
    import style_transfer_b200 as stb
    return stb


# ---------------------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize('content,style,exc', [
    ([22], [1, 6, 3], KeyError), ([8], [1], KeyError), ([22, 22], [1], ValueError), ([22], [6, 1, 6], ValueError),
    ([22], [13], KeyError)])
def test_invalid_layers_raise_before_any_device_call(content, style, exc):
    from style_transfer_b200.style_transfer import check_layers
    with pytest.raises(exc):
        check_layers(content, style)


def test_valid_layers_pass_validation():
    from style_transfer_b200.style_transfer import check_layers
    for content, style, _ in CONFIGS.values():
        check_layers(content, style)
    check_layers([22, 11], [29, 1])   # any order, a tap in both lists


def test_tap_pixel_counts_follow_the_taps():
    from style_transfer_b200 import distributed as D
    assert D.tap_pixel_counts(181, 136, [22, 1, 29]) == [22 * 17, 181 * 136, 11 * 8]
    assert D.tap_pixel_counts(181, 136) == D.tap_pixel_counts(181, 136, [1, 6, 11, 20, 29])


def test_oracle_default_lists_equal_the_default_oracle(vgg_weights):
    """With the default lists the layer-aware closure is the oracle's default closure, bit for bit; the Adam trace
    restated above is the oracle's stylize()."""
    content, style = O.synth_image(1, 16, 40, 32), O.synth_image(2, 32, 36, 28)
    tg, _ = O.make_targets(content, [style], [1.0], 40, vgg_weights, 'max', 0.015, 2.0)
    tg2, _ = oracle_scale_targets(content, style, 40, vgg_weights, [22], [1, 6, 11, 20, 29])
    img = O.to_tensor(content.resize((40, 32)))
    l1, g1 = O.loss_and_grad(img, vgg_weights, tg)
    l2, g2 = oracle_loss_and_grad(img, vgg_weights, tg2, 'max', [22], [1, 6, 11, 20, 29], DEFAULT_W)
    assert float(l1) == float(l2)
    assert torch.equal(g1, g2)
    kw = dict(min_scale=24, end_scale=34, iterations=2, initial_iterations=2)
    trace = []
    O.stylize(content, [style], vgg_weights, callback=lambda si, i, loss, s: trace.append(loss), **kw)
    assert trace == oracle_stylize_trace(content, style, vgg_weights, [22], [1, 6, 11, 20, 29], DEFAULT_W, **kw)[0]


@pytest.mark.parametrize('name', list(MLG.CONFIGS))
def test_oracle_reproduces_the_reference_goldens(vgg_weights, name):
    """The layer-aware closure and stylize() above against the unmodified reference with the attributes set
    (tests/golden/make_layers_golden.py), at the bars of test_oracle_golden.py."""
    gold = np.load(GOLD / f'layers_{name}.npz')
    content_layers, style_layers, lw = MLG.CONFIGS[name]
    eff_style, eff_w = style_layers[:len(lw)], lw[:len(style_layers)]
    content, style = O.synth_image(*MLG.CONTENT), O.synth_image(*MLG.STYLE)
    for prefix, kw in (('single', MLG.SINGLE), ('pyr', MLG.PYRAMID)):
        trace, out = oracle_stylize_trace(content, style, vgg_weights, content_layers, eff_style, eff_w, **kw)
        np.testing.assert_allclose(trace, gold[f'{prefix}_losses'], rtol=2e-4)
        diff = np.abs(out.numpy() - gold[f'{prefix}_final'])
        assert diff.mean() < 2e-4 and np.quantile(diff, 0.999) < 2e-2
    tg, _ = oracle_scale_targets(content, style, 64, vgg_weights, content_layers, eff_style)
    det = {}
    loss, grad = oracle_loss_and_grad(torch.from_numpy(gold['image']), vgg_weights, tg, 'max', content_layers,
                                      eff_style, eff_w, detail=det)
    np.testing.assert_allclose(det['terms'], gold['terms'], rtol=3e-4)
    np.testing.assert_allclose(float(loss), float(gold['total']), rtol=1e-4)
    assert np.linalg.norm(grad.numpy() - gold['grad']) / np.linalg.norm(gold['grad']) < 2e-3


# ---------------------------------------------------------------------------------------------------------- GPU
def _targets(st, content_layers, style_layers, lw, cimg, simg, H, W):
    """Set the layer table and the targets through the list calls, as stylize() does."""
    m = st.model
    m.set_layers(content_layers, style_layers)
    m.ensure_workspace([(H, W), tuple(simg.shape[2:])])
    cts = m.content_features_list(cimg.cuda())
    means, srms = m.style_stats(simg.cuda())
    m.set_targets_list(H, W, cts, [0.015 / len(content_layers)] * len(content_layers), means, srms,
                       lw[:len(style_layers)], 2.0)
    return cts, means, srms


CASES = [(n, H, W, p) for n in CONFIGS for (H, W, p) in
         [(48, 64, 'max'), (56, 80, 'average'), (72, 72, 'l2'), (45, 34, 'max'), (16, 16, 'max')]]
CASES += [('A', 512, 512, 'max'), ('B', 512, 512, 'max')]


@gpu
@pytest.mark.parametrize('name,H,W,pooling', CASES)
def test_layers_loss_and_gradient(vgg_weights, name, H, W, pooling):
    import gpu_util as G
    content_layers, style_layers, lw = CONFIGS[name]
    st = G.make_st(pooling, vgg_weights)
    cimg = O.to_tensor(O.synth_image(1, 16, W, H))
    simg = O.to_tensor(O.synth_image(2, 32, max(W - 8, 16), max(H - 4, 16)))
    cts, means, srms = _targets(st, content_layers, style_layers, lw, cimg, simg, H, W)
    torch.cuda.synchronize()
    acts_c = O.vgg_forward(cimg, vgg_weights, pooling, 29)
    for t, ct in zip(content_layers, cts):
        assert G.rel_err(G.nchw(ct), acts_c[t]) < 3e-2
    acts_s = O.vgg_forward(simg, vgg_weights, pooling, 29)
    for li, t in enumerate(style_layers):
        om, osrm = O.style_stats(acts_s[t])
        assert G.rel_err(means[li], om) < 1e-2
        assert G.rel_err(srms[li], osrm) < 1e-2
    torch.manual_seed(0)
    img = (cimg + 0.05 * torch.randn_like(cimg)).clamp(0, 1)
    st.image = img.to(G.DEV).contiguous()
    terms, grad = st.loss_and_grad()
    nc, ns = len(content_layers), len(style_layers)
    assert terms.numel() == 2 + nc + ns
    total_rtol = TOTAL_RTOL_C if name == 'C' else TOTAL_RTOL
    # the 512^2 cases against the fp32 oracle only (the CPU oracle is the slow part of this test)
    for sim in (False,) + ((True,) if H < 512 else ()):
        tg = oracle_targets(cimg, simg, vgg_weights, pooling, content_layers, style_layers, sim)
        det = {}
        ol, og = oracle_loss_and_grad(img, vgg_weights, tg, pooling, content_layers, style_layers, lw, sim=sim,
                                      detail=det)
        print(name, H, W, pooling, sim, 'native', terms.tolist(), 'oracle', float(ol), det['terms'])
        assert abs(terms[0].item() - float(ol)) / float(ol) < total_rtol[sim]
        np.testing.assert_allclose(terms[1 + nc:1 + nc + ns + 1].numpy(), det['terms'][nc:], rtol=TERM_RTOL[sim],
                                   atol=2e-6)
        # content MSEs: a small difference of two independently rounded bf16 feature maps (see test_gpu_iterate.py)
        for k, t in enumerate(content_layers):
            np.testing.assert_allclose(terms[1 + k].item(), det['terms'][k],
                                       rtol=CONTENT_RTOL.get(t, CONTENT_RTOL_OTHER)[sim], atol=2e-6)
        cos = F.cosine_similarity(grad.cpu().flatten(), og.flatten(), dim=0).item()
        print(name, H, W, pooling, sim, 'gradient cosine', cos)
        assert cos > (COS_C if name == 'C' else COS)[sim]


@gpu
def test_set_layers_rejects_bad_tables(vgg_weights):
    import gpu_util as G
    st = G.make_st('max', vgg_weights)
    lib, ctx = st.model.lib, st.model.ctx

    def call(content, style):
        ca = (ctypes.c_int * max(len(content), 1))(*content)
        sa = (ctypes.c_int * max(len(style), 1))(*style)
        return lib.stb_set_layers(ctx, len(content), ca, len(style), sa)

    assert call([22], [1, 6, 11, 20, 29]) == 0
    for content, style in (([], [1]), ([22], [1, 3]), ([22, 22], [1]), ([22], [1, 1]), ([23], [1]),
                           ([22], [1, 6, 11, 20, 22, 29, 1])):
        assert call(content, style) == -1, (content, style)
    # the default calls are refused under another table: there is one code path
    assert call([11], [1]) == 0
    n = ctypes.c_size_t()
    assert lib.stb_workspace_bytes(ctx, 64, 64, ctypes.byref(n)) == 0
    with pytest.raises(RuntimeError):
        st.model.content_features(torch.zeros(1, 3, 64, 64, device=G.DEV))


def _iterate_adam(st, cimg, simg, set_default_layers, its=6, lbfgs=False):
    """Default targets through the default calls, `its` graphed iterations; returns image, EMA and loss terms."""
    m = st.model
    H, W = cimg.shape[2:]
    if set_default_layers:
        m.set_layers([22], [1, 6, 11, 20, 29])
    m.ensure_workspace([(H, W), tuple(simg.shape[2:])])
    with torch.cuda.stream(st._stream):
        ct = m.content_features(cimg.cuda())
        means, srms = m.style_stats(simg.cuda())
        m.set_targets(H, W, ct, 0.015, means, srms, st.style_weights, 2.0)
        st.image = cimg.cuda().clone()
        st.average = _pkg().style_transfer.EMA(st.image, 0.99)
        terms = []
        if lbfgs:
            state = st._lbfgs_state(H, W)
            for step in range(1, its + 1):
                st._iterate_lbfgs(state, step, 0.99)
                terms.append(st._wait_loss(step))
        else:
            ea, eas = torch.zeros_like(st.image), torch.zeros_like(st.image)
            for step in range(1, its + 1):
                st._iterate(ea, eas, step, 0.02, 0.99, True)
                terms.append(st._wait_loss(step))
        st._stream.synchronize()
    return st.image.cpu(), st.average.value.cpu(), torch.stack(terms), m.launch_count()


@gpu
@pytest.mark.parametrize('lbfgs', [False, True])
def test_explicit_default_table_is_bit_identical(vgg_weights, lbfgs):
    import gpu_util as G
    cimg = O.to_tensor(O.synth_image(1, 16, 96, 80))
    simg = O.to_tensor(O.synth_image(2, 32, 88, 72))
    a = _iterate_adam(G.make_st('max', vgg_weights), cimg, simg, False, lbfgs=lbfgs)
    b = _iterate_adam(G.make_st('max', vgg_weights), cimg, simg, True, lbfgs=lbfgs)
    for x, y in zip(a[:3], b[:3]):
        assert torch.equal(x, y)
    assert a[3][0] > 0 and a[3][2] == b[3][2]   # graph replays, same kernel nodes


def _banded_phases(st, cimg, simg, set_default_layers, its=4):
    """The two halves of a band's closure (stb_iterate_fwd / stb_iterate_bwd) on a band that owns every row: gradient
    and loss terms of `its` graphed closures."""
    m = st.model
    H, W = cimg.shape[2:]
    if set_default_layers:
        m.set_layers([22], [1, 6, 11, 20, 29])
    m.ensure_workspace([(H, W), tuple(simg.shape[2:])])
    with torch.cuda.stream(st._stream):
        ct = m.content_features(cimg.cuda())
        means, srms = m.style_stats(simg.cuda())
        m.set_band(True, H, 0, H)
        m.set_targets(H, W, ct, 0.015, means, srms, st.style_weights, 2.0)
        img = cimg.cuda().clone()
        grad = torch.empty_like(img)
        out = []
        for _ in range(its):
            m.iterate_fwd(img)
            m.iterate_bwd(img, grad, st._loss_host)
            st._stream.synchronize()
            out.append((grad.cpu(), st._loss_host.clone()))
    return out, m.launch_count()[2]


@gpu
def test_explicit_default_table_is_bit_identical_on_the_band_phases(vgg_weights):
    import gpu_util as G
    cimg = O.to_tensor(O.synth_image(1, 16, 96, 80))
    simg = O.to_tensor(O.synth_image(2, 32, 88, 72))
    a, per_a = _banded_phases(G.make_st('max', vgg_weights), cimg, simg, False)
    b, per_b = _banded_phases(G.make_st('max', vgg_weights), cimg, simg, True)
    for (ga, la), (gb, lb) in zip(a, b):
        assert torch.equal(ga, gb) and torch.equal(la, lb)
    assert per_a[1] > 0 and per_a == per_b   # the fwd / bwd phases replayed as graphs, with the same kernel nodes


@gpu
@pytest.mark.parametrize('devices', [1, 2])
@pytest.mark.parametrize('content,style,exc', [([], [1], ZeroDivisionError), ([22], [1, 3], KeyError),
                                               ([22, 22], [1], ValueError), ([22], [6, 1, 6], ValueError)])
def test_stylize_rejects_bad_layers_before_any_device_work(vgg_weights, devices, content, style, exc):
    """Through the public call, with one device and with two (where rank 1 validates its copy on its own thread):
    the error comes before any iteration, and the contexts keep their layer tables."""
    stb = _pkg()
    st = stb.StyleTransfer(devices=['cuda:0'] * devices, pooling='max', vgg_weights=vgg_weights)
    st.content_layers, st.style_layers = content, style
    calls = []
    with contextlib.redirect_stdout(io.StringIO()), pytest.raises(exc):
        st.stylize(O.synth_image(1, 16, 64, 48), [O.synth_image(2, 32, 56, 40)], min_scale=64, end_scale=64,
                   initial_iterations=2, callback=calls.append)
    assert calls == [] and st.image is None
    for obj in [st] + ([st._peer] if devices == 2 else []):
        assert obj.model.content_layers == [22] and obj.model.style_layers == [1, 6, 11, 20, 29]


@gpu
def test_truncated_table_launches_fewer_kernels(vgg_weights):
    import gpu_util as G
    cimg = O.to_tensor(O.synth_image(1, 16, 96, 80))
    simg = O.to_tensor(O.synth_image(2, 32, 88, 72))
    _, _, _, (_, _, per_default) = _iterate_adam(G.make_st('max', vgg_weights), cimg, simg, False)
    st = G.make_st('max', vgg_weights)
    m = st.model
    H, W = 80, 96
    content_layers, style_layers, lw = CONFIGS['A']
    with torch.cuda.stream(st._stream):
        _targets(st, content_layers, style_layers, lw, O.to_tensor(O.synth_image(1, 16, W, H)), simg, H, W)
        st.image = cimg.cuda().clone()
        st.average = _pkg().style_transfer.EMA(st.image, 0.99)
        ea, eas = torch.zeros_like(st.image), torch.zeros_like(st.image)
        for step in range(1, 5):
            st._iterate(ea, eas, step, 0.02, 0.99, True)
            assert st._wait_loss(step).numel() == 6
        st._stream.synchronize()
    per_a = m.launch_count()[2]
    print('kernel nodes per iteration graph: default', per_default[0], 'A', per_a[0])
    # config A stops at conv 4: 8 forward convs and 8 dgrad convs fewer, and two W2 layers fewer
    assert 0 < per_a[0] <= per_default[0] - 16
    # the workspace holds activations through conv 4 only
    out = torch.empty(1 << 20, dtype=torch.uint8, device=G.DEV)
    with pytest.raises(ValueError):
        _pkg()._lib.check(m.lib.stb_debug_activation(m.ctx, H, W, 5, _pkg()._lib.ptr(out), out.numel(),
                                                     _pkg()._lib.cur_stream()))


def _stylize(st, content, style, name, kw):
    content_layers, style_layers, lw = CONFIGS[name]
    st.content_layers, st.style_layers, st.style_weights = list(content_layers), list(style_layers), list(lw)
    recs = []
    with contextlib.redirect_stdout(io.StringIO()):
        img = st.stylize(content, [style], callback=lambda it: recs.append(
            (it.loss, it.w, it.h, it.i, st.image.detach().cpu().clone(), st.last_loss_terms.clone())), **kw)
    return recs, np.asarray(img, dtype=np.float32)


@gpu
@pytest.mark.parametrize('run', ['single', 'pyr'])
@pytest.mark.parametrize('name', ['A', 'B', 'C'])
def test_stylize_matches_the_reference_goldens(vgg_weights, name, run):
    """stylize() with the attributes set after construction, against the unmodified reference's run: the first loss
    and the trace; then every iteration's loss against the layer-aware oracle (pinned to the same goldens on the CPU)
    evaluated at the native iterate, as test_gpu_iterate.py does for the default layers."""
    import gpu_util as G
    gold = np.load(GOLD / f'layers_{name}.npz')
    content_layers, style_layers, lw = MLG.CONFIGS[name]
    eff_style, eff_w = style_layers[:len(lw)], lw[:len(style_layers)]
    content, style = O.synth_image(*MLG.CONTENT), O.synth_image(*MLG.STYLE)
    kw = MLG.SINGLE if run == 'single' else MLG.PYRAMID
    recs, _ = _stylize(G.make_st('max', vgg_weights), content, style, name, dict(kw))
    for r in recs:
        assert r[5].numel() == 2 + len(content_layers) + len(eff_style)
        assert r[5][0].item() == r[0]
    native, ref = np.array([r[0] for r in recs]), gold[f'{run}_losses']
    print(name, run, 'vs reference', (np.abs(native - ref) / ref).tolist())
    assert len(native) == len(ref)
    assert abs(native[0] - ref[0]) / ref[0] < 1e-3
    np.testing.assert_allclose(native, ref, rtol=5e-3)
    scales = O.gen_scales(kw['min_scale'], kw['end_scale'])
    tgs, prev, rel = {}, None, []
    for loss, w, h, i, img, _ in recs:
        if (w, h) not in tgs:
            scale = next(s for s in scales if O.size_to_fit(content.size, s, scale_up=True) == (w, h))
            tgs[(w, h)] = oracle_scale_targets(content, style, scale, vgg_weights, content_layers, eff_style)[0]
        if i > 1:
            ol, _ = oracle_loss_and_grad(prev, vgg_weights, tgs[(w, h)], 'max', content_layers, eff_style, eff_w)
            rel.append(abs(loss - float(ol)) / float(ol))
        prev = img
    print(name, run, 'at the native iterate', rel)
    assert max(rel) < (ITERATE_RTOL_C if name == 'C' else 1e-3), rel


def _run_tiled(world, content, style, wts, name, kw, optimizer):
    stb = _pkg()
    from style_transfer_b200 import distributed as D
    shared = D.ThreadGroup.Shared(world)
    results, errors = [None] * world, []

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts,
                                   distributed=D.ThreadGroup(shared, rank))
            recs, img = _stylize(st, content, style, name, dict(kw, optimizer=optimizer))
            results[rank] = (np.array([r[0] for r in recs]), img, 'halo' if st._halo_now else 'apron')
        except BaseException as e:  # noqa: BLE001 -- report and release the other ranks
            errors.append((rank, repr(e)))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    assert not errors, errors
    return results


@gpu
@pytest.mark.parametrize('optimizer', ['adam', 'lbfgs'])
@pytest.mark.parametrize('tile', ['halo', 'apron'])
@pytest.mark.parametrize('name,world', [('A', 2), ('C', 3)])
def test_tiled_layers_equal_untiled(vgg_weights, monkeypatch, name, world, tile, optimizer):
    import gpu_util as G
    monkeypatch.setenv('STB_TILE', tile)
    monkeypatch.setenv('STB_COMM_TIMEOUT_S', '20')
    W, H = 256, 384
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
    kw = dict(min_scale=H, end_scale=H, initial_iterations=4)
    tiled = _run_tiled(world, content, style, vgg_weights, name, kw, optimizer)
    recs, img_s = _stylize(G.make_st('max', vgg_weights), content, style, name, dict(kw, optimizer=optimizer))
    tr_s = np.array([r[0] for r in recs])
    for tr, img, mode in tiled:
        assert mode == tile
        drift = np.abs(tr - tr_s) / np.abs(tr_s)
        print(name, world, tile, optimizer, 'loss drift tiled vs untiled', drift.tolist())
        if optimizer == 'adam':   # the bars of test_gpu_tiled.py / test_gpu_lbfgs_tiled.py
            assert drift.max() < (TILED_DRIFT_C if name == 'C' else 5e-4)
            assert np.abs(img - img_s).mean() < (TILED_IMG_C if name == 'C' else 0.5)
        else:
            assert drift[:2].max() <= 5e-4 and drift.max() <= 1e-2
            assert np.abs(img - img_s).mean() < 2.0
    for tr, img, _ in tiled[1:]:
        np.testing.assert_array_equal(img, tiled[0][1])


@gpu
def test_two_device_object_copies_the_layers_to_rank_1(vgg_weights, monkeypatch):
    """StyleTransfer(devices=['cuda:0', 'cuda:0']) with A set on rank 0 only: both ranks run A."""
    import gpu_util as G
    stb = _pkg()
    W, H = 256, 384
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
    kw = dict(min_scale=H, end_scale=H, initial_iterations=4)
    st = stb.StyleTransfer(devices=['cuda:0', 'cuda:0'], pooling='max', vgg_weights=vgg_weights)
    recs, img = _stylize(st, content, style, 'A', kw)
    assert st._peer.model.content_layers == [11] and st._peer.model.style_layers == [1, 6, 11]
    recs_s, img_s = _stylize(G.make_st('max', vgg_weights), content, style, 'A', kw)
    np.testing.assert_allclose([r[0] for r in recs], [r[0] for r in recs_s], rtol=5e-4)
    assert np.abs(img - img_s).mean() < 0.5
