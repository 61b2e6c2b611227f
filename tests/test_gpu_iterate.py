"""-m gpu: the whole hot path through the public class / C-ABI against the oracle and the reference goldens.

Bar (BASELINE.json north_star): loss within 1e-3 relative of the reference's own PyTorch path on identical
inputs/seeds.  The CUDA path stores activations in bf16 (fp32 accumulate); the oracle's `sim_bf16` mode models those
rounding points, so the comparison against it is much tighter (3e-4) and isolates real bugs from quantisation.
"""
import importlib.util
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import st_oracle as O  # noqa: E402

TERM_RTOL = {False: 5e-3, True: 2e-3}   # vs the fp32 oracle / vs the oracle that models the bf16 storage points

GOLD = Path(__file__).resolve().parent / 'golden'
_spec = importlib.util.spec_from_file_location('make_golden', GOLD / 'make_golden.py')
MG = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(MG)


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    return g


@pytest.mark.parametrize('H,W,pooling', [(48, 64, 'max'), (56, 80, 'average'), (72, 72, 'l2'), (45, 34, 'max'),
                                         (16, 16, 'max')])
def test_targets_loss_and_gradient(G, vgg_weights, H, W, pooling):
    st = G.make_st(pooling, vgg_weights)
    cimg = O.to_tensor(O.synth_image(1, 16, W, H))
    simg = O.to_tensor(O.synth_image(2, 32, max(W - 8, 16), max(H - 4, 16)))
    m = st.model
    m.ensure_workspace([(H, W), tuple(simg.shape[2:])])
    ct = m.content_features(cimg.to(G.DEV))
    means, srms = m.style_stats(simg.to(G.DEV))
    torch.cuda.synchronize()
    acts_s = O.vgg_forward(simg, vgg_weights, pooling, 29)
    for li, layer in enumerate(O.STYLE_LAYERS):
        om, osrm = O.style_stats(acts_s[layer])
        assert G.rel_err(means[li], om) < 1e-2
        assert G.rel_err(srms[li], osrm) < 1e-2
    acts_c = O.vgg_forward(cimg, vgg_weights, pooling, 22)
    assert G.rel_err(G.nchw(ct), acts_c[22]) < 3e-2
    m.set_targets(H, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    torch.manual_seed(0)
    img = (cimg + 0.05 * torch.randn_like(cimg)).clamp(0, 1)
    st.image = img.to(G.DEV).contiguous()
    terms, grad = st.loss_and_grad()
    for sim, tol_loss, tol_cos in ((False, 1e-3, 0.995), (True, 3e-4, 0.9995)):
        a_s = O.vgg_forward(simg, vgg_weights, pooling, 29, sim)
        a_c = O.vgg_forward(cimg, vgg_weights, pooling, 22, sim)
        tg = O.ScaleTargets(a_c[22], [O.StyleTarget.build(*O.style_stats(a_s[layer])) for layer in O.STYLE_LAYERS],
                            0.015, 2.0)
        det = {}
        ol, og = O.loss_and_grad(img, vgg_weights, tg, pooling, sim_bf16=sim, detail=det)
        assert abs(terms[0].item() - float(ol)) / float(ol) < tol_loss
        # every term on its own (a 2 % error of one style layer must not hide inside a 1e-3 total): the W2 terms are
        # fp32-accurate on bf16 features, the content MSE is a small difference of bf16 features
        np.testing.assert_allclose(terms[2:8].numpy(), det['terms'][1:], rtol=TERM_RTOL[sim], atol=2e-6)
        # the content MSE of these tiny cases is ~4e-4: a small difference of two independently rounded bf16 feature
        # maps, whose rounding noise adds its variance to it (1-2.5 % here; see tests/test_gpu_parity_big.py)
        np.testing.assert_allclose(terms[1].item(), det['terms'][0], rtol=3e-2 if not sim else 1e-2, atol=2e-6)
        cos = F.cosine_similarity(grad.cpu().flatten(), og.flatten(), dim=0).item()
        assert cos > tol_cos


def test_loss_parity_at_512(G, vgg_weights):
    """The loss bar must hold where the accumulation chains are long: at 512^2 every style term's Gram runs over
    262 144 pixels and the ill-conditioned (eps = 1e-4) covariances amplify any bias of the tensor-core accumulation
    (a mirrored / long-chain W2 engine was -1.3e-3 here while passing every small case)."""
    H = W = 512
    st = G.make_st('max', vgg_weights)
    cimg = O.to_tensor(O.synth_image(1, 16, W, H))
    simg = O.to_tensor(O.synth_image(2, 32, W - 8, H - 4))
    m = st.model
    m.ensure_workspace([(H, W), tuple(simg.shape[2:])])
    ct = m.content_features(cimg.to(G.DEV))
    means, srms = m.style_stats(simg.to(G.DEV))
    m.set_targets(H, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    torch.manual_seed(0)
    img = (cimg + 0.05 * torch.randn_like(cimg)).clamp(0, 1)
    st.image = img.to(G.DEV).contiguous()
    terms, _ = st.loss_and_grad()
    a_s = O.vgg_forward(simg, vgg_weights, 'max', 29)
    a_c = O.vgg_forward(cimg, vgg_weights, 'max', 22)
    tg = O.ScaleTargets(a_c[22], [O.StyleTarget.build(*O.style_stats(a_s[layer])) for layer in O.STYLE_LAYERS],
                        0.015, 2.0)
    det = {}
    ol, _ = O.loss_and_grad(img, vgg_weights, tg, 'max', detail=det)
    assert abs(terms[0].item() - float(ol)) / float(ol) < 1e-3   # north_star bar; measured 1.5e-4
    # the two large style terms (relu1_1, relu2_1 = 2/3 of the loss) individually
    np.testing.assert_allclose(terms[2:4].numpy(), det['terms'][1:3], rtol=1e-3)


@pytest.mark.parametrize('name', ['max_64x48_single', 'avg_80x56_two_styles', 'l2_72x72_single', 'max_pyramid_32_64',
                                  'max_128_noise_tv', 'max_pyramid_128_512'])
def test_stylize_matches_reference_golden(G, vgg_weights, name):
    """Public API end to end (pyramid, Adam warm start with carried step, EMA) vs the UNMODIFIED reference's trace."""
    gold = np.load(GOLD / f'{name}.npz')
    content, styles, pooling, kw = MG.build_case(name)
    st = G.make_st(pooling, vgg_weights)
    trace = []
    out = st.stylize(content, styles, callback=lambda it: trace.append((it.loss, it.w, it.h, it.i)), **kw)
    assert len(trace) == len(gold['losses'])
    np.testing.assert_array_equal(np.array([t[1:] for t in trace]), gold['sizes'][:, :3])
    losses = np.array([t[0] for t in trace])
    # first iteration of the first scale: identical inputs -> the 1e-3 bar of the north star
    assert abs(losses[0] - gold['losses'][0]) / gold['losses'][0] < 1e-3
    # later iterations: trajectories of a bf16 and an fp32 optimiser drift slowly (SURVEY.md section 7.2); the bar per
    # iteration is held with re-synchronised state in test_every_iteration_matches_the_oracle_at_the_native_iterate
    np.testing.assert_allclose(losses, gold['losses'], rtol=5e-3)
    # same uint8 truncation as get_image() on both sides; the residual is trajectory drift of a sign-like optimiser
    img = np.asarray(out, dtype=np.float32).transpose(2, 0, 1) / 255
    fin = gold['final_image']
    gold_q = fin.astype(np.float32) / 255 if fin.dtype == np.uint8 else np.floor(fin * 255) / 255
    # 60 sign-like Adam steps (the 512 pyramid) let a bf16 and an fp32 run end ~2.5 uint8 levels apart per pixel; the
    # short cases stay within 1.5 levels
    assert np.abs(img - gold_q).mean() < (6e-3 if len(losses) <= 10 else 1.5e-2)


def test_iterate_state_update_matches_oracle(G, vgg_weights):
    """One stb_iterate: Adam moments, clamped image and EMA vs the oracle fed with the native gradient's oracle twin."""
    H, W = 48, 64
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, 56, 40)
    st = G.make_st('max', vgg_weights)
    tr = []
    st.stylize(content, [style], min_scale=64, end_scale=64, initial_iterations=1, callback=lambda it: tr.append(it.loss))
    tg, _ = O.make_targets(content, [style], [1.0], 64, vgg_weights, 'max', 0.015, 2.0, sim_bf16=True)
    s0 = O.IterState.fresh(O.to_tensor(content))
    loss = O.iterate(s0, vgg_weights, tg, 'max', sim_bf16=True)
    assert abs(tr[0] - loss) / loss < 3e-4
    # after one Adam step every pixel moved by lr * sign(g) (bias-corrected); stylize() then copies the
    # bias-corrected EMA back into the image (ST:496-497): compare both with the oracle's EMA
    ema_native = st.average.get().cpu()
    assert (ema_native - s0.ema_get()).abs().mean() < 1e-3   # sign flips only where |g| ~ 0
    assert (st.image.cpu() - s0.ema_get()).abs().mean() < 1e-3


def test_errors_are_reported(G, vgg_weights):
    st = G.make_st('max', vgg_weights)
    m = st.model
    m.ensure_workspace([(32, 32)])
    with pytest.raises(ValueError):  # ST:82-83
        m.style_stats(torch.zeros(1, 3, 8, 40, device=G.DEV))
    with pytest.raises(RuntimeError):  # iterate before set_targets
        st.image = torch.zeros(1, 3, 32, 32, device=G.DEV)
        st.loss_and_grad()
    with pytest.raises(ValueError):
        st.stylize(O.synth_image(1, 8, 32, 32), [O.synth_image(2, 8, 32, 32)], style_weights=[1, 2])
    with pytest.raises(ValueError):
        st.stylize(O.synth_image(1, 8, 32, 32), [O.synth_image(2, 8, 32, 32)], init='bogus')


def test_full_size_properties(G, vgg_weights):
    """2048x2048 (BASELINE.json config 3) is too big for the CPU oracle in a test, so check size-independent
    properties: finite decreasing loss, image stays in [0,1], EMA bias correction, determinism of the loss."""
    size = 2048
    content, style = O.synth_image(1, 16, size, size), O.synth_image(2, 32, size, size)
    st = G.make_st('max', vgg_weights)
    tr = []
    st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=8, callback=lambda it: tr.append(it.loss))
    assert all(np.isfinite(tr)) and tr[-1] < tr[0]
    assert float(st.image.min()) >= 0.0 and float(st.image.max()) <= 1.0
    st2 = G.make_st('max', vgg_weights)
    tr2 = []
    st2.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=2, callback=lambda it: tr2.append(it.loss))
    np.testing.assert_allclose(tr2, tr[:2], rtol=1e-5)  # split-K / reductions are order-deterministic
    # translation-of-scale property: the first-iteration loss at 2048^2 of a low-frequency pair is close to the
    # 256^2 loss of the same pair evaluated by the ORACLE (statistics of smooth fields are resolution independent
    # only loosely, so this is a sanity bound, not a parity claim)
    assert 0.0 < tr[0] < 10.0


def test_two_gpu_banded_equals_single_gpu():
    """Spatial tiling over 2 GPUs (NCCL): loss trace and result vs the single-GPU run (tools/dist_check.py)."""
    import subprocess
    import sys
    if torch.cuda.device_count() < 2:
        pytest.skip('needs 2 GPUs')
    root = Path(__file__).resolve().parent.parent
    r = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
                        '--master-addr', '127.0.0.1', '--master-port', '29533', str(root / 'tools' / 'dist_check.py'),
                        '384', '512', '5'], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------- per-iteration parity
def _resync_case(G, vgg_weights, content, styles, pooling, kw, style_weights=None):
    """Runs the public API and returns (native losses, oracle losses evaluated AT the native iterate of every
    iteration).  The loss an iteration reports (ST:481: the pre-update loss) is a pure function of the image it starts
    from, so feeding the native image back into the oracle's closure each step removes trajectory drift from the
    comparison: what is left is the 1e-3 bar of the north star, on every iteration and on every scale."""
    st = G.make_st(pooling, vgg_weights)
    recs = []

    def cb(it):
        recs.append((it.loss, it.w, it.h, it.i, st.image.detach().cpu().clone()))

    st.stylize(content, styles, callback=cb, **kw)
    sw = style_weights or [1.0 / len(styles)] * len(styles)
    norm = sum(abs(w) for w in sw)
    sw = [w / norm for w in sw]
    native, oracle = [], []
    tg_cache = {}
    scales = O.gen_scales(min(kw.get('min_scale', 128), kw.get('end_scale', 512)), kw.get('end_scale', 512))
    prev = None
    for loss, w, h, i, img in recs:
        key = (w, h)
        if key not in tg_cache:
            scale = next(s for s in scales if O.size_to_fit(content.size, s, scale_up=True) == (w, h))
            tg_cache[key] = O.make_targets(content, styles, sw, scale, vgg_weights, pooling,
                                           kw.get('content_weight', 0.015), kw.get('tv_weight', 2.0),
                                           kw.get('style_scale_fac', 1.0), kw.get('style_size'))[0]
        if i == 1:   # first iteration of a scale: the start image is not visible through the callback
            prev = img
            continue
        ol, _ = O.loss_and_grad(prev, vgg_weights, tg_cache[key], pooling)
        native.append(loss)
        oracle.append(float(ol))
        prev = img
    return np.array(native), np.array(oracle)


@pytest.mark.parametrize('name', ['max_64x48_single', 'avg_80x56_two_styles', 'l2_72x72_single', 'max_pyramid_32_64'])
def test_every_iteration_matches_the_oracle_at_the_native_iterate(G, vgg_weights, name):
    content, styles, pooling, kw = MG.build_case(name)
    native, oracle = _resync_case(G, vgg_weights, content, styles, pooling, dict(kw), kw.get('style_weights'))
    assert len(native) >= 2
    rel = np.abs(native - oracle) / oracle
    assert rel.max() < 1e-3, rel


def test_512_pyramid_every_checked_iteration_within_the_bar(G, vgg_weights):
    """BASELINE.json configs[1]: 512 x 512 end_scale, default multi-scale (128, 181, 256, 362, 512; 20 + 4 x 10
    iterations).  Every iteration but the first of each scale is re-evaluated by the fp32 oracle at the native
    iterate: 1e-3 on each.  (The reference's own trace of this case is tests/golden/max_pyramid_128_512.npz, replayed by
    test_stylize_matches_reference_golden.)"""
    content, styles, pooling, kw = MG.build_case('max_pyramid_128_512')
    native, oracle = _resync_case(G, vgg_weights, content, styles, pooling, dict(kw))
    assert len(native) == 20 + 4 * 10 - 5
    rel = np.abs(native - oracle) / oracle
    print('512 pyramid: max rel', rel.max(), 'mean', rel.mean())
    assert rel.max() < 1e-3, rel


# ---------------------------------------------------------------------------------------------- optimiser state
def _adam_reference(state, g, step, lr=0.02, b1=0.9, b2=0.99, eps=1e-8, decay=0.99):
    """torch/optim/adam.py:413-546 single-tensor math + clamp_ (ST:483-485) + EMA (ST:250-253), in float64 from fp32
    inputs; returns the new (image, exp_avg, exp_avg_sq, ema)."""
    x, m, v, e = (t.double() for t in state)
    g = g.double()
    m = m + (g - m) * (1 - b1)
    v = v * b2 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    x = (x - (lr / bc1) * m / (v.sqrt() / bc2 ** 0.5 + eps)).clamp(0, 1)
    e = e * decay + (1 - decay) * x
    return x, m, v, e


def _state_setup(G, vgg_weights, H=48, W=64):
    import style_transfer_b200 as stb
    st = G.make_st('max', vgg_weights)
    m = st.model
    cimg = O.to_tensor(O.synth_image(1, 16, W, H)).to(G.DEV)
    simg = O.to_tensor(O.synth_image(2, 32, 56, 40)).to(G.DEV)
    m.ensure_workspace([(H, W), (40, 56)])
    ct = m.content_features(cimg)
    means, srms = m.style_stats(simg)
    m.set_targets(H, W, ct, 0.015, means, srms, st.style_weights, 2.0)
    torch.manual_seed(3)
    img = (cimg + 0.05 * torch.randn_like(cimg)).clamp(0, 1).contiguous()
    return st, m, img, stb


def test_adam_moments_image_and_ema_after_1_2_5_steps(G, vgg_weights):
    """exp_avg / exp_avg_sq / image / EMA of the fused native update, compared DIRECTLY with the reference formulas fed
    the gradient the native iteration itself used (stb_iterate_ex returns it): bias correction at step > 1, the carried
    step counter (start at step 7, as after a previous scale) and the fused conv0-backward epilogue are all in play."""
    from style_transfer_b200 import _lib
    st, m, img, _ = _state_setup(G, vgg_weights)
    for first_step in (1, 7):
        x = img.clone()
        ea, eas = torch.zeros_like(x), torch.zeros_like(x)
        if first_step > 1:   # a warm-started state
            torch.manual_seed(first_step)
            ea = 1e-4 * torch.randn_like(x)
            eas = (1e-4 * torch.randn_like(x)) ** 2
        ema = x * 0.01
        ref = (x.cpu(), ea.cpu(), eas.cpu(), ema.cpu())
        grad = torch.empty_like(x)
        for k in range(5):
            step = first_step + k
            _lib.check(m.lib.stb_iterate_ex(m.ctx, _lib.ptr(x), _lib.ptr(ea), _lib.ptr(eas), _lib.ptr(ema), step, 0.02, 0.9,
                                            0.99, 1e-8, 0.99, 1, _lib.ptr(grad), None, _lib.cur_stream()))
            torch.cuda.synchronize()
            ref = _adam_reference(ref, grad.cpu(), step)
            if k in (0, 1, 4):
                for name, got, want in zip(('image', 'exp_avg', 'exp_avg_sq', 'ema'), (x, ea, eas, ema), ref):
                    err = (got.cpu().double() - want).abs().max().item()
                    scale = want.abs().max().item()
                    assert err <= 2e-6 * max(scale, 1e-30) + 1e-12, (first_step, step, name, err, scale)
            # keep the comparison a per-step one: continue from the native fp32 state
            ref = (x.cpu(), ea.cpu(), eas.cpu(), ema.cpu())


def test_graphed_iterations_equal_eager_ones(G, vgg_weights):
    """stb_iterate replays a CUDA graph from its third call on; the device-side step counter must advance exactly like
    the host-driven one: ten graphed steps == ten eager (grad_out != NULL disables the graph) steps, bit for bit."""
    from style_transfer_b200 import _lib
    st, m, img, _ = _state_setup(G, vgg_weights)
    outs = []
    side = torch.cuda.Stream()
    for eager in (False, True):
        x = img.clone()
        ea, eas, ema = torch.zeros_like(x), torch.zeros_like(x), x * 0.01
        grad = torch.empty_like(x) if eager else None
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for step in range(1, 11):
                _lib.check(m.lib.stb_iterate_ex(m.ctx, _lib.ptr(x), _lib.ptr(ea), _lib.ptr(eas), _lib.ptr(ema), step, 0.02,
                                                0.9, 0.99, 1e-8, 0.99, 1, _lib.ptr(grad), None, _lib.cur_stream()))
        side.synchronize()
        outs.append((x.cpu(), ea.cpu(), eas.cpu(), ema.cpu()))
    assert m.graph_status()[0] == 1
    for a, b in zip(*outs):
        torch.testing.assert_close(a, b, rtol=0, atol=0)


# ---------------------------------------------------------------------------------------------- SURVEY 8(f) rows
def test_lbfgs_runs_on_the_native_closure(G, vgg_weights):
    """optimizer='lbfgs' (ST:464-465): torch's L-BFGS on the host, closure = stb_iterate_ex(apply_update=0).  The loss
    must go down monotonically-ish and the first closure value equals the Adam path's first loss (same closure)."""
    content, style = O.synth_image(1, 16, 64, 48), O.synth_image(2, 32, 56, 40)
    kw = dict(min_scale=64, end_scale=64, initial_iterations=6)
    st = G.make_st('max', vgg_weights)
    tr_l, tr_a = [], []
    out = st.stylize(content, [style], optimizer='lbfgs', callback=lambda it: tr_l.append(it.loss), **kw)
    G.make_st('max', vgg_weights).stylize(content, [style], callback=lambda it: tr_a.append(it.loss), **kw)
    assert out.size == (64, 48) and len(tr_l) == 6 and np.isfinite(tr_l).all()
    assert abs(tr_l[0] - tr_a[0]) / tr_a[0] < 1e-5
    assert tr_l[-1] < 0.7 * tr_l[0]
    with pytest.raises(ValueError):
        st.stylize(content, [style], optimizer='sgd', **kw)


def test_async_writer_saves_a_device_snapshot(G, vgg_weights, tmp_path):
    """image_io.AsyncImageWriter.submit_snapshot: device-side uint8 snapshot -> pinned host -> PNG on a worker thread
    (the CLI's save path, off the loop); the file must hold exactly what get_image() returns."""
    from PIL import Image
    from style_transfer_b200.image_io import AsyncImageWriter
    content, style = O.synth_image(1, 16, 64, 48), O.synth_image(2, 32, 56, 40)
    st = G.make_st('max', vgg_weights)
    wr = AsyncImageWriter()
    path = tmp_path / 'snap.png'
    st.stylize(content, [style], min_scale=64, end_scale=64, initial_iterations=3,
               callback=lambda it: wr.submit_snapshot(st, path))
    wr.close()
    saved = np.asarray(Image.open(path))
    np.testing.assert_array_equal(saved, np.asarray(st.get_image()))


def test_default_devices_argument_lands_on_cuda(vgg_weights):
    """The reference's default is devices=['cpu'] (ST:310): call sites relying on it must keep working -- on the GPU."""
    import style_transfer_b200 as stb
    with pytest.warns(UserWarning, match='no CPU fallback'):
        st = stb.StyleTransfer(vgg_weights=vgg_weights)
    assert st.devices[0].type == 'cuda'
    with pytest.raises(ValueError):
        stb.StyleTransfer(devices=['cuda:0', 'cuda:0', 'cuda:0'], vgg_weights=vgg_weights)
