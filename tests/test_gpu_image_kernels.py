"""-m gpu: the kernels at the two ends of the VGG trunk (conv0 forward, conv0 backward with the fused Adam step, TV,
pool backward, the fused pool forward, the content SSE) element by element against float64 references.

Every bar below is derived from the kernel's arithmetic, not fitted to measurements; u = 2^-24 is the unit roundoff
of fp32.  Each output is filled with NaN before a call, so an element the kernel does not write fails its bar.  The
conv references run on the device in float64 (cuDNN / ATen double kernels, independent of this library) and are
cross-checked against the CPU oracle once.  The persistent kernels are tested at shapes where every CTA walks two or
more work items (test_tested_shapes_give_every_cta_two_items).
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import st_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
NAN = float('nan')
# the fp32 constants of Normalize as the kernels (and the reference's fp32 tensors) hold them
MEAN32 = torch.tensor(O.NORM_MEAN, dtype=torch.float32).double().view(1, 3, 1, 1)
STD32 = torch.tensor(O.NORM_STD, dtype=torch.float32).double().view(1, 3, 1, 1)


def f32(x):
    return torch.tensor(x, dtype=torch.float32).item()


# Adam hyper-parameters as the fp32 values the kernels receive; the fp64 reference starts from the same values
LR, BETA1, BETA2, EPS, DECAY = f32(0.02), f32(0.9), f32(0.99), f32(1e-8), f32(0.99)
TV_WEIGHT = 2.0

CONV0_FWD_SHAPES = [(16, 16), (17, 127), (18, 128), (19, 129), (33, 257), (517, 1029), (1024, 1024), (2048, 1024)]
CONV0_BWD_SHAPES = [(1, 40), (40, 1), (2, 40), (3, 3), (16, 16), (20, 32), (21, 33), (33, 126), (34, 127), (35, 128),
                    (64, 252), (66, 253), (1024, 1024), (2048, 1024), (1024, 2048)]
POOL_BWD_SHAPES = [(64, 1024, 1024), (128, 363, 513), (256, 181, 91), (512, 45, 33), (64, 2, 2), (64, 3, 5)]
SSE_SIZES = [8, 4096, 512 * 16 ** 2, 512 * 128 ** 2, 512 * 256 ** 2]


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return g


@pytest.fixture(scope='module')
def conv0_weights(G):
    w0, b0 = O.make_vgg_weights(7)[0]
    return w0.to(G.DEV), b0.to(G.DEV)


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def nchw(x_hwc):
    return x_hwc.permute(2, 0, 1)[None]


# ------------------------------------------------------------------------------------------------ reference helpers
def conv0_fwd_ref(img, w0, b0):
    """conv0 pre-activation conv(pad(normalise(x)), bf16(w0)) + b in float64 and its magnitude
    A = conv(|v|, |bf16(w0)|) + |b|; img [1,3,H,W] fp32, result [1,64,H,W]."""
    v = F.pad((img.double() - MEAN32.to(img.device)) / STD32.to(img.device), (1, 1, 1, 1), mode='replicate')
    wb = w0.bfloat16().double()
    pre = F.conv2d(v, wb, b0.double())
    A = F.conv2d(v.abs(), wb.abs()) + b0.double().abs().view(1, -1, 1, 1)
    return pre, A


def fold_pad(gp):
    """Adjoint of the one-pixel replicate pad: [.., H+2, W+2] -> [.., H, W]."""
    gp = gp.clone()
    gp[..., 1, :] += gp[..., 0, :]
    gp[..., -2, :] += gp[..., -1, :]
    gp[..., :, 1] += gp[..., :, 0]
    gp[..., :, -2] += gp[..., :, -1]
    return gp[..., 1:-1, 1:-1]


def border_ring(H, W, device):
    ring = torch.ones(H, W, dtype=torch.bool, device=device)
    ring[1:-1, 1:-1] = False
    return ring


def conv0_bwd_ref(g0, w0):
    """d loss / d image of conv0 (replicate pad + Normalize) in float64 for g0 [H][W][64] bf16, and its magnitude A,
    both [3,H,W].  As the kernels compute it: the interior pixels on bf16(w0) (wgmma kernel), the border ring on the
    fp32 w0 (SIMT kernel), where the pad's adjoint folds the outer taps onto the pixel."""
    g = nchw(g0).double()
    std = STD32.to(g.device)
    H, W = g0.shape[:2]
    ring = border_ring(H, W, g.device)

    def grad(gg, wb, wf):
        inner = fold_pad(F.conv_transpose2d(gg, wb)) / std     # the fold touches the ring only
        outer = fold_pad(F.conv_transpose2d(gg, wf)) / std
        return torch.where(ring, outer, inner)[0]

    wb, wf = w0.bfloat16().double(), w0.double()
    return grad(g, wb, wf), grad(g.abs(), wb.abs(), wf.abs())


def tv_grad_magnitude(x, tv_weight):
    """B of the TV gradient bar: the TV gradient's stencil with every difference e = a - b replaced by |a| + |b|
    (same k1 / k3 weights, same fold of the pad ring); x [1,3,H,W] float64."""
    p = F.pad(x, (1, 1, 1, 1), mode='replicate').abs()
    n1 = x.numel()
    n3 = 3 * (x.shape[2] + 1) * (x.shape[3] + 1)
    k1, k3 = tv_weight * 4 / (3 * n1), tv_weight * 4 / (12 * n3)
    s1, s2, s3, s4 = slice(1, -1), slice(2, None), slice(None, -1), slice(1, None)
    gp = torch.zeros_like(p)
    for k, (ya, xa), (yb, xb) in ((k1, (s1, s2), (s1, s1)), (k1, (s2, s1), (s1, s1)),
                                  (k3, (s4, s4), (s3, s3)), (k3, (s4, s3), (s3, s4))):
        mag = k * (p[..., ya, xa] + p[..., yb, xb])
        gp[..., ya, xa] += mag
        gp[..., yb, xb] += mag
    return fold_pad(gp)


def adam_ref(g, m, v, p, e, step, lr):
    """torch's single-tensor Adam step (lerp form) + clamp_(0, 1) + EMA in float64, and the bar of every output.
    Each bar is c * u times the magnitudes of its formula's operands (first-order rounding analysis, c <= 16):
      m' = m + (g - m)(1 - b1): a difference, a product, a sum              -> 4 u (|m| + (1 - b1)(|g| + |m|))
      v' = v b2 + (1 - b2) g g: three products, one sum (nonnegative terms) -> 4 u (b2 |v| + (1 - b2) g^2)
      p' = p - S m' / (sqrt(v') / sqrt(bc2) + eps): m' carries 4 u Mm absolutely, the denominator 2 u from v' plus
           four roundings, then the division, S = lr / bc1 rounded to fp32, the product and the subtraction
           -> 16 u (|p| + S (|m'| + Mm) / denom); the clamp is 1-Lipschitz
      e' = e d + (1 - d) p': the error of p' times (1 - d), plus two products and a sum -> (1 - d) bar_p + 4 u (...)
    """
    b1, b2, d = BETA1, BETA2, DECAY
    m1 = m + (g - m) * (1 - b1)
    v1 = v * b2 + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    denom = v1.sqrt() / math.sqrt(bc2) + EPS
    S = lr / bc1
    pre = p - S * m1 / denom
    p1 = pre.clamp(0, 1)
    e1 = e * d + (1 - d) * p1
    Mm = m.abs() + (1 - b1) * (g.abs() + m.abs())
    bar_m = 4 * U * Mm
    bar_v = 4 * U * (b2 * v.abs() + (1 - b2) * g * g)
    bar_p = 16 * U * (p.abs() + S * (m1.abs() + Mm) / denom)
    bar_e = (1 - d) * bar_p + 4 * U * (d * e.abs() + (1 - d) * p1.abs())
    return (m1, v1, p1, e1), (bar_m, bar_v, bar_p, bar_e), pre


def check_bar(name, got, ref, bar):
    """|got - ref| <= bar everywhere (NaN fails); returns the largest error / bar."""
    err = (got.double() - ref).abs()
    ok = err <= bar
    ratio = (err / bar.clamp_min(1e-300)).max().item()
    assert ok.all(), (f'{name}: {int((~ok).sum())} of {ok.numel()} elements over the bar, worst error / bar '
                      f'{ratio:.3g}')
    return ratio


def bitwise_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


# ------------------------------------------------------------------------------------------------ persistent loops
def _launch_grids(sms):
    """Work items and grid of every persistent kernel tested here, as their launchers compute them."""
    def cdiv(a, b):
        return -(-a // b)
    conv0_fwd = [(cdiv(H, 4) * cdiv(W, 128), 2 * sms) for H, W in CONV0_FWD_SHAPES]        # 4 rows x 128 px
    conv0_bwd = [(cdiv(W, 126) * cdiv(H, 32), 2 * sms) for H, W in CONV0_BWD_SHAPES]       # 32 rows x 126 cols
    # grid-stride kernels: one item = one thread, 256 threads per block, at most 16 blocks per SM (grid_for)
    pool = [(cdiv(H, 2) * cdiv(W, 2) * (C // 8), 16 * sms * 256) for C, H, W in POOL_BWD_SHAPES]
    sse = [(n // 8, min(16 * sms, 1024) * 256) for n in SSE_SIZES]
    return {'conv0 fwd': conv0_fwd, 'conv0 bwd interior': conv0_bwd, 'pool bwd': pool, 'content sse': sse}


def test_tested_shapes_give_every_cta_two_items(G):
    """Fails on a device with more SMs than these shapes were planned for, rather than silently testing less: the
    next-item halo prefetch of conv0 forward, the D-ring restart and state reload of conv0 backward and the
    grid-stride loops only run when a CTA (thread) gets a second item."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for kernel, cases in _launch_grids(sms).items():
        per_cta = [items / min(items, cap) for items, cap in cases]
        assert max(per_cta) >= 2, f'{kernel}: on {sms} SMs no tested shape wraps (items per CTA {per_cta})'


# ------------------------------------------------------------------------------------------------ oracle cross-check
def test_references_match_cpu_oracle(G, conv0_weights):
    """The device float64 references above are the oracle's functions (up to the fp32 rounding of the Normalize
    constants, far below every bar), and the magnitudes bound the values."""
    w0, b0 = conv0_weights
    H, W = 19, 23
    g = torch.Generator().manual_seed(11)
    img = torch.rand(1, 3, H, W, generator=g)
    g0 = (torch.randn(H, W, 64, generator=g) * (torch.rand(H, W, 64, generator=g) > 0.5)).bfloat16()
    wb = [(w0.cpu().bfloat16().double(), b0.cpu().double())]
    wf = [(w0.cpu().double(), b0.cpu().double())]

    pre, A = conv0_fwd_ref(img.to(G.DEV), w0, b0)
    oracle = O.vgg_forward(img.double(), wb, 'max', 1)[1]
    assert ((torch.relu(pre).cpu() - oracle).abs() <= 2.0 ** -20 * A.cpu()).all()
    assert (pre.abs() <= A).all()

    ref, Ab = conv0_bwd_ref(g0.to(G.DEV), w0)
    ones = {1: torch.ones(1, 64, H, W, dtype=torch.float64)}
    ring = border_ring(H, W, 'cpu')
    o_int = O.vgg_backward({1: nchw(g0).double()}, ones, wb, 'max')[0]
    o_ring = O.vgg_backward({1: nchw(g0).double()}, ones, wf, 'max')[0]
    expect = torch.where(ring, o_ring, o_int)
    assert ((ref.cpu() - expect).abs() <= 2.0 ** -20 * Ab.cpu()).all()
    assert (ref.abs() <= Ab).all()

    _, tvg = O.tv_loss_and_grad(img.double())
    assert ((tvg * TV_WEIGHT).abs() <= tv_grad_magnitude(img.double(), TV_WEIGHT) * (1 + 1e-12)).all()


# ------------------------------------------------------------------------------------------------ conv0 forward
@pytest.mark.parametrize('H,W', CONV0_FWD_SHAPES)
def test_conv0_forward_elementwise(G, conv0_weights, H, W):
    """got == RN_bf16(ref), except within delta = 2^-15 A of a rounding boundary, where either neighbour passes.
    The kernel's pre-activation differs from ref by at most
      * the input split: v in fp32 ((x - mean) * fl(1/std): 3 u |v|), hi = RN_bf16(v) exact, lo = RN_bf16(v - hi) off
        by 2^-9 |v - hi| <= 2^-18 |v|, so hi + lo = v (1 +- (2^-18 + 3 u));
      * the products hi * w, lo * w of bf16 values, exact in fp32, and the fp32 sum of 54 of them plus the bias:
        <= 55 u sum|terms| ~ 2^-18.2 A;
    about 2^-17 A in all, so delta = 2^-15 A leaves a factor 4 for the tensor cores' accumulation order.  Dropping
    the lo half moves the value by up to 2^-9 |v| |w|, far outside."""
    w0, b0 = conv0_weights
    img = torch.rand(1, 3, H, W, generator=_gen(H * 7919 + W), device=G.DEV)
    out = torch.full((H, W, 64), NAN, dtype=torch.bfloat16, device=G.DEV)
    G.check(G.lib().stb_test_conv0_fwd(G.P(img), G.P(w0), G.P(b0), G.P(out), H, W, 0.0, None, None, None, G.S()))
    torch.cuda.synchronize()
    pre, A = conv0_fwd_ref(img, w0, b0)
    got = nchw(out).double()
    delta = 2.0 ** -15 * A
    ok = G.rn_window(got, pre, delta, relu=True)
    bad = int((~ok).sum())
    assert bad == 0, f'{bad} of {ok.numel()} elements outside the RN window (first at {(~ok).nonzero()[0].tolist()})'
    print(f'RATIO conv0_fwd {H}x{W} {G.rn_window_ratio(got, pre, delta, relu=True):.3g}')


# ------------------------------------------------------------------------------------------------ conv0 backward
def _conv0_bwd(G, g0, w0, gtv, H, W, state=None, step=0, lr=0.0):
    grad = torch.full((3, H, W), NAN, device=G.DEV)
    if state is None:
        G.check(G.lib().stb_test_conv0_bwd(G.P(g0), G.P(w0), G.P(gtv), G.P(grad), H, W, G.S()))
    else:
        img, m, v, e = state
        G.check(G.lib().stb_test_conv0_bwd_adam(G.P(g0), G.P(w0), G.P(gtv), G.P(grad), H, W, G.P(img), G.P(m), G.P(v),
                                                G.P(e), step, lr, BETA1, BETA2, EPS, DECAY, 1, G.S()))
    torch.cuda.synchronize()
    return grad


def _adam_state(case, grad, seed):
    """(img, exp_avg, exp_avg_sq, ema, step, lr) before the update."""
    gen = _gen(seed)
    gscale = grad.abs().mean().item()
    p = torch.rand(grad.shape, generator=gen, device='cuda')
    if case == 'warm7':
        m = torch.randn(grad.shape, generator=gen, device='cuda') * gscale
        v = (torch.randn(grad.shape, generator=gen, device='cuda') * gscale) ** 2 + (0.1 * gscale) ** 2
        e = torch.rand(grad.shape, generator=gen, device='cuda')
        return p, m, v, e, 7, LR
    if case == 'clamp':
        # the first step moves every pixel by lr = 0.02 against the gradient's sign: channels 0 and 1 start within
        # 0.005 of the bound it moves towards, so they clamp; channel 2 stays uniform
        t = 0.005 * torch.rand(grad.shape, generator=gen, device='cuda')
        p[:2] = torch.where(grad[:2] > 0, t[:2], 1 - t[:2])
    z = torch.zeros_like(p)
    return p, z, z.clone(), (1 - DECAY) * p, 1, LR


@pytest.mark.parametrize('H,W', CONV0_BWD_SHAPES)
def test_conv0_backward_and_adam_elementwise(G, conv0_weights, H, W):
    """grad_out: |got - ref| <= 2^-16 A, ref and A as conv0_bwd_ref, plus the gtv plane.
      * interior (wgmma kernel): the bf16 x bf16 products are exact in fp32, the 64-term channel sum <= 64 u, the
        9-term col2im sum 9 u, * fl(1/std) 2 u, + gtv u: ~76 u = 2^-17.8 A;
      * border ring (SIMT kernel): per lane 2 channels x 9 taps x at most 6 folded positions of fmaf, a 5-level
        butterfly, / std, + gtv: <= 116 u = 2^-17.1 A.
    The update of both kernels is then compared with torch's Adam formula in float64 fed the kernel's own grad_out
    (adam_ref for the bars).  Recomputing the interior with fp32 weights moves it by ~2^-9 A, and an extra or a
    missing Adam step moves img by ~lr: orders of magnitude over the bars."""
    w0, _ = conv0_weights
    gen = _gen(H * 7907 + W)
    g0 = (torch.randn(H, W, 64, generator=gen, device=G.DEV) *
          (torch.rand(H, W, 64, generator=gen, device=G.DEV) > 0.5)).bfloat16()
    conv_part, A = conv0_bwd_ref(g0, w0)
    gscale = conv_part.abs().mean().item()
    gtv = 0.1 * gscale * torch.randn(3, H, W, generator=gen, device=G.DEV)
    ref = conv_part + gtv.double()
    A = A + gtv.double().abs()

    grad0 = _conv0_bwd(G, g0, w0, gtv, H, W)
    r = check_bar(f'grad {H}x{W}', grad0, ref, 2.0 ** -16 * A)
    print(f'RATIO conv0_bwd_grad {H}x{W} {r:.3g}')

    ring = border_ring(H, W, G.DEV).expand(3, H, W)
    for k, case in enumerate(('step1', 'warm7', 'clamp')):
        p, m, v, e, step, lr = _adam_state(case, grad0, H * 7901 + W * 13 + k)
        runs = []
        for _ in range(2):
            st = [t.clone() for t in (p, m, v, e)]
            runs.append((_conv0_bwd(G, g0, w0, gtv, H, W, st, step, lr), st))
        (grad1, st1), (grad2, st2) = runs
        assert bitwise_equal(grad1, grad2) and all(bitwise_equal(a, b) for a, b in zip(st1, st2)), \
            f'{case}: the second run is not bit-identical'
        assert bitwise_equal(grad1, grad0), f'{case}: grad_out with the update differs from grad_out without'
        refs, bars, pre = adam_ref(grad1.double(), m.double(), v.double(), p.double(), e.double(), step, lr)
        got = (st1[1], st1[2], st1[0], st1[3])
        ratios = [check_bar(f'{case} {name} {H}x{W}', gt, rf, br)
                  for name, gt, rf, br in zip(('exp_avg', 'exp_avg_sq', 'img', 'ema'), got, refs, bars)]
        print(f'RATIO conv0_bwd_adam {case} {H}x{W} ' + ' '.join(f'{x:.3g}' for x in ratios))
        if case == 'clamp':
            clamped = (pre < 0) | (pre > 1)
            assert clamped[ring].any() and (H < 3 or W < 3 or clamped[~ring].any()), 'the clamp was not exercised'


# ------------------------------------------------------------------------------------------------ TV
def _tv(G, img, H, W, row0, rows, H_norm):
    gx = -(-W // 256)
    gtv = torch.full((3, H, W), NAN, device=G.DEV)
    parts = torch.full((gx * rows,), NAN, device=G.DEV)
    n = ctypes.c_int()
    G.check(G.lib().stb_test_tv(G.P(img), H, W, row0, rows, H_norm, TV_WEIGHT, G.P(gtv), G.P(parts), ctypes.byref(n),
                                G.S()))
    torch.cuda.synchronize()
    assert n.value == gx * rows
    return gtv, parts


@pytest.mark.parametrize('H,W', [(2, 2), (16, 16), (255, 257), (1024, 1024)])
def test_tv_elementwise(G, H, W):
    """Gradient: |got - ref| <= 2^-20 B (tv_grad_magnitude).  Every term k (a - b) costs a rounding in the
    difference and one in the product with k (itself rounded to fp32), and sits at most 8 + 4 deep in the sums of a
    corner pixel's slow path (<= 8 terms per padded position, <= 4 positions), so the error is <= 15 u B < 2^-20 B;
    the interior path's 4 + 4 differences, 2 products and a sum stay under 7 u B.
    Loss: the fp64 sum of the partials within 24 u relative: every squared difference (difference, square, two
    sums, the weight l rounded to fp32 and the product, two far-border extras) passes <= 8 roundings, then the
    3-channel sum, the 5-level warp sum and the 8-term block sum: <= 23 roundings on any term's path, and the terms
    are nonnegative."""
    img = torch.rand(1, 3, H, W, generator=_gen(H * 31 + W), device=G.DEV)
    gtv, parts = _tv(G, img, H, W, 0, H, H)
    loss, grad = O.tv_loss_and_grad(img.double())
    r = check_bar(f'tv grad {H}x{W}', gtv[None], grad * TV_WEIGHT, 2.0 ** -20 * tv_grad_magnitude(img.double(),
                                                                                                   TV_WEIGHT))
    assert torch.isfinite(parts).all()
    rl = abs(parts.double().sum().item() - loss.item()) / (24 * U * loss.item())
    assert rl <= 1, f'tv loss error / bar {rl:.3g}'
    print(f'RATIO tv {H}x{W} grad {r:.3g} loss {rl:.3g}')


@pytest.mark.parametrize('H,W', [(255, 257), (1024, 1024)])
def test_tv_band_windows_match_whole_image(G, H, W):
    """A band's call (own rows of a local image with up to 80 apron rows, H_norm = the global height) computes every
    own row exactly as the whole-image call does: the gradient rows and per-row partials are bit-identical, and rows
    outside the window are not written."""
    img = torch.rand(1, 3, H, W, generator=_gen(H * 37 + W), device=G.DEV)
    gtv_all, parts_all = _tv(G, img, H, W, 0, H, H)
    gx = -(-W // 256)
    cuts = [0, H // 3, 2 * H // 3, H]
    for own0, own1 in zip(cuts[:-1], cuts[1:]):
        lo, hi = max(0, own0 - 80), min(H, own1 + 80)
        local = img[:, :, lo:hi].contiguous()
        gtv, parts = _tv(G, local, hi - lo, W, own0 - lo, own1 - own0, H)
        assert bitwise_equal(gtv[:, own0 - lo:own1 - lo], gtv_all[:, own0:own1]), f'band [{own0}, {own1})'
        assert bitwise_equal(parts, parts_all[own0 * gx:own1 * gx]), f'band [{own0}, {own1}) partials'
        outside = torch.ones(hi - lo, dtype=torch.bool, device=G.DEV)
        outside[own0 - lo:own1 - lo] = False
        assert torch.isnan(gtv[:, outside]).all(), f'band [{own0}, {own1}) wrote rows outside its window'


# ------------------------------------------------------------------------------------------------ pool backward
def _pool_input(C, H, W, gen):
    """relu(randn) with exact ties (the top row of every window in rows 0 mod 4 repeats its left value) and
    all-zero windows (rows 4, 5 mod 10)."""
    x = torch.relu(torch.randn(H, W, C, generator=gen, device='cuda'))
    w2 = 2 * (W // 2)
    x[0::4, 1:w2:2] = x[0::4, 0:w2:2]
    x[4::10] = 0
    x[5::10] = 0
    x[::3, ::2] = 0
    return x.bfloat16()


@pytest.mark.parametrize('C,H,W', POOL_BWD_SHAPES)
@pytest.mark.parametrize('pooling', ['max', 'average', 'l2'])
def test_pool_backward_elementwise(G, C, H, W, pooling):
    """Max: the routed gradient itself, bit-exact (first maximum in scan order).  Average: g * 0.5, exact in bf16,
    bit-exact.  L2: g x / s * 0.78 with s = sqrtf of four exact bf16 squares (3 u / 2 + u / 2), the fp32 0.78 and the
    quotient and two products: < 6 u relative, so RN_bf16(ref) within delta = 2^-21 |ref|.  The floor-mode ragged
    row / column gets exact zeros (ref 0, delta 0)."""
    code = {'max': 0, 'average': 1, 'l2': 2}[pooling]
    gen = _gen(C * 1009 + H * 17 + W)
    x = _pool_input(C, H, W, gen)
    go = torch.randn(H // 2, W // 2, C, generator=gen, device=G.DEV).bfloat16()
    gin = torch.full((H, W, C), NAN, dtype=torch.bfloat16, device=G.DEV)
    G.check(G.lib().stb_test_pool_bwd(code, G.P(go), G.P(x), G.P(gin), H, W, C, G.S()))
    torch.cuda.synchronize()
    xd = nchw(x).double()
    ref = O.pool_bwd(nchw(go).double(), xd, pooling) * (xd > 0)
    got = nchw(gin).double()
    if pooling != 'l2':
        bad = ~(got == ref)
        assert not bad.any(), f'{int(bad.sum())} elements differ (first at {bad.nonzero()[0].tolist()})'
        return
    delta = 2.0 ** -21 * ref.abs()
    ok = G.rn_window(got, ref, delta)
    assert ok.all(), f'{int((~ok).sum())} elements outside the RN window (first at {(~ok).nonzero()[0].tolist()})'
    print(f'RATIO pool_bwd_l2 {C},{H},{W} {G.rn_window_ratio(got.abs(), ref.abs(), delta):.3g}')


# ------------------------------------------------------------------------------------------------ fused pool forward
@pytest.mark.parametrize('H,W,Cin,Cout', [(362, 512, 64, 64), (181, 256, 128, 128), (91, 64, 256, 256),
                                          (45, 33, 512, 512), (32, 24, 64, 64), (37, 21, 64, 128), (18, 50, 128, 256),
                                          (6, 6, 512, 512)])
@pytest.mark.parametrize('pooling', ['max', 'average', 'l2'])
def test_fused_pool_forward_elementwise(G, H, W, Cin, Cout, pooling):
    """The pool of the conv output as stored (bf16), floor mode.  Max: bit-exact.  Average: bit-exact against the
    epilogue's fp32 arithmetic, ((a + b) + c) + d, * 0.25, * 2 (exact), RN to bf16 (the build uses no fast-math).
    L2: sqrtf of a sum of four exact squares (3 u / 2 + u / 2), * 0.78f (2 u): RN_bf16(ref) within 2^-21 |ref|.
    The stored conv output itself is checked element by element in test_gpu_pixel_gemm.py, on the same launches."""
    code = {'max': 0, 'average': 1, 'l2': 2}[pooling]
    gen = _gen(H * W + Cout)
    x = torch.randn(H, W, Cin, generator=gen, device=G.DEV).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, generator=gen, device=G.DEV) * (2.0 / (9 * Cin)) ** 0.5
    b = torch.randn(Cout, generator=gen, device=G.DEV) * 0.1
    wp = G.pack(w, False)
    out = torch.full((H, W, Cout), NAN, dtype=torch.bfloat16, device=G.DEV)
    pooled = torch.full((H // 2, W // 2, Cout), NAN, dtype=torch.bfloat16, device=G.DEV)
    G.check(G.lib().stb_test_conv_pool(H, W, Cin, Cout, G.P(x), G.P(wp), G.P(b), G.P(out), G.P(pooled), code, G.S()))
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    o = out.float()
    h2, w2 = 2 * (H // 2), 2 * (W // 2)
    a, bb, c, d = o[0:h2:2, 0:w2:2], o[0:h2:2, 1:w2:2], o[1:h2:2, 0:w2:2], o[1:h2:2, 1:w2:2]
    if pooling == 'max':
        ref = torch.maximum(torch.maximum(a, bb), torch.maximum(c, d)).bfloat16()
    elif pooling == 'average':
        ref = ((((a + bb) + c) + d) * 0.25 * 2.0).bfloat16()
    else:
        r64 = (a.double() ** 2 + bb.double() ** 2 + c.double() ** 2 + d.double() ** 2).sqrt() * 0.78
        delta = 2.0 ** -21 * r64
        ok = G.rn_window(pooled.double(), r64, delta)
        assert ok.all(), f'{int((~ok).sum())} pooled elements outside the RN window'
        print(f'RATIO pool_fwd_l2 {H}x{W}x{Cout} {G.rn_window_ratio(pooled.double(), r64, delta):.3g}')
        return
    bad = ~(pooled == ref)
    assert not bad.any(), f'{int(bad.sum())} pooled elements differ (first at {bad.nonzero()[0].tolist()})'


# ------------------------------------------------------------------------------------------------ content SSE
def _sse(G, a, b, n):
    parts = torch.full((1024,), NAN, device=G.DEV)
    k = ctypes.c_int()
    rc = G.lib().stb_test_sse(G.P(a), G.P(b), n, G.P(parts), ctypes.byref(k), G.S())
    torch.cuda.synchronize()
    return rc, parts, k.value


def _sse_bar(n, n_parts):
    """(elements per thread + 16) u relative: each thread fmaf-sums its elements (one rounding each, after the exact
    bf16 difference and square), then a 5-level warp sum, the 8-term block sum and the rounding of a difference of
    bf16 values with far-apart exponents; the fp64 sum of the partials adds nothing measurable.  All terms are
    nonnegative, so the bound is relative to the sum."""
    per_thread = 8 * -(-(n // 8) // (n_parts * 256))
    return (per_thread + 16) * U


def _check_sse(name, parts, k, n, a, b):
    assert 1 <= k <= 1024 and torch.isfinite(parts[:k]).all()
    ref = ((a.double() - b.double()) ** 2).sum().item()
    r = abs(parts[:k].double().sum().item() - ref) / (_sse_bar(n, k) * ref)
    assert r <= 1, f'{name}: error / bar {r:.3g}'
    return r


@pytest.mark.parametrize('n', SSE_SIZES)
def test_content_sse(G, n):
    gen = _gen(n)
    a = torch.relu(torch.randn(n, generator=gen, device=G.DEV)).bfloat16()
    b = torch.relu(torch.randn(n, generator=gen, device=G.DEV)).bfloat16()
    rc, parts, k = _sse(G, a, b, n)
    G.check(rc)
    print(f'RATIO sse n={n} {_check_sse(f"n={n}", parts, k, n, a, b):.3g}')


def test_content_sse_band_offset(G):
    """A band passes a pointer to its own rows inside the whole layer; the rows around them must not count."""
    rows, w, c, r0, own = 64, 32, 512, 24, 16
    gen = _gen(5)
    a = torch.relu(torch.randn(rows, w, c, generator=gen, device=G.DEV))
    b = torch.relu(torch.randn(rows, w, c, generator=gen, device=G.DEV))
    a[:r0], a[r0 + own:], b[:r0], b[r0 + own:] = 1e3, 1e3, -1e3, -1e3
    a, b = a.bfloat16(), b.bfloat16()
    n = own * w * c
    rc, parts, k = _sse(G, a[r0:r0 + own], b[r0:r0 + own], n)
    G.check(rc)
    _check_sse('band', parts, k, n, a[r0:r0 + own], b[r0:r0 + own])


def test_content_sse_rejects_ragged_n(G):
    from style_transfer_b200 import _lib
    a = torch.ones(64, dtype=torch.bfloat16, device=G.DEV)
    for n in (1, 7, 12, 63):
        assert _sse(G, a, a, n)[0] == _lib.STB_ERR_INVALID, n
