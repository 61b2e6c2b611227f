"""-m gpu: every CUDA kernel, called through the C-ABI, against the CPU oracle (oracle/st_oracle.py).

Tolerances (floating point; north_star: 1e-3 relative on the loss):
  * tensor-core kernels take bf16 operands and write bf16: the comparison is against an fp32 evaluation on the
    SAME bf16-rounded operands, so the only differences are fp32 summation order and the final bf16 rounding
    (2^-9 relative) -> 6e-3 of the output range;
  * fp32 kernels (TV, conv0 dgrad, Gram accumulation, W2 chain): 1e-5 .. 2e-3 as noted per test.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from oracle import st_oracle as O  # noqa: E402


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return g


@pytest.mark.parametrize('H,W,Cin,Cout,c2,content,only_c2,mode', [
    (32, 24, 64, 64, 0, False, False, 1), (45, 34, 64, 128, 0, False, False, 1), (22, 22, 256, 512, 0, False, False, 1),
    (37, 19, 512, 512, 512, False, False, 1), (32, 24, 64, 64, 64, True, False, 1),
    (20, 12, 512, 512, 512, False, True, 1)])
def test_conv3x3_dgrad_with_tap_gradient(G, H, W, Cin, Cout, c2, content, only_c2, mode):
    """dgrad of a conv Cin->Cout (gout [H,W,Cout] -> gin [H,W,Cin]) + F Gs + gmu + content term, ReLU-masked."""
    g = torch.Generator().manual_seed(7 * H + W)
    go = torch.randn(H, W, Cout, generator=g).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, generator=g) * (2.0 / (9 * Cin)) ** 0.5
    y = torch.relu(torch.randn(H, W, Cin, generator=g)).bfloat16()
    ref = torch.zeros(1, Cin, H, W)
    keep = [go.to(G.DEV), w.to(G.DEV), y.to(G.DEV)]
    kw = {}
    if not only_c2:
        ref = F.conv_transpose2d(G.nchw(go), w.bfloat16().float(), padding=1)
        kw.update(A=keep[0], Bw=G.pack(keep[1], True))
    if c2:
        f2 = torch.randn(H, W, c2, generator=g).bfloat16()
        gs = (torch.randn(Cin, c2, generator=g) * 0.05).bfloat16()
        gmu = torch.randn(Cin, generator=g) * 0.1
        ref = ref + G.nchw((f2.float().reshape(-1, c2) @ gs.float().t()).reshape(H, W, Cin) + gmu)
        keep += [f2.to(G.DEV), gs.to(G.DEV), gmu.to(G.DEV)]
        kw.update(A2=keep[-3], B2=keep[-2], bias=keep[-1])
    cs = 0.0
    if content:
        ct = torch.relu(torch.randn(H, W, Cin, generator=g)).bfloat16()
        cs = 0.37
        ref = ref + cs * G.nchw(y.float() - ct.float())
        keep.append(ct.to(G.DEV))
        kw.update(ctarget=keep[-1])
    if mode == 1:
        ref = ref * G.nchw(y.float() > 0)
    out = G.pixel_gemm(H, W, 0 if only_c2 else Cout, Cin, c2, mode, mask=keep[2] if mode == 1 else None, cscale=cs, **kw)
    assert G.rel_err(G.nchw(out), ref) < 6e-3


def test_tap_gradient_row_window(G):
    """Second source restricted to rows [a2_row0, a2_row0+rows): the multi-GPU 'own rows' mechanism."""
    H, W, C = 40, 16, 64
    g = torch.Generator().manual_seed(3)
    f2 = torch.randn(H, W, C, generator=g).bfloat16()
    gs = (torch.randn(C, C, generator=g) * 0.05).bfloat16()
    gmu = torch.randn(C, generator=g) * 0.1
    y = torch.ones(H, W, C).bfloat16()
    r0, rows = 16, 16
    f2d, gsd, gmud, yd = f2.to(G.DEV), gs.to(G.DEV), gmu.to(G.DEV), y.to(G.DEV)
    win = f2d[r0:r0 + rows].contiguous()
    out = G.pixel_gemm(H, W, 0, C, C, 1, A2=win, a2_row0=r0, a2_rows=rows, B2=gsd, bias=gmud, mask=yd, row_lo=r0,
                       row_hi=r0 + rows)
    ref = torch.zeros(H, W, C)
    ref[r0:r0 + rows] = (f2[r0:r0 + rows].float().reshape(-1, C) @ gs.float().t()).reshape(rows, W, C) + gmu
    assert G.rel_err(out, ref) < 6e-3


@pytest.mark.parametrize('H,W', [(16, 16), (37, 70), (64, 130)])
def test_conv0_tv_forward_and_backward(G, H, W):
    g = torch.Generator().manual_seed(H * 1000 + W)
    img = torch.rand(1, 3, H, W, generator=g)
    w = O.make_vgg_weights(7)
    w0, b0 = w[0]
    out = torch.empty(H, W, 64, dtype=torch.bfloat16, device=G.DEV)
    gtv = torch.empty(3, H, W, device=G.DEV)
    parts = torch.zeros(((W + 63) // 64) * H, device=G.DEV)
    n = ctypes.c_int()
    img_d, w0_d, b0_d = img.to(G.DEV), w0.to(G.DEV), b0.to(G.DEV)
    G.check(G.lib().stb_test_conv0_fwd(G.P(img_d), G.P(w0_d), G.P(b0_d), G.P(out), H, W, 2.0, G.P(gtv), G.P(parts),
                                       ctypes.byref(n), G.S()))
    torch.cuda.synchronize()
    acts = O.vgg_forward(img, w, 'max', 1)
    assert G.rel_err(G.nchw(out), acts[1]) < 6e-3
    tvl, tvg = O.tv_loss_and_grad(img.double())
    assert abs(parts.sum().item() - tvl.item()) / tvl.item() < 1e-5
    assert G.rel_err(gtv[None], (tvg * 2.0).float()) < 1e-5
    g0 = (torch.randn(H, W, 64, generator=g) * (torch.rand(H, W, 64, generator=g) > 0.5)).bfloat16()
    grad = torch.empty(1, 3, H, W, device=G.DEV)
    g0_d = g0.to(G.DEV)
    G.check(G.lib().stb_test_conv0_bwd(G.P(g0_d), G.P(w0_d), None, G.P(grad), H, W, G.S()))
    torch.cuda.synchronize()
    acts0 = {1: torch.ones(1, 64, H, W, dtype=torch.float64)}  # mask already applied in g0
    ref = O.vgg_backward({1: G.nchw(g0).double()}, acts0, [(w0.double(), b0.double())], 'max')
    # interior pixels come from the wgmma dgrad with bf16 weights and a bf16 result (2^-9 relative), the border
    # ring (replicate-pad adjoint) is evaluated in fp32
    assert G.rel_err(grad, ref.float()) < 6e-3
    ring = torch.ones(1, 3, H, W, dtype=torch.bool)
    ring[:, :, 1:-1, 1:-1] = False
    assert G.rel_err(grad.cpu()[ring], ref.float()[ring]) < 1e-5


@pytest.mark.parametrize('H,W,C', [(16, 16, 64), (37, 21, 128), (2, 2, 512)])
@pytest.mark.parametrize('pooling', ['max', 'average', 'l2'])
def test_pool_backward(G, H, W, C, pooling):
    code = {'max': 0, 'average': 1, 'l2': 2}[pooling]
    g = torch.Generator().manual_seed(5)
    x = torch.relu(torch.randn(H, W, C, generator=g)).bfloat16()
    x[::3, ::2] = 0  # all-zero windows and ties
    go = torch.randn(H // 2, W // 2, C, generator=g).bfloat16()
    x_d, go_d = x.to(G.DEV), go.to(G.DEV)
    gin = torch.full((H, W, C), float('nan'), dtype=torch.bfloat16, device=G.DEV)
    G.check(G.lib().stb_test_pool_bwd(code, G.P(go_d), G.P(x_d), G.P(gin), H, W, C, G.S()))
    torch.cuda.synchronize()
    xin = G.nchw(x)
    gref = O.pool_bwd(G.nchw(go), xin, pooling) * (xin > 0)
    if pooling == 'max':
        assert torch.equal(G.nchw(gin).cpu(), gref)  # argmax routing (first maximum wins) is exact
    else:
        assert G.rel_err(G.nchw(gin), gref) < 5e-3


@pytest.mark.parametrize('P_,C', [(16, 512), (1000, 64), (4096, 128), (3001, 256), (5000, 512), (1, 64)])
def test_gram_and_sums(G, P_, C):
    g = torch.Generator().manual_seed(P_ + C)
    f = torch.relu(torch.randn(P_, C, generator=g)).bfloat16().to(G.DEV)
    nf = G.lib().stb_test_gram_partials_floats(P_, C)
    ws = torch.empty(nf, device=G.DEV)
    Sr = torch.empty(C, C, device=G.DEV)
    sm = torch.empty(C, device=G.DEV)
    G.check(G.lib().stb_test_gram(G.P(f), P_, C, G.P(ws), nf, G.P(Sr), G.P(sm), G.S()))
    torch.cuda.synchronize()
    fd = f.double().cpu()
    assert G.rel_err(Sr, (fd.t() @ fd).float()) < 2e-5   # fp32 accumulation of exact bf16 products
    assert G.rel_err(sm, fd.sum(0).float()) < 2e-5
    assert torch.equal(Sr.cpu(), Sr.cpu().t())            # symmetric by construction of the tile schedule


@pytest.mark.parametrize('C', [64, 128, 256, 512])
def test_w2_loss_sqrtm_and_backward(G, C):
    """fp32 W2 engine (cov, sqrtm_ns x12, Lyapunov backward x12) vs the oracle's restatement of ST:149-181/SQ:9-47."""
    g = torch.Generator().manual_seed(C)
    n = 4 * C

    def moments(scale):
        f = torch.relu(torch.randn(C, n, generator=g) * scale + 0.2)
        return f.mean(1), (f @ f.t()) / n

    mt, st = moments(1.0)
    mc, sc = moments(1.2)
    npix, weight = float(n), 0.37
    wsb = G.lib().stb_test_w2_workspace_bytes()
    ws = torch.empty(wsb, dtype=torch.uint8, device=G.DEV)
    loss = torch.zeros(1, device=G.DEV)
    gs = torch.empty(C, C, device=G.DEV)
    gmu = torch.empty(C, device=G.DEV)
    cs = torch.empty(C, C, device=G.DEV)
    keep = [mt.to(G.DEV), st.to(G.DEV), (sc * npix).to(G.DEV), (mc * npix).to(G.DEV)]
    G.check(G.lib().stb_test_w2(G.P(keep[0]), G.P(keep[1]), G.P(keep[2]), G.P(keep[3]), C, npix, weight, G.P(ws), wsb,
                                G.P(loss), G.P(gs), G.P(gmu), G.P(cs), G.S()))
    torch.cuda.synchronize()
    dt = torch.float64
    tgt = O.StyleTarget.build(mt.to(dt), st.to(dt))
    eye = torch.eye(C, dtype=dt)
    cov = sc.to(dt) - torch.outer(mc.to(dt), mc.to(dt)) + eye * 1e-4
    md = ((mc.to(dt) - tgt.mean) ** 2).mean()
    r = O.sqrtm_ns(tgt.cov_sqrt @ cov @ tgt.cov_sqrt, 12)
    l = (md + torch.diagonal(tgt.cov + cov - 2 * r).mean()) * weight
    g_m = O.sqrtm_ns_lyap_backward(r, eye * (-2.0 * weight / C), 12)
    g_cov = tgt.cov_sqrt.t() @ g_m @ tgt.cov_sqrt.t() + eye * (weight / C)
    gsr = g_cov + g_cov.t()
    gmr = 2.0 * weight * (mc.to(dt) - tgt.mean) / C - gsr @ mc.to(dt)
    assert G.rel_err(cs, tgt.cov_sqrt) < 1e-4
    assert abs(loss.item() - l.item()) / abs(l.item()) < 1e-3   # cancellation: fp32 vs fp64
    assert G.rel_err(gs, gsr) < 2e-3
    assert G.rel_err(gmu * npix, gmr) < 2e-3


@pytest.mark.parametrize('C,H,W,Ho,Wo', [(3, 96, 128, 136, 181), (3, 181, 136, 256, 192), (3, 64, 64, 64, 64),
                                         (3, 50, 70, 35, 49), (1, 17, 33, 24, 47)])
def test_native_resize_matches_interpolate(G, C, H, W, Ho, Wo):
    """stb_resize vs F.interpolate(align_corners=False) for the per-scale warm start (ST:285-295, 420): bicubic and
    bilinear, with the relu / clamp epilogues; the CPU kernels of torch are the yardstick (1e-6: same formulas, fp32)."""
    from style_transfer_b200 import _lib
    g = torch.Generator().manual_seed(C * H + W)
    x = torch.rand(1, C, H, W, generator=g) * 1.4 - 0.2
    xd = x.to(G.DEV)
    for mode, code in (('bilinear', 0), ('bicubic', 1)):
        want = F.interpolate(x, (Ho, Wo), mode=mode, align_corners=False)
        for post, fn in ((0, lambda t: t), (1, torch.relu), (2, lambda t: t.clamp(0, 1))):
            out = torch.empty(1, C, Ho, Wo, device=G.DEV)
            _lib.check(_lib.load().stb_resize(_lib.ptr(xd), C, H, W, _lib.ptr(out), Ho, Wo, code, post, _lib.cur_stream()))
            torch.cuda.synchronize()
            assert (out.cpu() - fn(want)).abs().max().item() < 2e-6, (mode, post)
