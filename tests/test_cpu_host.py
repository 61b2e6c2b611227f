"""-m "not gpu": host-side logic, the C-ABI library (loads + exports, no compute), the plain-C oracle."""
import ctypes
import re
import subprocess
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import st_oracle as O

ROOT = Path(__file__).resolve().parent.parent


def test_library_exports_every_declared_symbol():
    """libstb200.so exports exactly what include/stb200.h declares; the kernel-level test hooks live in a separate
    library (libstb200_test.so / include/stb200_test.h) and are NOT exported by the product."""
    import __graft_entry__ as ge
    ge.build()
    from style_transfer_b200 import _lib
    pat = r'STB_API\s+[\w\s\*]+?\b(stb_\w+)\s*\('
    declared = set(re.findall(pat, (ROOT / 'include' / 'stb200.h').read_text()))
    declared_test = set(re.findall(pat, (ROOT / 'include' / 'stb200_test.h').read_text()))
    assert len(declared) >= 20 and len(declared_test) >= 10
    lib = ctypes.CDLL(str(ROOT / 'style-transfer-pytorch_b200' / 'libstb200.so'))
    tlib = ctypes.CDLL(str(ROOT / 'style-transfer-pytorch_b200' / 'libstb200_test.so'))
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in stb200.h but not exported'
    for name in declared_test:
        assert hasattr(tlib, name), f'{name} declared in stb200_test.h but not exported by the test library'
        assert not hasattr(lib, name), f'test hook {name} leaked into the product library'
    assert declared == set(_lib.EXPORTS)
    assert declared_test == set(_lib.TEST_EXPORTS)
    out = subprocess.run(['nm', '-D', '--defined-only', str(ROOT / 'style-transfer-pytorch_b200' / 'libstb200.so')],
                         capture_output=True, text=True, check=True).stdout
    exported = {ln.split()[-1] for ln in out.splitlines() if ' T ' in ln and ln.split()[-1].startswith('stb_')}
    assert exported == declared, exported ^ declared


def test_product_does_not_touch_the_oracle():
    """The shipped path may not import, link or execute anything under oracle/."""
    for p in (ROOT / 'style-transfer-pytorch_b200').rglob('*'):
        if 'build' in p.relative_to(ROOT).parts[1:] or p.suffix not in ('.py', '.cu', '.cuh', '.h'):
            continue
        txt = p.read_text()
        assert not re.search(r'^\s*(from|import)\s+oracle', txt, re.M), p
        assert 'st_oracle' not in txt and 'libst_oracle' not in txt and 'reference_harness' not in txt, p


def test_no_cpu_fallback(monkeypatch):
    import torch
    import style_transfer_b200 as stb
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)   # a host without CUDA, also on a GPU machine
    with pytest.raises(RuntimeError):
        stb.StyleTransfer(devices=['cpu'])
    with pytest.raises(ValueError):
        stb.StyleTransfer(devices=['cuda:0', 'cuda:1', 'cuda:2'])


def test_stylize_signature_matches_reference_surface():
    """cli.py:150-153 scrapes defaults/annotations from stylize(); they must be the reference's (ST:349-363)."""
    import style_transfer_b200 as stb
    kw = stb.StyleTransfer.stylize.__kwdefaults__
    assert kw == dict(style_weights=None, content_weight=0.015, tv_weight=2., optimizer='adam', min_scale=128,
                      end_scale=512, iterations=500, initial_iterations=1000, step_size=0.02, avg_decay=0.99,
                      init='content', style_scale_fac=1., style_size=None, callback=None)
    ann = stb.StyleTransfer.stylize.__annotations__
    assert {k: (v if isinstance(v, str) else v.__name__) for k, v in ann.items()} == dict(
        content_weight='float', tv_weight='float', optimizer='str', min_scale='int', end_scale='int',
        iterations='int', initial_iterations='int', step_size='float', avg_decay='float', init='str',
        style_scale_fac='float', style_size='int')
    fields = [f for f in stb.STIterate.__dataclass_fields__]
    assert fields == ['w', 'h', 'i', 'i_max', 'loss', 'time', 'gpu_ram']


def test_scale_helpers_match_oracle():
    import style_transfer_b200 as stb
    for a, b in ((128, 512), (128, 2896), (64, 64), (300, 200)):
        assert stb.gen_scales(a, b) == O.gen_scales(a, b)
    for size in ((2896, 2172), (100, 50), (50, 100), (640, 480)):
        for dim in (128, 181, 512):
            for up in (False, True):
                assert stb.size_to_fit(size, dim, up) == O.size_to_fit(size, dim, up)


# ------------------------------------------------------------------ plain-C oracle vs the torch primitives
@pytest.fixture(scope='module')
def clib():
    subprocess.run(['make', '-C', str(ROOT / 'oracle')], check=True, capture_output=True)
    lib = ctypes.CDLL(str(ROOT / 'oracle' / 'libst_oracle_c.so'))
    return lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize('replicate', [0, 1])
def test_c_conv_matches_torch(clib, replicate):
    rng = np.random.default_rng(0)
    cin, cout, h, w = 5, 7, 9, 11
    x = rng.standard_normal((cin, h, w), dtype=np.float32)
    wt = rng.standard_normal((cout, cin, 3, 3), dtype=np.float32)
    b = rng.standard_normal(cout, dtype=np.float32)
    out = np.empty((cout, h, w), np.float32)
    clib.stc_conv3x3(_p(x), _p(wt), _p(b), _p(out), cin, cout, h, w, replicate, 1)
    xt = torch.from_numpy(x)[None]
    if replicate:
        ref = F.conv2d(F.pad(xt, (1, 1, 1, 1), mode='replicate'), torch.from_numpy(wt), torch.from_numpy(b))
    else:
        ref = F.conv2d(xt, torch.from_numpy(wt), torch.from_numpy(b), padding=1)
    np.testing.assert_allclose(out, torch.relu(ref)[0].numpy(), rtol=1e-4, atol=1e-5)
    # dgrad vs the oracle's manual backward
    g = rng.standard_normal((cout, h, w), dtype=np.float32)
    gin = np.empty((cin, h, w), np.float32)
    clib.stc_conv3x3_dgrad(_p(g), _p(wt), _p(gin), cin, cout, h, w, replicate)
    xt.requires_grad_()
    if replicate:
        y = F.conv2d(F.pad(xt, (1, 1, 1, 1), mode='replicate'), torch.from_numpy(wt))
    else:
        y = F.conv2d(xt, torch.from_numpy(wt), padding=1)
    y.backward(torch.from_numpy(g)[None])
    np.testing.assert_allclose(gin, xt.grad[0].numpy(), rtol=1e-4, atol=1e-5)


def test_c_pool_gram_sqrtm_adam_match_oracle(clib):
    rng = np.random.default_rng(1)
    c, h, w = 3, 7, 10
    x = rng.standard_normal((c, h, w), dtype=np.float32)
    x[:, :2, :2] = 0.5  # ties: first maximum wins
    out = np.empty((c, h // 2, w // 2), np.float32)
    clib.stc_maxpool2(_p(x), _p(out), c, h, w)
    xt = torch.from_numpy(x)[None]
    np.testing.assert_array_equal(out, O.pool_fwd(xt, 'max')[0].numpy())
    g = rng.standard_normal(out.shape, dtype=np.float32)
    gin = np.empty_like(x)
    clib.stc_maxpool2_bwd(_p(g), _p(x), _p(gin), c, h, w)
    np.testing.assert_array_equal(gin, O.pool_bwd(torch.from_numpy(g)[None], xt, 'max')[0].numpy())
    xr = xt.clone().requires_grad_()
    F.max_pool2d(xr, 2).backward(torch.from_numpy(g)[None])
    np.testing.assert_array_equal(gin, xr.grad[0].numpy())  # and ATen's own tie rule
    # gram / mean
    f = rng.standard_normal((6, 50), dtype=np.float32)
    mean, srm = np.empty(6, np.float32), np.empty((6, 6), np.float32)
    clib.stc_style_stats(_p(f), _p(mean), _p(srm), 6, 50)
    om, osr = O.style_stats(torch.from_numpy(f).reshape(1, 6, 5, 10))
    np.testing.assert_allclose(mean, om.numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(srm, osr.numpy(), rtol=1e-5, atol=1e-6)
    # sqrtm_ns + lyapunov backward
    n = 12
    a = rng.standard_normal((n, 3 * n)).astype(np.float32)
    a = (a @ a.T / (3 * n) + 0.1 * np.eye(n)).astype(np.float32)
    r = np.empty_like(a)
    clib.stc_sqrtm_ns(_p(a), _p(r), n, 12)
    ro = O.sqrtm_ns(torch.from_numpy(a), 12)
    np.testing.assert_allclose(r, ro.numpy(), rtol=1e-4, atol=1e-5)
    go = rng.standard_normal((n, n)).astype(np.float32)
    gi = np.empty_like(a)
    clib.stc_sqrtm_lyap_bwd(_p(r), _p(go), _p(gi), n, 12)
    np.testing.assert_allclose(gi, O.sqrtm_ns_lyap_backward(ro, torch.from_numpy(go), 12).numpy(), rtol=2e-3, atol=1e-5)
    # adam + clamp + ema, three steps against torch.optim.Adam
    xs = rng.random(100).astype(np.float32)
    p = torch.nn.Parameter(torch.from_numpy(xs.copy()))
    opt = torch.optim.Adam([p], lr=0.02, betas=(0.9, 0.99))
    m, v, ema = np.zeros(100, np.float32), np.zeros(100, np.float32), (xs * 0.01).astype(np.float32)
    ema_t = torch.from_numpy(ema.copy())
    for step in range(1, 4):
        gr = rng.standard_normal(100).astype(np.float32)
        clib.stc_adam_clamp_ema(_p(xs), _p(gr), _p(m), _p(v), _p(ema), ctypes.c_long(100), step, ctypes.c_float(0.02),
                                ctypes.c_float(0.9), ctypes.c_float(0.99), ctypes.c_float(1e-8), ctypes.c_float(0.99))
        p.grad = torch.from_numpy(gr.copy())
        opt.step()
        with torch.no_grad():
            p.clamp_(0, 1)
            ema_t = ema_t * 0.99 + 0.01 * p
        np.testing.assert_allclose(xs, p.detach().numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(ema, ema_t.numpy(), rtol=1e-5, atol=1e-6)


def test_oracle_pool_variants_match_torch_modules():
    """Scale(AvgPool2d(2),2.0) and Scale(LPPool2d(2,2),0.78) forward/backward vs autograd (ST:21-22, 41-46)."""
    x = torch.rand(1, 4, 7, 9) + 0.1
    x[0, 0, :2, :2] = 0
    g = torch.randn(1, 4, 3, 4)
    for name, mod, scale in (('average', torch.nn.AvgPool2d(2), 2.0), ('l2', torch.nn.LPPool2d(2, 2), 0.78)):
        xr = x.clone().requires_grad_()
        y = mod(xr) * scale
        y.backward(g)
        np.testing.assert_allclose(O.pool_fwd(x, name).numpy(), y.detach().numpy(), rtol=1e-5, atol=1e-6)
        ref = torch.nan_to_num(xr.grad, nan=0.0)
        np.testing.assert_allclose(O.pool_bwd(g, x, name).numpy(), ref.numpy(), rtol=1e-4, atol=1e-6)


def test_async_image_writer_saves_newest_snapshot(tmp_path):
    """SURVEY.md section 8f row 3: periodic saves go through a worker thread; newest snapshot wins, files are whole."""
    import numpy as np
    from PIL import Image
    from style_transfer_b200 import image_io
    w = image_io.AsyncImageWriter()
    out = tmp_path / 'out.png'
    for k in range(5):
        w.submit_array(np.full((32, 48, 3), 40 * k, dtype=np.uint8), out)
    other = tmp_path / 'other.png'
    w.submit_array(np.zeros((8, 8, 3), dtype=np.uint8), other)
    w.close()
    img = np.asarray(Image.open(out))
    assert img.shape == (32, 48, 3) and int(img[0, 0, 0]) == 160
    assert other.exists() and not list(tmp_path.glob('*.part*'))
