"""-m gpu: the dgrad epilogue of the 3x3 conv kernel (MODE 1: + gmu on the own rows, + the content term, * (y > 0))
element by element against a float64 evaluation on the same bf16 operands.

The epilogue takes the ReLU mask y and the content target from shared memory: either streamed per output tile and
64-channel chunk through the A ring, or, on the 64- and 128-channel style taps whose tap operand A2 IS the mask,
from the A2 chunks the tap-gradient GEMM has just used.  The cases below cover both paths at every BN, with ragged
right and bottom edges, and a band-style A2 row window where the kernel must stream the mask although A2 is a view
of it.  Each output is filled with NaN before the call (gpu_util.pixel_gemm).

Bar of an element whose mask is > 0 (u = 2^-24, the fp32 unit roundoff): the kernel's fp32 value is
    v = ((sum of K products) + gmu) + cscale * (y - t),   K = 9 * (channels of A) + C2,
the products of bf16 operands are exact in fp32; the tensor cores add them in some order, each addition losing at
most 2 u (truncating, not rounding) of a partial sum no larger than M = sum |a b|; the bias, the difference, the
product with cscale and the last sum are four more roundings of values bounded by M + |gmu| + |cscale| (|y| + |t|).
So |v - ref| <= delta = 2 u (K + 4) (M + |gmu| + |cscale| (|y| + |t|)), and the stored bf16 must be what
round-to-nearest gives somewhere in [ref - delta, ref + delta] (rn_window).  An element whose mask is <= 0 must be
exactly 0.

Every case runs a second time on exactly summable operands (gpu_util.check_exact: integer gradients, masks and
content targets, dyadic weights, Gs, gmu and cscale), where the live outputs must be RN_bf16(ref) bit for bit: the
window above is wider than one bf16 ulp for many elements at K = 4608, so it cannot see a wrong rounding mode.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return g


# (name, H, W, channels of A (0: none), Cout, C2, A2 source ('mask', 'other' or None), content target)
CASES = [
    ('bn64_reuse', 317, 323, 64, 64, 64, 'mask', False),
    ('bn128_reuse', 317, 323, 128, 128, 128, 'mask', False),
    ('bn128_reuse_content', 317, 323, 128, 128, 128, 'mask', True),
    ('bn128_c2_not_mask', 317, 323, 128, 128, 128, 'other', False),
    ('bn64_no_c2', 317, 323, 128, 64, 0, None, False),
    ('bn256_c2', 317, 165, 256, 256, 256, 'mask', False),
    ('bn256_two_ntiles_c2_content', 161, 150, 512, 512, 512, 'mask', True),
    ('bn256_two_ntiles_no_c2', 161, 150, 256, 512, 0, None, False),
]


def test_every_cta_walks_three_tiles(G):
    """The tile loop (ring phases carried across tiles, slots held over a tile boundary) only runs when a CTA gets
    several tiles: fails on a device with more SMs than these shapes were planned for, rather than testing less."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for name, H, W, _, Cout, *_ in CASES:
        assert G.tiles(H, W, Cout) // sms >= 3, f'{name}: {G.tiles(H, W, Cout)} tiles on {sms} SMs'
    assert G.tiles(*APRON[:2], APRON[3]) // sms >= 3


def run_case(G, seed, H, W, Cin, Cout, C2, a2_src, content, a2_row0=0, a2_rows=0, row_lo=0, row_hi=1 << 30,
             grid=False):
    """grid: operands on the dyadic grid (gpu_util.check_exact) and a bit-exact check instead of the RN window."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    dev = G.DEV

    def act(C, lo=-3):        # activations, gradients and the mask: bf16 randn, or integers in [lo, 3]
        if grid:
            return G.integers((H, W, C), lo, 3, gen)
        x = torch.randn(H, W, C, generator=gen, device=dev)
        return (torch.relu(x) if lo == 0 else x).bfloat16()

    def small(shape, scale):  # weights, Gs, gmu: scaled randn, or dyadic
        return G.dyadic(shape, gen) if grid else torch.randn(shape, generator=gen, device=dev) * scale

    y = act(Cout)                                                              # mask: about half <= 0
    ref = torch.zeros(H, W, Cout, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(ref)
    kw = {}
    K = 0
    if Cin:
        go = act(Cin)
        w = small((Cin, Cout, 3, 3), (2.0 / (9 * Cin)) ** 0.5)
        g64, w64 = go.double().permute(2, 0, 1)[None], w.bfloat16().double()
        ref += F.conv_transpose2d(g64, w64, padding=1)[0].permute(1, 2, 0)
        mag += F.conv_transpose2d(g64.abs(), w64.abs(), padding=1)[0].permute(1, 2, 0)
        kw.update(A=go, Bw=G.pack(w, True))
        K += 9 * Cin
    rows = slice(max(row_lo, 0), min(row_hi, H))
    gmu = torch.zeros(Cout, device=dev)
    if C2:
        f2 = y if a2_src == 'mask' else act(C2)
        gs = small((Cout, C2), 0.05).bfloat16()
        gmu = small((Cout,), 0.1)
        r0, nr = a2_row0, a2_rows or H
        win = f2[r0:r0 + nr]                       # a view: A2 is the mask's rows r0.. when a2_src == 'mask'
        ref[r0:r0 + nr] += (win.double().reshape(-1, C2) @ gs.double().t()).reshape(nr, W, Cout)
        mag[r0:r0 + nr] += (win.double().abs().reshape(-1, C2) @ gs.double().abs().t()).reshape(nr, W, Cout)
        kw.update(A2=win, a2_row0=a2_row0, a2_rows=a2_rows, B2=gs, bias=gmu)
        K += C2
    ref[rows] += gmu.double()
    mag[rows] += gmu.double().abs()
    cs = 0.0
    if content:
        ct = act(Cout, lo=0)
        cs = 0.375 if grid else 0.37
        ref[rows] += cs * (y[rows].double() - ct[rows].double())
        mag[rows] += cs * (y[rows].double().abs() + ct[rows].double().abs())
        kw.update(ctarget=ct)
    out = G.pixel_gemm(H, W, Cin, Cout, C2, 1, mask=y, cscale=cs, row_lo=row_lo, row_hi=row_hi, **kw)
    got = out.double()
    live = y > 0
    dead_bad = live.logical_not() & (got != 0)
    assert not dead_bad.any(), (f'{int(dead_bad.sum())} masked elements are not 0 '
                                f'(first at {dead_bad.nonzero()[0].tolist()})')
    if grid:
        G.check_exact(got, ref, mag, live)
        return None
    delta = 2 * G.U * (K + 4) * mag
    bad = live & ~G.rn_window(got, ref, delta)
    assert not bad.any(), (f'{int(bad.sum())} of {int(live.sum())} live elements outside the RN window '
                           f'(first at {bad.nonzero()[0].tolist()}: got {got[tuple(bad.nonzero()[0])].item()}, '
                           f'ref {ref[tuple(bad.nonzero()[0])].item()})')
    return G.rn_window_ratio(torch.where(live, got, 0), torch.where(live, ref, 0), delta)


@pytest.mark.parametrize('name,H,W,Cin,Cout,C2,a2_src,content', CASES, ids=[c[0] for c in CASES])
def test_dgrad_epilogue_elementwise(G, name, H, W, Cin, Cout, C2, a2_src, content):
    r = run_case(G, H * 1000 + W + Cin + C2 + content, H, W, Cin, Cout, C2, a2_src, content)
    print(f'RATIO dgrad_epilogue {name} {r:.3g}')


@pytest.mark.parametrize('name,H,W,Cin,Cout,C2,a2_src,content', CASES, ids=[c[0] for c in CASES])
def test_dgrad_epilogue_exact_on_dyadic_grid(G, name, H, W, Cin, Cout, C2, a2_src, content):
    run_case(G, H * 1000 + W + Cin + C2 + content + 1, H, W, Cin, Cout, C2, a2_src, content, grid=True)


# a band computing its aprons: the output covers the whole local image, A2 (a view of the mask) only the own rows
APRON = (317, 323, 64, 64, 80, 150)


def test_dgrad_epilogue_apron_window_streams_the_mask(G):
    """A2 is the mask's rows [r0, r0 + rows), the launch computes all H rows: outside the window the kernel must take
    the mask from the mask tensor (the A2 box is zero-filled there), inside it adds gmu and the tap gradient."""
    H, W, Cin, C, r0, nr = APRON
    r = run_case(G, 11, H, W, Cin, C, C, 'mask', False, a2_row0=r0, a2_rows=nr, row_lo=r0, row_hi=r0 + nr)
    print(f'RATIO dgrad_epilogue apron {r:.3g}')


def test_dgrad_epilogue_apron_window_exact_on_dyadic_grid(G):
    H, W, Cin, C, r0, nr = APRON
    run_case(G, 12, H, W, Cin, C, C, 'mask', False, a2_row0=r0, a2_rows=nr, row_lo=r0, row_hi=r0 + nr, grid=True)
