"""-m gpu: the 3x3 conv kernel's forward (MODE 0: + bias, ReLU) and its pre-pool dgrad (MODE 2: no bias, no mask)
element by element against a float64 evaluation on the same bf16 operands, on whole images.

The references run on the device in float64 (ATen / cuDNN double kernels, independent of this library): F.conv2d for
the forward, F.conv_transpose2d for the dgrad, on the bf16-rounded operands; the weights reach the kernel through
the library's own packing (stb_pack_weights), so the packing and the dgrad's tap rotation are tested with it.  M is
the same convolution on absolute values.  Every output is filled with NaN before a call and allocated with one
extra NaN row after the tensor, which must stay NaN: the TMA store boxes must clip at the ragged bottom and right
edges.  The forward is checked both alone and with each fused 2x2 pool (stb_test_conv_pool), whose epilogue reads
the staging buffer between the store of `out` and its commit.

Bars (u = 2^-24, the fp32 unit roundoff; K = 9 * Cin products of bf16 operands, exact in fp32; the tensor cores add
them in some order, each addition losing at most 2 u of a partial sum no larger than M):
  MODE 0  v = (sum of K products) + bias, ReLU, RN to bf16:  delta = 2 u (K + 4) (M + |bias|), rn_window(relu=True)
  MODE 2  v = sum of K products, RN to bf16:                 delta = 2 u (K + 2) M,            rn_window
That window is wider than one bf16 ulp for many elements at large K, so every case also runs on exactly summable
operands (gpu_util.check_exact), where the output must be RN_bf16(reference) bit for bit.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

POOLINGS = {'max': 0, 'average': 1, 'l2': 2}

# (name, mode, H, W, channels of A, Cout, also with each fused pool): the production (Cin, Cout) pairs of the VGG-19
# trunk at shapes where every CTA walks three or more tiles (test_every_cta_walks_three_tiles)
BIG = [
    ('fwd_64_64_pool', 0, 317, 323, 64, 64, True),
    ('fwd_64_128', 0, 317, 323, 64, 128, False),
    ('fwd_128_128_pool', 0, 317, 323, 128, 128, True),
    ('fwd_128_256', 0, 317, 165, 128, 256, False),
    ('fwd_256_256_pool', 0, 317, 165, 256, 256, True),
    ('fwd_256_512', 0, 161, 150, 256, 512, False),
    ('fwd_512_512_pool', 0, 161, 150, 512, 512, True),
    ('dgrad_128_64', 2, 317, 323, 128, 64, False),
    ('dgrad_256_128', 2, 317, 323, 256, 128, False),
    ('dgrad_512_256', 2, 317, 165, 512, 256, False),
    ('dgrad_512_512', 2, 161, 150, 512, 512, False),
]
# small and ragged launches: single tiles, partial sub-tiles, H < 16 and W < 8, one-column second sub-tiles (W = 9)
SMALL = [
    ('fwd_16x8', 0, 16, 8, 64, 64, False),
    ('fwd_32x24_pool', 0, 32, 24, 64, 64, True),
    ('fwd_45x34', 0, 45, 34, 64, 128, False),
    ('fwd_37x21_pool', 0, 37, 21, 64, 128, True),
    ('fwd_33x17', 0, 33, 17, 128, 256, False),
    ('fwd_18x50_pool', 0, 18, 50, 128, 256, True),
    ('fwd_22x22', 0, 22, 22, 256, 512, False),
    ('fwd_37x19', 0, 37, 19, 512, 512, False),
    ('fwd_6x6_pool', 0, 6, 6, 512, 512, True),
    ('fwd_1x1', 0, 1, 1, 512, 512, False),
    ('fwd_200x300', 0, 200, 300, 128, 128, False),
    ('fwd_11x6', 0, 11, 6, 128, 128, False),
    ('fwd_20x9', 0, 20, 9, 64, 128, False),
    ('fwd_19x9_bn256', 0, 19, 9, 256, 256, False),
    ('fwd_17x40', 0, 17, 40, 256, 256, False),
    ('fwd_2x3_pool', 0, 2, 3, 64, 64, True),
    ('dgrad_45x34', 2, 45, 34, 256, 128, False),
    ('dgrad_11x6', 2, 11, 6, 128, 64, False),
    ('dgrad_17x9', 2, 17, 9, 512, 256, False),
    ('dgrad_1x1', 2, 1, 1, 512, 512, False),
]
CASES = BIG + SMALL


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return g


def test_every_cta_walks_three_tiles(G):
    """The tile loop (ring phases and accumulators carried across tiles) only runs when a CTA gets several tiles:
    fails on a device with more SMs than these shapes were planned for, rather than testing less."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for name, _, H, W, _, Cout, _ in BIG:
        assert G.tiles(H, W, Cout) // sms >= 3, f'{name}: {G.tiles(H, W, Cout)} tiles on {sms} SMs'


def operands(G, seed, mode, H, W, Cin, Cout, grid):
    """Input activation (forward: nonnegative, as the ReLU'd layers feed it; dgrad: signed), fp32 weights in the
    layout the packer takes (forward [Cout][Cin][3][3], dgrad the forward conv's [Cin][Cout][3][3]) and the bias."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    lo = 0 if mode == 0 else -3
    if grid:
        x = G.integers((H, W, Cin), lo, 3, gen)
        w = G.dyadic((Cout, Cin, 3, 3) if mode == 0 else (Cin, Cout, 3, 3), gen)
        b = G.dyadic((Cout,), gen)
    else:
        x = torch.randn(H, W, Cin, generator=gen, device=G.DEV)
        x = (torch.relu(x) if mode == 0 else x).bfloat16()
        w = torch.randn((Cout, Cin, 3, 3) if mode == 0 else (Cin, Cout, 3, 3), generator=gen, device=G.DEV)
        w *= (2.0 / (9 * Cin)) ** 0.5
        b = torch.randn(Cout, generator=gen, device=G.DEV) * 0.1
    return x, w, b


def reference(mode, x, w, b):
    """Pre-activation (forward: with the bias) in float64 and its magnitude M (+ |bias|), both [H, W, Cout]."""
    x64, w64 = x.double().permute(2, 0, 1)[None], w.bfloat16().double()
    if mode == 0:
        ref = F.conv2d(x64, w64, b.double(), padding=1)
        mag = F.conv2d(x64.abs(), w64.abs(), b.double().abs(), padding=1)
    else:
        ref = F.conv_transpose2d(x64, w64, padding=1)
        mag = F.conv_transpose2d(x64.abs(), w64.abs(), padding=1)
    return ref[0].permute(1, 2, 0), mag[0].permute(1, 2, 0)


def launches(G, mode, H, W, Cin, Cout, x, wp, b, pool):
    """(label, out) of the plain launch and, with pool, of the three fused-pool launches; checks the guard rows."""
    nan = float('nan')
    buf = torch.full((H + 1, W, Cout), nan, dtype=torch.bfloat16, device=G.DEV)
    G.pixel_gemm(H, W, Cin, Cout, 0, mode, A=x, Bw=wp, bias=b if mode == 0 else None, out=buf[:H])
    assert torch.isnan(buf[H]).all(), 'the plain launch wrote the row after the output'
    yield 'plain', buf[:H]
    if not pool:
        return
    for pooling, code in POOLINGS.items():
        buf = torch.full((H + 1, W, Cout), nan, dtype=torch.bfloat16, device=G.DEV)
        pbuf = torch.full((H // 2 + 1, W // 2, Cout), nan, dtype=torch.bfloat16, device=G.DEV)
        G.check(G.lib().stb_test_conv_pool(H, W, Cin, Cout, G.P(x), G.P(wp), G.P(b), G.P(buf), G.P(pbuf), code, G.S()))
        torch.cuda.synchronize()
        assert torch.isnan(buf[H]).all(), f'{pooling} pool: the launch wrote the row after the output'
        assert torch.isnan(pbuf[H // 2]).all(), f'{pooling} pool: the launch wrote the row after the pooled output'
        assert not torch.isnan(pbuf[:H // 2]).any(), f'{pooling} pool: pooled elements not written'
        yield f'{pooling} pool', buf[:H]


def run(G, name, mode, H, W, Cin, Cout, pool, grid):
    seed = (H * 1000 + W) * 7 + Cin + Cout + mode + grid
    x, w, b = operands(G, seed, mode, H, W, Cin, Cout, grid)
    ref, mag = reference(mode, x, w, b)
    K = 9 * Cin
    relu = mode == 0
    delta = 2 * G.U * (K + (4 if mode == 0 else 2)) * mag
    wp = G.pack(w, mode == 2)
    ratios = []
    for label, out in launches(G, mode, H, W, Cin, Cout, x, wp, b, pool):
        got = out.double()
        if grid:
            G.check_exact(got, ref.clamp_min(0) if relu else ref, mag, torch.ones_like(got, dtype=torch.bool))
            continue
        ok = G.rn_window(got, ref, delta, relu=relu)
        bad = ~ok
        assert ok.all(), (f'{label}: {int(bad.sum())} of {ok.numel()} elements outside the RN window (first at '
                          f'{bad.nonzero()[0].tolist()}: got {got[tuple(bad.nonzero()[0])].item()}, '
                          f'ref {ref[tuple(bad.nonzero()[0])].item()})')
        ratios.append(G.rn_window_ratio(got, ref, delta, relu=relu))
    if not grid:
        print(f'RATIO pixel_gemm {name} ' + ' '.join(f'{r:.3g}' for r in ratios))


@pytest.mark.parametrize('name,mode,H,W,Cin,Cout,pool', CASES, ids=[c[0] for c in CASES])
def test_pixel_gemm_elementwise(G, name, mode, H, W, Cin, Cout, pool):
    run(G, name, mode, H, W, Cin, Cout, pool, grid=False)


@pytest.mark.parametrize('name,mode,H,W,Cin,Cout,pool', CASES, ids=[c[0] for c in CASES])
def test_pixel_gemm_exact_on_dyadic_grid(G, name, mode, H, W, Cin, Cout, pool):
    run(G, name, mode, H, W, Cin, Cout, pool, grid=True)
