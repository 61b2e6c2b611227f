"""Shared helpers of the -m gpu parity tests (all calls go through the C-ABI of libstb200.so)."""
import ctypes

import torch

import style_transfer_b200 as stb
from style_transfer_b200 import _lib

DEV = torch.device('cuda:0')
U = 2.0 ** -24          # unit roundoff of fp32
TILE_H, TILE_W = 16, 8  # output pixels of one pixel-GEMM sub-tile (csrc/conv_tc.cu)


def lib():
    """libstb200_test.so: kernel-level hooks (include/stb200_test.h).  The product library is reached through the
    `style_transfer_b200` package (gpu_util.make_st / st.model.lib)."""
    return _lib.load_test()


P = _lib.ptr
S = _lib.cur_stream


def check(rc):
    _lib.check(rc, test_lib=True)


def rel_err(got, ref):
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    assert torch.isfinite(got).all(), 'non-finite values in the CUDA result'
    return ((got - ref).abs().max() / (ref.abs().max() + 1e-30)).item()


def nchw(x_hwc):
    return x_hwc.float().permute(2, 0, 1)[None]


def rn_bf16(x):
    """Round-to-nearest-even to bf16, as a float64 tensor.  Through fp32: both steps are monotone, which is all the
    window test below needs, and exact where x is an fp32 value."""
    return x.float().bfloat16().double()


def rn_window(got, ref, delta, relu=False):
    """True where `got` is what RN_bf16 gives somewhere in [ref - delta, ref + delta]: the kernel's fp32 value lies in
    that interval, and rounding is monotone, so RN of it lies between RN(ref - delta) and RN(ref + delta).  relu:
    the kernel rounds max(acc, 0), and RN commutes with max(., 0)."""
    lo, hi = rn_bf16(ref - delta), rn_bf16(ref + delta)
    if relu:
        lo, hi = lo.clamp_min(0), hi.clamp_min(0)
    return (got >= lo) & (got <= hi)


def rn_window_ratio(got, ref, delta, relu=False):
    """Largest |ref - b| / delta over the elements where got != RN(ref), b the rounding boundary between the two
    (<= 1 when the window test passes); 0 if every element is RN(ref)."""
    rn = rn_bf16(ref)
    off = got != rn
    if relu:
        off &= (got > 0) & (rn > 0)
    if not off.any():
        return 0.0
    return ((ref - (got + rn) / 2).abs() / delta)[off].max().item()


GRID_BITS = 6           # dyadic operands of the exact cases: k / 64, |k| <= 16


def integers(shape, lo, hi, gen):
    """Integers in [lo, hi] as bf16 (exact)."""
    return torch.randint(lo, hi + 1, shape, generator=gen, device=DEV).bfloat16()


def dyadic(shape, gen):
    """fp32 values k / 2^GRID_BITS, |k| <= 16: exact in bf16, so packing and staging keep them."""
    return torch.randint(-16, 17, shape, generator=gen, device=DEV).float() / 2 ** GRID_BITS


def check_exact(got, ref, mag, live):
    """got == RN_bf16(ref) on the live elements, for operands on the dyadic grid (integer activations, k / 2^g
    weights, biases and scales).  Every product, and every partial sum in any order, is then a multiple of 2^-g no
    larger than the magnitude M; with M 2^g < 2^24 all of them are fp32 values, so an fp32 accumulator (which the
    window bars already assume inside the tensor cores) is exact, and only the final RN to bf16 remains.  The case
    must exercise that rounding: some live references are not bf16 values, and some are ties (RN-even decides)."""
    assert mag.max().item() * 2 ** GRID_BITS < 2 ** 24, f'M = {mag.max().item()}: sums may not be exact in fp32'
    low = (ref[live].float().view(torch.int32) & 0xFFFF)     # the fp32 bits below the bf16 significand
    assert (low != 0).any(), 'no live reference needs rounding'
    assert (low == 0x8000).any(), 'no live reference is a rounding tie'
    bad = live & (got != rn_bf16(ref))
    assert not bad.any(), (f'{int(bad.sum())} of {int(live.sum())} live elements differ from RN_bf16(ref) (first at '
                           f'{bad.nonzero()[0].tolist()}: got {got[tuple(bad.nonzero()[0])].item()}, '
                           f'ref {ref[tuple(bad.nonzero()[0])].item()})')


def tiles(H, W, Cout):
    """CTA tiles of a whole-image pixel-GEMM launch, as launch_pixel_gemm counts them."""
    bn = 256 if Cout >= 256 else Cout
    mt = 1 if bn == 256 else 2
    return -(-H // TILE_H) * -(-W // (TILE_W * mt)) * (Cout // bn)


def pack(w, bwd):
    co, ci = w.shape[:2]
    out = torch.empty(9 * co * ci, dtype=torch.bfloat16, device=DEV)
    check(lib().stb_pack_weights(P(w), P(out), co, ci, int(bwd), S()))
    return out


def pixel_gemm(H, W, Cin, Cout, C2, mode, A=None, Bw=None, A2=None, a2_row0=0, a2_rows=0, B2=None, bias=None,
               mask=None, ctarget=None, cscale=0.0, row_lo=0, row_hi=1 << 30, out=None):
    """One launch of the 3x3 conv kernel; `out` (default: a new [H, W, Cout] tensor) is filled with NaN first."""
    if out is None:
        out = torch.empty((H, W, Cout), dtype=torch.bfloat16, device=DEV)
    out.fill_(float('nan'))
    check(lib().stb_test_pixel_gemm(H, W, Cin, Cout, C2, mode, P(A), P(Bw), P(A2), a2_row0, a2_rows, P(B2), P(out),
                                    P(bias), P(mask), P(ctarget), ctypes.c_float(cscale), row_lo, row_hi, S()))
    torch.cuda.synchronize()
    return out


def make_st(pooling, wts):
    return stb.StyleTransfer(devices=['cuda:0'], pooling=pooling, vgg_weights=wts)
