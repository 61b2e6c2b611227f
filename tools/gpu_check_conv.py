"""GPU bring-up check for the wgmma pixel-GEMM kernel.  Compares against torch fp32 conv2d
on bf16-rounded operands and times the VGG layer shapes at 2048^2.  Not a pytest file: prints diagnostics."""
import ctypes
import sys
import time
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parent.parent
lib = ctypes.CDLL(str(ROOT / 'style-transfer-pytorch_b200' / 'libstb200_test.so'))
lib.stb_test_last_error.restype = ctypes.c_char_p
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device('cuda:0')


def P(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def check(rc):
    if rc != 0:
        raise RuntimeError(f'rc={rc}: {lib.stb_test_last_error().decode()}')


def pack(w, bwd):
    co, ci = w.shape[:2]
    out = torch.empty(9 * co * ci, dtype=torch.bfloat16, device=dev)
    check(lib.stb_pack_weights(P(w), P(out), co, ci, int(bwd), stream()))
    return out


def pixel_gemm(H, W, Cin, Cout, C2, mode, A=None, Bw=None, A2=None, a2_row0=0, a2_rows=0, B2=None, bias=None,
               mask=None, ctarget=None, cscale=0.0, row_lo=0, row_hi=1 << 30, out=None):
    if out is None:
        out = torch.full((H, W, Cout), float('nan'), dtype=torch.bfloat16, device=dev)
    check(lib.stb_test_pixel_gemm(H, W, Cin, Cout, C2, mode, P(A), P(Bw), P(A2), a2_row0, a2_rows, P(B2), P(out),
                                  P(bias), P(mask), P(ctarget), ctypes.c_float(cscale), row_lo, row_hi, stream()))
    return out


def report(name, got, ref, tol=1.5e-2):
    got = got.float()
    err = (got - ref).abs()
    denom = ref.abs().max().item() + 1e-12
    bad = ~torch.isfinite(got)
    rel = (err.max() / denom).item() if not bad.any() else float('nan')
    ok = (not bad.any()) and rel < tol
    print(f'[{"OK " if ok else "BAD"}] {name}: max_abs_err={err.max().item():.4e} rel_to_max={rel:.3e} '
          f'nonfinite={int(bad.sum())} refmax={denom:.3e}', flush=True)
    if not ok:
        idx = torch.nonzero((err > tol * denom) | bad)
        print('   first bad idx (y,x,c):', idx[:8].tolist(), ' count', idx.shape[0], 'of', got.numel())
        if idx.shape[0]:
            i = tuple(idx[0].tolist())
            print('   got', got[i].item(), 'ref', ref[i].item())
    return ok


def nhwc_to_nchw(x):
    return x.float().permute(2, 0, 1)[None]


def test_fwd(H, W, Cin, Cout, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(H, W, Cin, device=dev, generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device=dev, generator=g) * (2.0 / (9 * Cin)) ** 0.5)
    b = torch.randn(Cout, device=dev, generator=g) * 0.1
    out = pixel_gemm(H, W, Cin, Cout, 0, 0, A=x, Bw=pack(w, False), bias=b)
    torch.cuda.synchronize()
    ref = F.relu(F.conv2d(nhwc_to_nchw(x), w.bfloat16().float(), b, padding=1))[0].permute(1, 2, 0)
    return report(f'fwd {H}x{W} {Cin}->{Cout}', out, ref)


def test_bwd(H, W, Cin, Cout, seed=1, with_c2=0, content=False, only_c2=False):
    """dgrad of a conv Cin->Cout: gout [H,W,Cout] -> gin [H,W,Cin], masked by y (activation feeding the conv)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    go = torch.randn(H, W, Cout, device=dev, generator=g).bfloat16()
    w = (torch.randn(Cout, Cin, 3, 3, device=dev, generator=g) * (2.0 / (9 * Cin)) ** 0.5)
    y = torch.relu(torch.randn(H, W, Cin, device=dev, generator=g)).bfloat16()
    ref = torch.zeros(H, W, Cin, device=dev)
    kw = {}
    if not only_c2:
        ref = F.conv_transpose2d(nhwc_to_nchw(go), w.bfloat16().float(), padding=1)[0].permute(1, 2, 0)
        kw.update(A=go, Bw=pack(w, True))
    if with_c2:
        f2 = torch.randn(H, W, with_c2, device=dev, generator=g).bfloat16()
        gs = (torch.randn(Cin, with_c2, device=dev, generator=g) * 0.05).bfloat16()
        gmu = torch.randn(Cin, device=dev, generator=g) * 0.1
        ref = ref + (f2.float().reshape(-1, with_c2) @ gs.float().t()).reshape(H, W, Cin) + gmu
        kw.update(A2=f2, B2=gs, bias=gmu)
    ct = None
    cs = 0.0
    if content:
        ct = torch.relu(torch.randn(H, W, Cin, device=dev, generator=g)).bfloat16()
        cs = 0.37
        ref = ref + cs * (y.float() - ct.float())
    ref = ref * (y.float() > 0)
    out = pixel_gemm(H, W, 0 if only_c2 else Cout, Cin, with_c2, 1, mask=y, ctarget=ct, cscale=cs, **kw)
    torch.cuda.synchronize()
    return report(f'bwd {H}x{W} {Cout}->{Cin} c2={with_c2} content={content} only_c2={only_c2}', out, ref)


def bench(H, W, Cin, Cout, iters=10):
    x = torch.randn(H, W, Cin, device=dev).bfloat16()
    w = torch.randn(Cout, Cin, 3, 3, device=dev) * 0.05
    b = torch.zeros(Cout, device=dev)
    wp = pack(w, False)
    out = torch.empty(H, W, Cout, dtype=torch.bfloat16, device=dev)
    for _ in range(3):
        pixel_gemm(H, W, Cin, Cout, 0, 0, A=x, Bw=wp, bias=b, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        pixel_gemm(H, W, Cin, Cout, 0, 0, A=x, Bw=wp, bias=b, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    fl = 2.0 * H * W * 9 * Cin * Cout
    by = H * W * (Cin + Cout) * 2
    print(f'bench {H}x{W} {Cin}->{Cout}: {ms:.3f} ms  {fl / ms / 1e9:.1f} TFLOP/s  {by / ms / 1e6:.1f} GB/s(algo)',
          flush=True)
    # cuDNN bf16 channels_last for context
    xc = nhwc_to_nchw(x).bfloat16().contiguous(memory_format=torch.channels_last)
    wc = w.bfloat16().contiguous(memory_format=torch.channels_last)
    for _ in range(3):
        F.conv2d(xc, wc, None, padding=1)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        F.conv2d(xc, wc, None, padding=1)
    e1.record()
    torch.cuda.synchronize()
    ms2 = e0.elapsed_time(e1) / iters
    print(f'      cudnn bf16 NHWC: {ms2:.3f} ms  {fl / ms2 / 1e9:.1f} TFLOP/s', flush=True)


if __name__ == '__main__':
    print(torch.cuda.get_device_name(0), flush=True)
    ok = True
    t0 = time.time()
    ok &= test_fwd(16, 8, 64, 64)
    ok &= test_fwd(32, 24, 64, 64)
    ok &= test_fwd(45, 34, 64, 128)
    ok &= test_fwd(33, 17, 128, 256)
    ok &= test_fwd(22, 22, 256, 512)
    ok &= test_fwd(37, 19, 512, 512)
    ok &= test_fwd(200, 300, 128, 128)
    ok &= test_bwd(32, 24, 64, 64)
    ok &= test_bwd(45, 34, 64, 128)
    ok &= test_bwd(22, 22, 256, 512)
    ok &= test_bwd(37, 19, 512, 512, with_c2=512)
    ok &= test_bwd(32, 24, 64, 64, with_c2=64, content=True)
    ok &= test_bwd(20, 12, 512, 512, with_c2=512, only_c2=True)
    print('correctness', 'PASS' if ok else 'FAIL', f'{time.time() - t0:.1f}s', flush=True)
    if '--bench' in sys.argv:
        bench(2048, 2048, 64, 64)
        bench(1024, 1024, 64, 128)
        bench(1024, 1024, 128, 128)
        bench(512, 512, 128, 256)
        bench(512, 512, 256, 256)
        bench(256, 256, 256, 512)
        bench(256, 256, 512, 512)
        bench(128, 128, 512, 512)
    sys.exit(0 if ok else 1)
