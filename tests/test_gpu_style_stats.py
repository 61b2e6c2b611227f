"""-m gpu: the Gram and W2 kernels at the shapes and on the inputs the iteration gives them.

Gram (gram_tc.cu), at the production pixel count of every style tap at 512^2, 2048^2 and 4096^2 and on ragged counts,
against F^T F and the channel sums in fp64 (products of bf16 values are exact in fp64, so the reference is exact to
~P 2^-53).  Inputs are post-ReLU bf16 features (about half zeros, channel scales 2^-6 .. 2^6, dead and constant
channels), plus one signed case and one band window read through an offset pointer with NaN rows around it.

Per-element bar |got - ref| <= gamma * sum_p |f_pi| |f_pj|, gamma from the launcher's own arithmetic (mirrored below as
test_gpu_image_kernels.py mirrors its launchers' grids):
  - 32 k-steps x 2^-22 = 2^-17: a chunk of at most 32 k-steps (GCfg::CHUNK_STAGES stages) in one MMA accumulator, 2 ulps
    (2^-22 relative to the running sum) per k-step for the truncating accumulate and the alignment inside the
    instruction;
  - 2^-24 per round-to-nearest add of a chunk into `tot`: ceil(stages per split / CHUNK_STAGES) adds;
  - 2^-24 per add of gram_reduce_kernel's fixed order: a partial passes through at most ceil(n_splits / 16) + 4 adds
    (its accumulator, two tree levels per split lane, two in the final combine); n_splits + 4 is allowed.
The channel sums get the same bar with sum_p |f_pi|.

Bias bar: on the nonnegative cases every product is >= 0, so every truncation loses.  The only truncating sums are the
chunks: each loses at most 32 k-steps x 2^-22 = 2^-17 of its own sum, and the RN adds after them are unbiased, so with the
drain the mean of (got - ref) / ref over all nonzero elements is bounded in magnitude by 2^-17 = 7.6e-6.  One
accumulator per split instead loses ~n_k 2^-24.5 over n_k k-steps: ~4e-5 at 2048^2 (2000 k-steps per split on relu1_1),
~1.7e-4 at 4096^2.

W2 (w2_tc.cu), all five layers through the same grouped rounds (stb_test_w2_layers), with the production weights 256,
64, 16, 4, 1 (/341), on the statistics of a real iterate at 128^2, 256^2, 512^2 and 2048^2 (rank-deficient: relu5_1 has
64 pixels at 128^2) and on one synthetic set with dead and duplicated channels.  References: the oracle's
StyleTarget.build / sqrtm_ns / sqrtm_ns_lyap_backward chain on the same fp32 inputs, once in fp64 and once in fp32 on the
CPU with a fixed thread count; the second gives the noise floor e32 of an fp32 evaluation of the same chain.  e32 is the
largest error of N_ORDERS = 4 such evaluations, on the channels in the given order and in three random orders (every
quantity is invariant under a channel permutation, the summation order of every product is not): the error of a scalar
from one fp32 evaluation is one sample of a sum of signed roundings and can be far below its typical size (measured:
2.3e-7 for the relu2_1 loss term at 2048^2, where the other sizes gave 3e-6 ... 2e-5).  Per layer,
loss term, Gs, sqrt(cov_t) and gmu must be within max(16 e32, 2^-20) of fp64 (relative, Frobenius for matrices and
vectors).  16 = 2^-22 / 2^-24 x 4: the engine's unit is 2^-22 (the dropped lo*lo term, the TF32 and fp16 roundings of
lo) where fp32 has 2^-24, and 4 is headroom.  At 2048^2 every loss term must also be within 3e-4 of fp64 (the claim of
the w2_tc.cu header).  Exact checks: gs_bf16 == RN_bf16(fp32(Gs * fp32(1/npix))), Gs == Gs^T, and w2_gmu_kernel alone
against fp64 on the engine's own Gs and mu.  Bit identity: two forward_backward calls against one, targets built on other
statistics and reused, and one launch per round (STB_W2_CHAIN=0, in a subprocess: the variable is read once per
process) against the cooperative chain.

Measured on an NVIDIA H100 80GB HBM3 (400 W limit); the whole file runs in ~25 s there and allocates at most ~2.7 GiB
for its own inputs (4096^2 relu1_1: 2 GiB of bf16 features plus a 512 MiB fp64 chunk), ~4.5 GiB for the 2048^2 context:
  - Gram, 35 launches: max |got - ref| / (gamma sum |f_pi| |f_pj|) = 0.093 (signed case; 0.075 on the nonnegative ones,
    0.023 ... 0.034 at 2048^2 / 4096^2 on relu1_1 and relu2_1); channel sums 0.013.  Mean relative error (bias)
    -2.9e-7 ... -1.3e-8 against the bar 7.6e-6, channel sums within 2.2e-8.
  - W2, 25 layer problems: kernel error / bar at most 0.82 for the loss terms (relu2_1 at 512^2: 4.9e-5 against fp64,
    e32 3.7e-6), 0.11 for Gs, 0.14 for sqrt(cov_t), 0.17 for gmu.  Largest errors against fp64: loss 3.7e-4 (relu1_1
    at 128^2), Gs 3.2e-5, sqrt(cov_t) 2.1e-5, gmu 1.6e-4.  At 2048^2 the loss terms are within 2.4e-4 of fp64 (bar
    3e-4).  w2_gmu_kernel alone: at most 0.10 of its bar.  gs_bf16, the symmetry of Gs and all three bit identities
    hold exactly.
Hand-made mutations (not committed) and the tests of this file each one failed:
  1. Gram, one accumulator per split (CHUNK_STAGES = 2^30, no drain): the production counts relu1_1, relu2_1, relu3_1
     at 2048^2 and 4096^2 and relu4_1 at 4096^2 (per-element error up to 10.7 gamma at 4096^2 relu1_1; at 2048^2
     relu2_1 the bias bar, -1.1e-5 against 7.6e-6) and the signed case.  Of the rest of the suite only the 1024^2
     geometry of test_gpu_tiled_gradient.py fails, indirectly: the band-local chains are shorter, so the tiled and the
     untiled relu1_1 statistics drift apart (1.5e-5 against 1.5e-6); no kernel-level test there sees it.
  2. Gram, lower-triangle tiles read at their stored position in gram_reduce_kernel (C >= 256): every C >= 256 Gram
     case (production, ragged, signed, band window) and the W2 test on real statistics (24 tests).
  3. Gram, the last split stops one stage early: 41 of the 43 tests, every one that launches the Gram kernel (all Gram
     tests and every W2 test on real statistics).
  4. W2, the hi*hi product only (cross terms dropped): test_w2_five_layers_against_fp64 in all five cases (loss terms
     off by up to 7.6e-2, Gs by 5e-2).
  5. W2, the Gc-round gamma of layers 3 and 4 swapped: test_w2_five_layers_against_fp64 in all five cases (Gs of
     relu4_1 / relu5_1 off by 0.5 ... 3.2, gmu by 0.45 ... 7.9); the loss terms are unchanged.
  6. W2, gs_bf16 written without the 1/N: the bit-exact gs_bf16 check in all five cases.
  7. W2, gs_bf16 rounded toward zero (__float2bfloat16_rz): the bit-exact gs_bf16 check in all five cases.  The whole
     rest of the -m gpu suite passes with it.  Of 1-6 only 1 and 5 were run against the rest of the suite: 1 fails it
     as described above, 5 fails test_gpu_kernels.py's W2 test at C = 512 and end-to-end tests of test_gpu_iterate.py
     and test_gpu_lbfgs.py.
"""
import ctypes
import math
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import pytest
import torch

from style_transfer_b200 import _lib
from style_transfer_b200.style_transfer import NativeVGG, gen_scales
from oracle import st_oracle as O

pytestmark = pytest.mark.gpu

DEV = torch.device('cuda:0')
ROOT = Path(__file__).resolve().parent.parent
STYLE_C = [64, 128, 256, 512, 512]
STYLE_WEIGHTS = [w / 341 for w in (256, 64, 16, 4, 1)]
TAPS = ['relu1_1', 'relu2_1', 'relu3_1', 'relu4_1', 'relu5_1']   # pyramid level l: (H >> l) x (W >> l) pixels


def _tlib():
    return _lib.load_test()


def _check(rc):
    _lib.check(rc, test_lib=True)


def _sms():
    return torch.cuda.get_device_properties(DEV).multi_processor_count


# ---------------------------------------------------------------------------------------------- Gram: launch mirror
def _pk(C):            # gram_pk: pixels per pipeline stage
    return 256 if C == 64 else (128 if C == 128 else 64)


def _chunk_stages(C):  # GCfg::CHUNK_STAGES: stages per 32-k-step accumulator chunk (16 pixels per k-step)
    return 32 // (_pk(C) // 16)


def _tiles(C):         # gram_tiles: one tile row for C <= 128, upper-triangle 128 x 128 tiles otherwise
    t = C // 128
    return 1 if C < 256 else t * (t + 1) // 2


def _want_splits(C, sms):  # gram_want_splits: one CTA per SM
    return min(max(-(-sms // _tiles(C)), 1), 1024)


def _splits(P, C, sms):
    """gram_num_splits and the stages per split of launch_gram"""
    chunks = -(-P // _pk(C))
    want = max(min(_want_splits(C, sms), chunks), 1)
    per = -(-chunks // want)
    return -(-chunks // per), per


def _gamma(P, C, sms):
    n, per = _splits(P, C, sms)
    chunks_per_split = -(-per // _chunk_stages(C))
    return 32 * 2.0 ** -22 + (chunks_per_split + n + 4) * 2.0 ** -24


CHUNK_BIAS = 32 * 2.0 ** -22   # truncation loss bound of one chunk (module docstring)


def _features(P, C, seed, signed=False):
    """bf16 [P][C]: N(0,1) (ReLU'd unless signed) times a power of two per channel in 2^-6 .. 2^6, two dead channels,
    two constant ones"""
    g = torch.Generator(device=DEV).manual_seed(seed)
    f = torch.randn(P, C, generator=g, device=DEV, dtype=torch.bfloat16)
    if not signed:
        f.relu_()
    perm = torch.randperm(C, generator=torch.Generator().manual_seed(seed))
    scale = torch.pow(2.0, (perm % 13 - 6).float()).to(DEV, torch.bfloat16)
    f.mul_(scale)
    f[:, [1, C // 2 + 3]] = 0
    f[:, 5] = 0.75
    f[:, C - 2] = 1.5 * 2.0 ** -5
    return f, [1, C // 2 + 3]


def _gram(F_ptr, P, C):
    nf = _tlib().stb_test_gram_partials_floats(P, C)
    ws = torch.empty(nf, device=DEV)
    S = torch.empty(C, C, device=DEV)
    s = torch.empty(C, device=DEV)
    _check(_tlib().stb_test_gram(ctypes.c_void_p(F_ptr), P, C, _lib.ptr(ws), nf, _lib.ptr(S), _lib.ptr(s),
                                 _lib.cur_stream()))
    torch.cuda.synchronize()
    return S, s


def _gram_reference(f):
    """fp64 F^T F, |F|^T |F|, sums and sums of |F| on the device, in chunks of 2^26 elements"""
    P, C = f.shape
    S, A = torch.zeros(C, C, dtype=torch.float64, device=DEV), torch.zeros(C, C, dtype=torch.float64, device=DEV)
    s, sa = torch.zeros(C, dtype=torch.float64, device=DEV), torch.zeros(C, dtype=torch.float64, device=DEV)
    step = (1 << 26) // C
    for p0 in range(0, P, step):
        x = f[p0:p0 + step].double()
        S += x.t() @ x
        s += x.sum(0)
        x.abs_()
        A += x.t() @ x
        sa += x.sum(0)
    return S, A, s, sa


def _gram_case(f, P, C, dead, F_ptr=None, nonneg=True):
    """the per-element, bias and exact checks of one launch; returns the measured maxima"""
    ptr = f.data_ptr() if F_ptr is None else F_ptr
    S, s = _gram(ptr, P, C)
    S2, s2 = _gram(ptr, P, C)
    ref, A, sref, sa = _gram_reference(f)
    gamma = _gamma(P, C, _sms())
    assert torch.isfinite(S).all() and torch.isfinite(s).all()
    err, serr = (S.double() - ref).abs(), (s.double() - sref).abs()
    m = dict(P=P, C=C, gamma=gamma,
             elem=(err / A.clamp_min(1e-300)).max().item() / gamma,
             sums=(serr / sa.clamp_min(1e-300)).max().item() / gamma)
    assert (err <= gamma * A).all(), m
    assert (serr <= gamma * sa).all(), m
    if nonneg:
        nz = ref > 0
        m['bias'] = ((S.double() - ref)[nz] / ref[nz]).mean().item()
        m['sums_bias'] = ((s.double() - sref)[sref > 0] / sref[sref > 0]).mean().item()
        assert abs(m['bias']) <= CHUNK_BIAS and abs(m['sums_bias']) <= CHUNK_BIAS, m
    # exact: symmetric bit for bit, dead channels exactly 0, a second launch gives the same bits
    assert torch.equal(S, S.t())
    assert (S[dead] == 0).all() and (S[:, dead] == 0).all() and (s[dead] == 0).all()
    assert torch.equal(S, S2) and torch.equal(s, s2)
    print('METRICS gram', m)
    return m


def _enough_hbm(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + (2 << 30):
        pytest.skip(f'not enough free HBM ({free >> 20} MiB) for {nbytes >> 20} MiB of inputs')


@pytest.mark.parametrize('size', [512, 2048, 4096])
@pytest.mark.parametrize('layer', range(5), ids=TAPS)
def test_gram_production_pixel_counts(size, layer):
    """every style tap's pixel count at 512^2, 2048^2 and 4096^2: per-element bar, bias bar, exact invariants"""
    C, P = STYLE_C[layer], (size >> layer) ** 2
    _enough_hbm(P * C * 2 + (1 << 29))
    f, dead = _features(P, C, seed=size + layer)
    _gram_case(f, P, C, dead)
    del f
    torch.cuda.empty_cache()


def _ragged_cases():
    """(C, P, what): P one below / one above a multiple of PK x splits, P < PK, a short last split"""
    return [(C, what) for C in (64, 128, 256, 512) for what in ('below', 'above', 'lt_pk', 'short_last')]


@pytest.mark.parametrize('C,what', _ragged_cases())
def test_gram_ragged_pixel_counts(C, what):
    sms = _sms()
    unit = _pk(C) * _want_splits(C, sms)
    m = 20                                  # 20 stages per split: more than two 32-k-step chunks
    P = {'below': m * unit - 1, 'above': m * unit + 1, 'lt_pk': _pk(C) - 9,
         'short_last': (m * _want_splits(C, sms) - m // 2) * _pk(C) - 3}[what]
    n, per = _splits(P, C, sms)
    stages = -(-P // _pk(C))
    if what == 'short_last':
        assert stages - (n - 1) * per < per
    if what == 'above':
        assert stages - (n - 1) * per < per
    f, dead = _features(P, C, seed=P)
    _gram_case(f, P, C, dead)


def test_gram_signed_features():
    """the general path: signed features, where |F|^T |F| bounds the error of a cancelling sum"""
    P, C = 300_001, 256
    f, dead = _features(P, C, seed=11, signed=True)
    _gram_case(f, P, C, dead, nonneg=False)


@pytest.mark.parametrize('C,W,own0,rows', [(64, 512, 48, 200), (256, 128, 16, 37), (512, 64, 8, 23)])
def test_gram_band_window(C, W, own0, rows):
    """a band's own rows read as the iteration reads them, F + own0 W C with rows W pixels, NaN rows before and after
    the window: the TMA bound is P, not the allocation"""
    below = 7
    buf = torch.full(((own0 + rows + below) * W, C), float('nan'), dtype=torch.bfloat16, device=DEV)
    f, dead = _features(rows * W, C, seed=own0 + rows)
    buf[own0 * W:(own0 + rows) * W] = f
    _gram_case(f, rows * W, C, dead, F_ptr=buf[own0 * W:].data_ptr())


def test_gram_partials_within_the_planned_bound():
    """for every C, the split-K partials of every band and scale height the planner can produce (any own-row count at
    any level of the pyramid of a 4096 end scale) fit in gram_max_partials_floats(C) = want_splits (C^2 + C); the mirror
    of gram_num_splits above agrees with the library on every one of them"""
    sms = _sms()
    widths = sorted({w for s in gen_scales(64, 4096) for w in (s, (3 * s) // 4, s // 2)})
    for layer, C in enumerate(STYLE_C):
        bound = _want_splits(C, sms) * (C * C + C)
        for w in widths:
            wl = w >> layer
            if wl < 1:
                continue
            for rows in range(1, (4096 >> layer) + 1):
                P = rows * wl
                got = _tlib().stb_test_gram_partials_floats(P, C)
                assert got <= bound, (C, P, got, bound)
                assert got == _splits(P, C, sms)[0] * (C * C + C), (C, P)


# ---------------------------------------------------------------------------------------------- W2: five layers
_W2_WS = {}


def _w2_ws():
    if 'ws' not in _W2_WS:
        n = _tlib().stb_test_w2_workspace_bytes()
        _W2_WS['ws'] = torch.empty(n, dtype=torch.uint8, device=DEV)
    return _W2_WS['ws']


def _w2_layers(inp, build=1, n_calls=1, ws=None):
    """stb_test_w2_layers on inp = dict(mean_t, srm_t, S_raw, sums: 5 device tensors each; npix, weight: 5 floats)"""
    ws = _w2_ws() if ws is None else ws
    out = dict(loss=torch.full((5,), float('nan'), device=DEV),
               gs=[torch.full((c, c), float('nan'), device=DEV) for c in STYLE_C],
               gsb=[torch.full((c, c), float('nan'), dtype=torch.bfloat16, device=DEV) for c in STYLE_C],
               gmu=[torch.full((c,), float('nan'), device=DEV) for c in STYLE_C],
               mu=[torch.full((c,), float('nan'), device=DEV) for c in STYLE_C],
               cs=[torch.full((c, c), float('nan'), device=DEV) for c in STYLE_C])
    keep = []

    def arr(ts):
        p, a = _lib.ptr_array(ts)
        keep.append(a)
        return p

    f5 = ctypes.c_float * 5
    _check(_tlib().stb_test_w2_layers(arr(inp['mean_t']), arr(inp['srm_t']), arr(inp['S_raw']), arr(inp['sums']),
                                      f5(*inp['npix']), f5(*inp['weight']), build, n_calls, _lib.ptr(ws), ws.numel(),
                                      _lib.ptr(out['loss']), arr(out['gs']), arr(out['gsb']), arr(out['gmu']),
                                      arr(out['mu']), arr(out['cs']), _lib.cur_stream()))
    torch.cuda.synchronize()
    return {k: (v.cpu() if torch.is_tensor(v) else [t.cpu() for t in v]) for k, v in out.items()}


class _DeviceFloats:
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {'shape': (n,), 'typestr': '<f4', 'data': (ptr, False), 'version': 2}


_STYLE_MOMENTS = {}
_REAL = {}


def _real_stats(wts, size):
    """S_raw and channel sums of all five taps of a content-plus-noise iterate at size^2, read from the statistics
    block of a one-band context (as tests/test_gpu_tiled_gradient.py's Job), with the target moments of a synthetic
    style image"""
    if size in _REAL:
        return _REAL[size]
    style = O.to_tensor(O.synth_image(2, 32, 200, 152)).to(DEV).contiguous()
    content = O.to_tensor(O.synth_image(1, 16, size, size)).to(DEV).contiguous()
    m = NativeVGG(wts, 'max', DEV)
    m.ensure_workspace([(size, size), tuple(style.shape[2:])])
    means, srms = m.style_stats(style)
    ct = m.content_features(content)
    m.set_band(True, size, 0, size)
    m.set_targets(size, size, ct, 0.015, means, srms, STYLE_WEIGHTS, 2.0)
    g = torch.Generator(device=DEV).manual_seed(size)
    img = (content + 0.05 * torch.randn(content.shape, generator=g, device=DEV)).clamp(0, 1).contiguous()
    m.iterate_fwd(img)
    p, n = ctypes.c_void_p(), ctypes.c_size_t()
    _lib.check(m.lib.stb_stats_block(m.ctx, size, size, ctypes.byref(p), ctypes.byref(n)))
    block = torch.as_tensor(_DeviceFloats(p.value, n.value)).clone()
    torch.cuda.synchronize()
    S_raw, sums, o = [], [], 0
    for C in STYLE_C:
        S_raw.append(block[o:o + C * C].view(C, C).clone())
        sums.append(block[o + C * C:o + C * C + C].clone())
        o += C * C + C
    inp = dict(mean_t=[t.clone() for t in means], srm_t=[t.clone() for t in srms], S_raw=S_raw, sums=sums,
               npix=[float((size >> l) ** 2) for l in range(5)], weight=list(STYLE_WEIGHTS))
    del m, block
    torch.cuda.empty_cache()
    _REAL[size] = inp
    return inp


def _synthetic_stats():
    """rank-deficient moments with dead and duplicated channels (fewer samples than channels on the wide layers)"""
    g = torch.Generator().manual_seed(5)
    inp = dict(mean_t=[], srm_t=[], S_raw=[], sums=[], npix=[], weight=list(STYLE_WEIGHTS))
    for C in STYLE_C:
        n = C // 2 + 8

        def feats(scale):
            f = torch.relu(torch.randn(C, n, generator=g) * scale + 0.1)
            f[3] = 0
            f[C - 7] = 0
            f[10] = f[2]
            f[C - 1] = f[C // 2]
            return f

        ft, fc = feats(1.0), feats(1.3)
        inp['mean_t'].append(ft.mean(1).to(DEV))
        inp['srm_t'].append(((ft @ ft.t()) / n).to(DEV))
        inp['S_raw'].append((fc @ fc.t()).to(DEV))
        inp['sums'].append(fc.sum(1).to(DEV))
        inp['npix'].append(float(n))
    return inp


def _chain(mt, st, S, sm, npix, w, dt):
    """ST:149-181 / SQ:9-47 as test_gpu_kernels.test_w2_loss_sqrtm_and_backward states them, in dtype dt"""
    mt, st, mc, sc = mt.to(dt), st.to(dt), sm.to(dt) / npix, S.to(dt) / npix
    C = mt.numel()
    tgt = O.StyleTarget.build(mt, st)
    eye = torch.eye(C, dtype=dt)
    cov = sc - torch.outer(mc, mc) + eye * 1e-4
    md = ((mc - tgt.mean) ** 2).mean()
    r = O.sqrtm_ns(tgt.cov_sqrt @ cov @ tgt.cov_sqrt, 12)
    loss = (md + torch.diagonal(tgt.cov + cov - 2 * r).mean()) * w
    g_m = O.sqrtm_ns_lyap_backward(r, eye * (-2.0 * w / C), 12)
    g_cov = tgt.cov_sqrt.t() @ g_m @ tgt.cov_sqrt.t() + eye * (w / C)
    gs = g_cov + g_cov.t()
    gmu = (2.0 * w * (mc - tgt.mean) / C - gs @ mc) / npix
    return dict(loss=loss, gs=gs, gmu=gmu, cs=tgt.cov_sqrt)


def _rel(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).norm() / ref.norm().clamp_min(1e-300)).item()


def _chain_permuted(mt, st, S, sm, npix, w, dt, p):
    """_chain on the channels in order p, its results put back in the original order: every quantity is invariant, the
    summation order of every product is not"""
    r = _chain(mt[p], st[p][:, p], S[p][:, p], sm[p], npix, w, dt)
    inv = torch.argsort(p)
    return dict(loss=r['loss'], gs=r['gs'][inv][:, inv], gmu=r['gmu'][inv], cs=r['cs'][inv][:, inv])


N_ORDERS = 4


def _references(inp, layer):
    """the fp64 chain, and the fp32 chain in N_ORDERS channel orders (the identity first) on 4 CPU threads"""
    args = [inp[k][layer].cpu() for k in ('mean_t', 'srm_t', 'S_raw', 'sums')]
    args += [inp['npix'][layer], float(torch.tensor(inp['weight'][layer], dtype=torch.float32))]
    r64 = _chain(*args, torch.float64)
    C = STYLE_C[layer]
    g = torch.Generator().manual_seed(layer)
    orders = [torch.arange(C)] + [torch.randperm(C, generator=g) for _ in range(N_ORDERS - 1)]
    threads = torch.get_num_threads()
    torch.set_num_threads(4)
    try:
        r32 = [_chain_permuted(*args, torch.float32, p) for p in orders]
    finally:
        torch.set_num_threads(threads)
    return r64, r32


W2_FLOOR = 2.0 ** -20
W2_CASES = [128, 256, 512, 2048, 'synthetic']


@pytest.mark.parametrize('case', W2_CASES, ids=str)
def test_w2_five_layers_against_fp64(vgg_weights, case):
    """per layer: loss term, Gs, sqrt(cov_t), gmu within max(16 e32, 2^-20) of fp64; gs_bf16 and Gs^T exact; gmu
    element by element against fp64 on the engine's own Gs and mu"""
    if case == 2048:
        _enough_hbm(1100 * 2048 * 2048)
    inp = _synthetic_stats() if case == 'synthetic' else _real_stats(vgg_weights, case)
    out = _w2_layers(inp)
    fails = []
    for l, C in enumerate(STYLE_C):
        r64, r32 = _references(inp, l)
        got = dict(loss=out['loss'][l], gs=out['gs'][l], gmu=out['gmu'][l], cs=out['cs'][l])
        m = dict(case=case, layer=TAPS[l])
        for k in ('loss', 'gs', 'cs', 'gmu'):
            e32, e = max(_rel(r[k], r64[k]) for r in r32), _rel(got[k], r64[k])
            bar = max(16 * e32, W2_FLOOR)
            m[k] = (e, e32, bar)
            if not e <= bar:
                fails.append((TAPS[l], k, e, bar))
        if case == 2048:
            m['loss_2048'] = _rel(got['loss'], r64['loss'])
            if not m['loss_2048'] <= 3e-4:
                fails.append((TAPS[l], 'loss 3e-4', m['loss_2048']))
        # exact: the bf16 Gs / N the tap-gradient GEMM reads, and the symmetry of Gs
        gs = out['gs'][l]
        inv_n = torch.tensor([1.0], dtype=torch.float32) / torch.tensor([inp['npix'][l]], dtype=torch.float32)
        assert torch.equal(out['gsb'][l], (gs * inv_n).bfloat16()), (case, TAPS[l])
        assert torch.equal(gs, gs.t()), (case, TAPS[l])
        # w2_gmu_kernel alone: fmaf chain of n/32 steps per lane, 5-level warp sum, then ~3 roundings (module docstring)
        w = float(torch.tensor(inp['weight'][l], dtype=torch.float32))
        mu, mt, G = out['mu'][l].double(), inp['mean_t'][l].cpu().double(), gs.double()
        N = inp['npix'][l]
        t = 2.0 * w * (mu - mt) / C
        want = (t - G @ mu) / N
        bar = (C / 32 + 8) * 2.0 ** -24 * ((G * mu).abs().sum(1) + t.abs()) / N
        gerr = (out['gmu'][l].double() - want).abs()
        m['gmu_elem'] = (gerr / bar.clamp_min(1e-300)).max().item()
        assert (gerr <= bar).all(), m
        print('METRICS w2', m)
    assert not fails, fails


def _outputs_equal(a, b):
    bad = []
    for k in ('loss', 'gs', 'gsb', 'gmu', 'mu', 'cs'):
        for l in range(5 if k != 'loss' else 1):
            x, y = (a[k], b[k]) if k == 'loss' else (a[k][l], b[k][l])
            if not torch.equal(x, y):
                bad.append((k, l))
    return bad


def test_w2_state_carries_across_calls(vgg_weights):
    """forward_backward twice on one engine gives the bits of once; targets built on other statistics and reused
    (build_targets = 0) give the bits of targets built on these"""
    s1, s2 = _real_stats(vgg_weights, 512), _real_stats(vgg_weights, 256)
    once = _w2_layers(s2)
    twice = _w2_layers(s2, n_calls=2)
    _w2_layers(s1)
    reused = _w2_layers(s2, build=0)
    direct = _w2_layers(s2)
    assert _outputs_equal(once, twice) == []
    assert _outputs_equal(reused, direct) == []
    assert torch.isfinite(direct['loss']).all()


def _chain_child(d):
    """(subprocess, STB_W2_CHAIN=0) run the saved inputs through stb_test_w2_layers and save the outputs"""
    inp = torch.load(Path(d) / 'in.pt')
    for k in ('mean_t', 'srm_t', 'S_raw', 'sums'):
        inp[k] = [t.to(DEV) for t in inp[k]]
    torch.save(_w2_layers(inp), Path(d) / 'out.pt')


def test_w2_one_launch_per_round_equals_the_chain(vgg_weights):
    """STB_W2_CHAIN=0 (one launch per round, no grid barrier) gives the bits of the cooperative chain: a tile's
    arithmetic does not depend on which CTA runs it"""
    inp = _real_stats(vgg_weights, 256)
    chained = _w2_layers(inp)
    with tempfile.TemporaryDirectory() as d:
        torch.save({k: ([t.cpu() for t in v] if isinstance(v, list) and torch.is_tensor(v[0]) else v)
                    for k, v in inp.items()}, Path(d) / 'in.pt')
        code = (f'import sys; sys.path[:0] = [{str(ROOT)!r}, {str(ROOT / "tests")!r}]; '
                f'import test_gpu_style_stats as t; t._chain_child({d!r})')
        env = dict(os.environ, STB_W2_CHAIN='0')
        args = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code]
        r = subprocess.run(args, env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-4000:]
        per_round = torch.load(Path(d) / 'out.pt')
    assert _outputs_equal(per_round, chained) == []
