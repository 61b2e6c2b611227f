"""-m gpu: the device snapshot of the averaged image (stb_snapshot) and everything that saves through it:
get_image('pil' / 'np_uint16'), AsyncImageWriter (8-bit and 16-bit TIFF) and the CLI's `.tif` output with --proof.

The kernel's contract is bit-identity with the torch / numpy expressions it replaced:
  uint8 : (value / (1 - accum)).clamp(0, 1).mul(255).byte()              (to_pil_image)
  uint16: np.uint16(np.round((value / (1 - accum)).clamp(0, 1) * 65535)) (np_uint16)
"""
import contextlib
import io
import json
import os
import threading

import numpy as np
import pytest
import torch

import icc_profiles
from oracle import st_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    return g


def _old_u8(value, accum):
    return (value / (1 - accum))[0].clamp(0, 1).mul(255).byte().permute(1, 2, 0).cpu().numpy()


def _old_u16(value, accum):
    image = (value / (1 - accum))[0].clamp(0, 1)
    return np.uint16(np.round(image.cpu().movedim(0, 2).numpy() * 65535))


def _snap(value, h, w, denom, kind, out=None):
    from style_transfer_b200 import _lib
    if out is None:
        out = torch.empty(h, w, 3, dtype=(torch.uint8, torch.uint16)[kind], device=value.device)
    _lib.check(_lib.load().stb_snapshot(_lib.ptr(value), h, w, denom, kind, _lib.ptr(out), _lib.cur_stream()))
    return out.cpu().numpy()


def _values(h, w, denom, seed):
    """EMA storage for an image whose bias-corrected values are random in [-0.25, 1.25] plus, first, every special
    value: exact 0 and 1, out of range, uint8 truncation edges k/255 and uint16 ties (k + 0.5)/65535 with their float
    neighbours."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(3 * h * w, generator=g, dtype=torch.float64) * 1.5 - 0.25
    k8 = torch.arange(256, dtype=torch.float64) / 255
    k16 = (torch.randint(0, 65535, (512,), generator=g).double() + 0.5) / 65535
    edges = torch.cat([k8, k16]).float()
    special = torch.cat([torch.tensor([0., 1., -0., -1e-8, 1 + 1e-7, -3., 7., 0.5]), edges,
                         torch.nextafter(edges, torch.full_like(edges, 2.)),
                         torch.nextafter(edges, torch.full_like(edges, -2.))])
    n = min(special.numel(), x.numel())
    x = x.float()
    x[:n] = special[:n]
    v = x * denom if denom != 1 else x   # denom 1: the ties and edges reach the quantiser exactly
    return v.reshape(1, 3, h, w).cuda()


ACCUMS = [0.0] + [0.99 ** k for k in (1, 2, 3, 7, 50, 100, 333, 1000)]


@pytest.mark.parametrize('h,w', [(1, 1), (3, 5), (181, 136), (2047, 1365), (2048, 2048)])
def test_kernel_is_bit_identical_to_torch(h, w):
    for i, accum in enumerate(ACCUMS):
        v = _values(h, w, 1 - accum, seed=i)
        np.testing.assert_array_equal(_snap(v, h, w, 1 - accum, 0), _old_u8(v, accum), err_msg=f'uint8, accum {accum}')
        np.testing.assert_array_equal(_snap(v, h, w, 1 - accum, 1), _old_u16(v, accum),
                                      err_msg=f'uint16, accum {accum}')
    # an input that is not 16-byte aligned takes the element-wise path of the same kernel
    accum = 0.99 ** 7
    buf = _values(h, w + 1, 1 - accum, seed=99).reshape(-1)
    v = buf[1:1 + 3 * h * w].reshape(1, 3, h, w)
    np.testing.assert_array_equal(_snap(v, h, w, 1 - accum, 1), _old_u16(v, accum))
    np.testing.assert_array_equal(_snap(v, h, w, 1 - accum, 0), _old_u8(v, accum))


def test_kernel_rejects_bad_arguments():
    from style_transfer_b200 import _lib
    lib = _lib.load()
    v = torch.zeros(3, 4, 4, device='cuda')
    out = torch.zeros(4, 4, 3, dtype=torch.uint16, device='cuda')
    for args in [(None, 4, 4, 1.0, 0, out), (v, 4, 4, 1.0, 0, None), (v, 0, 4, 1.0, 1, out), (v, 4, 0, 1.0, 1, out),
                 (v, -1, 4, 1.0, 0, out), (v, 4, 4, 1.0, 2, out), (v, 4, 4, 1.0, -1, out)]:
        src, h, w, d, kind, o = args
        with pytest.raises(ValueError):
            _lib.check(lib.stb_snapshot(_lib.ptr(src), h, w, d, kind, _lib.ptr(o), _lib.cur_stream()))


def _stylize(G, wts, size=64, its=4, callback=None):
    st = G.make_st('max', wts)
    content, style = O.synth_image(1, 16, size, size * 3 // 4), O.synth_image(2, 32, size - 8, size * 3 // 4 - 8)
    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(content, [style], min_scale=size, end_scale=size, initial_iterations=its, callback=callback)
    return st


def test_get_image_matches_the_old_expressions(G, vgg_weights):
    st = _stylize(G, vgg_weights)
    value, accum = st.average.value, st.average.accum
    pil = st.get_image()
    assert pil.mode == 'RGB' and pil.size == (64, 48)
    np.testing.assert_array_equal(np.asarray(pil), _old_u8(value, accum))
    u16 = st.get_image('np_uint16')
    assert u16.dtype == np.uint16 and u16.shape == (48, 64, 3)
    np.testing.assert_array_equal(u16, _old_u16(value, accum))
    with pytest.raises(ValueError):
        st.get_image('float')


def test_banded_get_image_mid_scale(vgg_weights):
    """Two thread ranks on one GPU tile a 512 x 384 scale into bands.  Mid-scale, rank 0's get_image('np_uint16') is the
    uint16 expression on the gathered image; the other rank takes part in both gathers as the CLI does."""
    import style_transfer_b200 as stb
    from style_transfer_b200 import distributed as D
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '20')
    content, style = O.synth_image(1, 16, 512, 384), O.synth_image(2, 32, 296, 216)
    shared = D.ThreadGroup.Shared(2)
    got, errors = {}, []

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights,
                                   distributed=D.ThreadGroup(shared, rank))

            def cb(it):
                if it.i != 3:
                    return
                assert st._band is not None, 'the scale is not banded'
                if rank == 0:
                    got['snap'] = st.get_image('np_uint16')
                else:
                    st.get_image_tensor()
                t = st.get_image_tensor()
                if rank == 0:
                    got['want'] = np.uint16(np.round(t.cpu().movedim(0, 2).numpy() * 65535))

            with contextlib.redirect_stdout(io.StringIO()):
                img = st.stylize(content, [style], min_scale=512, end_scale=512, initial_iterations=6, callback=cb)
            got[rank] = np.asarray(img)
        except BaseException as e:  # noqa: BLE001 -- report and release the other rank
            errors.append((rank, repr(e)))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    assert not errors, errors
    assert got['snap'].shape == (384, 512, 3)
    np.testing.assert_array_equal(got['snap'], got['want'])
    np.testing.assert_array_equal(got[0], got[1])


def test_async_writer_tiff_does_not_wait_for_the_device(G, vgg_weights, tmp_path):
    """A .tif submit_snapshot at the last iteration: the callback returns before the work queued ahead of it on the
    iteration stream is done, and the file holds exactly get_image('np_uint16')."""
    cv2 = pytest.importorskip('cv2')
    from style_transfer_b200.image_io import AsyncImageWriter
    wr = AsyncImageWriter()
    path = tmp_path / 'snap.tif'
    pending = []

    def cb(it):
        if it.i != it.i_max:
            return
        st = holder[0]
        torch.cuda._sleep(200_000_000)          # ~0.1 s of device time queued ahead of the snapshot
        end = torch.cuda.Event()
        end.record(st._stream)
        wr.submit_snapshot(st, path)
        pending.append(end.query())

    holder = []
    st = G.make_st('max', vgg_weights)
    holder.append(st)
    content, style = O.synth_image(1, 16, 256, 192), O.synth_image(2, 32, 200, 160)
    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(content, [style], min_scale=256, end_scale=256, initial_iterations=3, callback=cb)
    wr.close()
    assert pending == [False], 'submit_snapshot waited for the device'
    saved = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    assert saved.dtype == np.uint16
    np.testing.assert_array_equal(saved[..., ::-1], st.get_image('np_uint16'))


def _read_tiff_tags(path):
    import test_image_io_cpu as T
    return T.parse_tiff(path.read_bytes())


@pytest.mark.parametrize('proof', [False, True])
def test_cli_writes_16bit_tiff(vgg_weights, tmp_path, monkeypatch, proof):
    from style_transfer_b200 import cli
    from style_transfer_b200 import style_transfer as S
    from style_transfer_b200.image_io import srgb_profile
    monkeypatch.setattr(S, 'load_vgg19_conv_weights', lambda: vgg_weights)   # no network for the ImageNet weights
    monkeypatch.chdir(tmp_path)
    O.synth_image(1, 16, 96, 72).save('c.png')
    O.synth_image(2, 32, 80, 64).save('s.png')
    argv = ['c.png', 's.png', '-s', '64', '-ms', '64', '-ii', '4', '-o', 'out.tif', '--save-every', '2']
    if proof:
        (tmp_path / 'cmyk.icc').write_bytes(icc_profiles.narrow_cmyk())
        argv += ['--proof', 'cmyk.icc']
    with contextlib.redirect_stdout(io.StringIO()):
        cli.main(argv)
    tags = _read_tiff_tags(tmp_path / 'out.tif')
    assert tags[256] == (64,) and tags[257] == (48,) and tags[258] == (16, 16, 16)
    assert tags[34675] == srgb_profile
    trace = json.load(open('trace.json'))
    assert len(trace['iterates']) == 4 and trace['args']['proof'] == ('cmyk.icc' if proof else None)
    assert not list(tmp_path.glob('*.part.*'))


def test_snapshot_leaves_the_iteration_graph_alone(G, vgg_weights):
    """Snapshots between iterations are launched outside the iteration's CUDA graph: the graph replays and the kernel
    nodes per graph are those of a run without them."""
    def snap_every(st_box):
        def cb(it):
            st_box[0]._snapshot(0)
            st_box[0]._snapshot(1)
        return cb

    counts = []
    for with_snap in (False, True):
        box = []
        st = G.make_st('max', vgg_weights)
        box.append(st)
        cb = snap_every(box) if with_snap else (lambda it: None)
        content, style = O.synth_image(1, 16, 128, 96), O.synth_image(2, 32, 100, 80)
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], min_scale=128, end_scale=128, initial_iterations=5, callback=cb)
        counts.append(st.model.launch_count())
    assert counts[0] == counts[1], counts
    assert counts[0][0] > 0
