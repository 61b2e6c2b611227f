"""-m gpu: the multi-GPU (spatially tiled) path on ONE GPU.

The ranks of `stb_iterate_banded` only ever read each other's mailboxes through device pointers, so the very same
library path -- halo pull, band-local statistics, peer all-reduce, seam reduce fused with Adam, one CUDA graph per
rank -- runs with the ranks as THREADS of this process, each with its own context and stream on cuda:0
(distributed.ThreadGroup; mailboxes connected with stb_comm_connect_local instead of CUDA IPC).  What this cannot
cover is the IPC mapping and NVLink itself: tools/dist_check.py does that under torchrun on a multi-GPU box, and
bench.py at N > 1 prints `parity_vs_n1`.
"""
import contextlib
import io
import os
import threading

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import st_oracle as O  # noqa: E402  (fixture generator: weights / synthetic images)


def run_tiled(world, content, style, wts, kw):
    import style_transfer_b200 as stb
    from style_transfer_b200 import distributed as D
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '20')
    shared = D.ThreadGroup.Shared(world)
    results, errors = [None] * world, []

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts,
                                   distributed=D.ThreadGroup(shared, rank))
            trace = []
            with contextlib.redirect_stdout(io.StringIO()):
                img = st.stylize(content, [style], callback=lambda it: trace.append(it.loss), **kw)
            results[rank] = (np.array(trace), np.asarray(img, dtype=np.float32),
                             (st._comm_mode, 'halo' if st._halo_now else 'apron'), st.model.graph_status())
        except BaseException as e:  # noqa: BLE001 -- report and release the other ranks
            errors.append((rank, repr(e)))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(300)
    assert not errors, errors
    assert all(r is not None for r in results), 'a rank did not finish'
    return results


def run_single(content, style, wts, kw):
    import style_transfer_b200 as stb
    st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=wts, distributed=False)
    trace = []
    with contextlib.redirect_stdout(io.StringIO()):
        img = st.stylize(content, [style], callback=lambda it: trace.append(it.loss), **kw)
    return np.array(trace), np.asarray(img, dtype=np.float32)


TILE = os.environ.get('STB_TILE', 'auto')


@pytest.mark.parametrize('tile', ['halo', 'apron'])
@pytest.mark.parametrize('world,W,H,its', [(2, 512, 384, 6), (3, 200, 400, 5), (2, 362, 384, 4), (4, 256, 512, 4)])
def test_tiled_threads_equal_single_gpu(vgg_weights, monkeypatch, tile, world, W, H, its):
    """Loss trace and result of the banded run (world ranks) vs the untiled run of the same job.  362 is not a multiple
    of 4 (scalar row kernels); 3 ranks give unequal bands; 4 ranks have two interior bands with aprons on both sides."""
    monkeypatch.setenv('STB_TILE', tile)
    global TILE
    TILE = tile
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, W // 2 + 40, H // 2 + 24)
    scale = max(H, W)
    kw = dict(min_scale=scale, end_scale=scale, initial_iterations=its)
    tiled = run_tiled(world, content, style, vgg_weights, kw)
    tr_s, img_s = run_single(content, style, vgg_weights, kw)
    for rank, (tr, img, mode, (gstat, note)) in enumerate(tiled):
        # exchanges inside the library; tile mode as requested (these images are narrow: 'auto' picks aprons)
        assert mode == ('peer', {'auto': 'apron'}.get(TILE, TILE))
        assert gstat == 1, f'rank {rank}: iterations did not replay as a CUDA graph ({note})'
        assert len(tr) == its
        rel = np.abs(tr - tr_s) / np.abs(tr_s)
        assert rel.max() < 5e-4, (rank, rel)        # summation order of the split statistics moves the loss ~1e-4
        assert np.abs(img - img_s).mean() < 0.5     # /255
    # every rank ends with the identical full image and saw the identical loss (bit-identical reduced statistics)
    for tr, img, _, _ in tiled[1:]:
        np.testing.assert_array_equal(tr, tiled[0][0])
        np.testing.assert_array_equal(img, tiled[0][1])


@pytest.mark.parametrize('tile', ['halo', 'apron'])
def test_tiled_pyramid_mixes_replicated_and_banded_scales(vgg_weights, monkeypatch, tile):
    """Small scales run replicated (too few rows to tile), the larger ones banded; Adam state and the step counter are
    carried across both kinds of scale (ST:285-295, 460-462), the mailboxes are sized once for the last scale."""
    monkeypatch.setenv('STB_TILE', tile)
    W, H = 288, 384
    content, style = O.synth_image(1, 16, W, H), O.synth_image(2, 32, 260, 300)
    kw = dict(min_scale=128, end_scale=384, iterations=3, initial_iterations=4)
    tiled = run_tiled(2, content, style, vgg_weights, kw)
    tr_s, img_s = run_single(content, style, vgg_weights, kw)
    tr, img = tiled[0][0], tiled[0][1]
    assert len(tr) == len(tr_s)
    np.testing.assert_allclose(tr, tr_s, rtol=2e-3)   # trajectories: sign-like Adam steps amplify 1e-4 differences
    assert np.abs(img - img_s).mean() < 1.0
    np.testing.assert_array_equal(tiled[1][1], img)


@pytest.mark.parametrize('optimizer', ['adam', 'lbfgs'])
def test_tiled_run_without_peer_memory_runs_replicated(vgg_weights, monkeypatch, optimizer):
    """When some rank cannot map the others' memory, every rank runs every scale untiled: the same loss trace and image
    as the single-GPU run, bit for bit.  The mapping is tried once, at the first scale tall enough to tile (272 rows);
    the style image (150 rows) is too short to band, so no statistics are split across the ranks either."""
    from style_transfer_b200 import _lib
    from style_transfer_b200.style_transfer import NativeVGG
    create, calls = NativeVGG.comm_create, []

    def comm_create(self, rank, *args):
        calls.append(rank)
        if rank == 1:
            raise _lib.NativeError('no peer memory on rank 1')
        return create(self, rank, *args)

    monkeypatch.setattr(NativeVGG, 'comm_create', comm_create)
    content, style = O.synth_image(1, 16, 288, 384), O.synth_image(2, 32, 200, 150)
    kw = dict(min_scale=272, end_scale=384, iterations=3, initial_iterations=4, optimizer=optimizer)
    tiled = run_tiled(2, content, style, vgg_weights, kw)
    tr_s, img_s = run_single(content, style, vgg_weights, kw)
    assert sorted(calls) == [0, 1]
    for tr, img, mode, _ in tiled:
        assert mode == ('off', 'apron')
        np.testing.assert_array_equal(tr, tr_s)
        np.testing.assert_array_equal(img, img_s)
