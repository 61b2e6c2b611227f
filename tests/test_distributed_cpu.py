"""-m "not gpu": the multi-GPU band scheme on CPU (2 and 3 bands), and the per-scale group collectives.

A small translation-invariant network stands in for VGG (same structure of the problem: local conv/pool trunk,
loss = function of GLOBAL pixel sums + a per-pixel term).  Each band works on its own rows + aprons, the "stats" of the
own rows are summed over the bands, the gradients of the apron rows are added to the neighbours' own rows, the image
halo is refreshed -- the three exchanges of a tiled iteration -- and the result must equal the full-image run.
"""
import pytest
import torch
import torch.nn.functional as F

import style_transfer_b200  # noqa: F401  (registers the package)
from style_transfer_b200 import distributed as D


def _net(x, w1, w2, w3):
    """3 convs + 2 floor-mode pools: receptive-field radius 1 + 2 + 4 = 7 px << APRON."""
    h = torch.relu(F.conv2d(F.pad(x, (1, 1, 1, 1), mode='replicate'), w1))
    h = F.max_pool2d(h, 2)
    h = torch.relu(F.conv2d(h, w2, padding=1))
    h = F.max_pool2d(h, 2)
    return torch.relu(F.conv2d(h, w3, padding=1))


def _weights():
    g = torch.Generator().manual_seed(0)
    return (torch.randn(8, 3, 3, 3, generator=g) * 0.3, torch.randn(8, 8, 3, 3, generator=g) * 0.2,
            torch.randn(6, 8, 3, 3, generator=g) * 0.2)


def _full_reference(x, target):
    w = _weights()
    x = x.clone().requires_grad_()
    f = _net(x, *w)
    n = f.shape[2] * f.shape[3]
    stats = f.sum(dim=(2, 3)) / n
    loss = ((stats - target) ** 2).sum() + 0.1 * (x ** 2).mean()
    loss.backward()
    return loss.item(), x.grad


@pytest.mark.parametrize('world,H', [(2, 256), (3, 400), (2, 211)])
def test_band_exchanges_equal_full(world, H):
    W = 40
    torch.manual_seed(1)
    x_full = torch.rand(1, 3, H, W)
    target = torch.linspace(0, 1, 6)[None]
    bands = D.all_bands(H, world)
    assert all(b is not None for b in bands)
    xs, stats_local, pix = [], [], []
    for band in bands:
        x = D.local_slice(x_full, band).requires_grad_()
        f = _net(x, *_weights())
        lo, rows = band.own0 // 4, band.own_rows // 4
        if band.own_end == H:
            rows = f.shape[2] - lo
        xs.append(x)
        stats_local.append(f[:, :, lo:lo + rows].sum(dim=(2, 3)))                        # own rows only
        pix.append(0.1 * (x[:, :, band.own0:band.own0 + band.own_rows] ** 2).sum() / (3 * H * W))
    stats = sum(s.detach() for s in stats_local)                      # == the stats-block all-reduce
    n_global = (H // 4) * (W // 4)
    g_stats = 2 * (stats / n_global - target) / n_global              # d loss / d stats from the reduced statistics
    # seam add: each band's gradient goes to its rows of the full gradient, so its aprons' share lands on the
    # neighbours' own rows
    grad = torch.zeros_like(x_full)
    for band, x, s, p in zip(bands, xs, stats_local, pix):
        (s * g_stats).sum().backward()
        p.backward()
        grad[:, :, band.loc_begin:band.loc_end] += x.grad
    loss = ((stats / n_global - target) ** 2).sum() + sum(p.detach() for p in pix)
    # "update" the own rows of every band, then refresh the halos: each band's local rows read back from the full image
    new = x_full.clone()
    for band in bands:
        own = slice(band.own_begin, band.own_end)
        new[:, :, own] -= 0.5 * grad[:, :, own]
    ref_loss, ref_grad = _full_reference(x_full, target)
    assert abs(loss.item() - ref_loss) < 1e-5 * max(1, abs(ref_loss))
    torch.testing.assert_close(grad, ref_grad, atol=1e-6, rtol=1e-4)
    expect_new = x_full - 0.5 * ref_grad
    for band in bands:
        torch.testing.assert_close(D.local_slice(new, band), expect_new[:, :, band.loc_begin:band.loc_end],
                                   atol=1e-6, rtol=1e-4)


def test_band_geometry():
    for H, world in ((4096, 8), (2048, 2), (2172, 4), (256, 2)):
        edges = D.band_edges(H, world)
        assert edges[0] == 0 and edges[-1] == H and all(e % 16 == 0 for e in edges[1:-1])
        bands = [D.make_band(H, r, world) for r in range(world)]
        assert all(b is not None for b in bands)
        for b in bands:
            assert b.own0 % 16 == 0 and b.top_apron in (0, D.APRON) and b.bottom_apron in (0, D.APRON)
    assert D.make_band(128, 0, 2) is None      # too small to tile: replicated mode
    assert D.make_band(2048, 0, 1) is None


def test_thread_group_collectives():
    """ThreadGroup (the ranks as threads of one process -- how tests/test_gpu_tiled.py runs the tiled path on ONE GPU)
    offers the same per-scale collectives as TorchGroup: all-reduce, all-gather, broadcast, object gather, row gather."""
    import threading
    world, H, W = 3, 400, 8
    shared = D.ThreadGroup.Shared(world)
    full = torch.arange(H * W, dtype=torch.float32).reshape(1, 1, H, W)
    out, errors = [None] * world, []

    def worker(rank):
        try:
            g = D.ThreadGroup(shared, rank)
            band = D.make_band(H, rank, world)
            t = torch.full((4,), float(rank + 1))
            g.all_reduce_sum(t)
            objs = g.all_gather_object(('r', rank))
            b = torch.full((2,), float(rank))
            g.broadcast(b, 1)
            local = D.local_slice(full, band).clone()
            local[:, :, :band.own0] = -1                      # aprons hold garbage: only own rows may be gathered
            local[:, :, band.own0 + band.own_rows:] = -1
            out[rank] = (t, objs, b, D.gather_rows(local, band, g))
        except BaseException as e:  # noqa: BLE001
            errors.append(repr(e))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(60)
    assert not errors, errors
    for rank in range(world):
        t, objs, b, gathered = out[rank]
        assert torch.equal(t, torch.full((4,), 6.0))
        assert objs == [('r', 0), ('r', 1), ('r', 2)]
        assert torch.equal(b, torch.full((2,), 1.0))
        assert torch.equal(gathered, full)


def test_tap_pixel_counts_and_all_bands():
    assert D.tap_pixel_counts(181, 136) == [181 * 136, 90 * 68, 45 * 34, 22 * 17, 11 * 8]
    bands = D.all_bands(2048, 8)
    assert [b.own_rows for b in bands] == [256] * 8 and bands[0].top_apron == 0 and bands[3].h_local == 256 + 160
