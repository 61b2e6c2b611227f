"""-m gpu: the live web monitor fed from device snapshots (WebInterface.put_iterate(it, st)).  A loopback client holds
the websocket and fetches /image back to back, as the page does; the run with the monitor must give exactly what the
run without it gives.  Every server binds 127.0.0.1 on an ephemeral port."""
import asyncio
import contextlib
import io
import json
import re
import threading
from dataclasses import asdict

import numpy as np
import pytest
import torch
from PIL import Image

from oracle import st_oracle as O

aiohttp = pytest.importorskip('aiohttp')
pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def G():
    import gpu_util as g
    return g


def _want_jpeg(pil):
    from style_transfer_b200.image_io import srgb_profile
    buf = io.BytesIO()
    pil.save(buf, format='jpeg', icc_profile=srgb_profile, quality=95, subsampling=0)
    return buf.getvalue()


class Client:
    """A browser stand-in on a thread of its own: holds the websocket, fetches /image back to back (one request in
    flight), and after WIDone fetches the final image once and disconnects."""

    def __init__(self, url):
        self.url = url
        self.messages, self.sizes, self.final, self.errors = [], [], None, []
        self.connected = threading.Event()
        self._thread = threading.Thread(target=lambda: asyncio.run(self._main()), name='test-web-client')
        self._thread.start()
        assert self.connected.wait(10), 'the client did not connect'

    async def _main(self):
        try:
            async with aiohttp.ClientSession() as s:
                async with s.ws_connect(self.url + 'websocket') as ws:
                    self.connected.set()
                    done = asyncio.Event()
                    fetcher = asyncio.ensure_future(self._fetch_loop(s, done))
                    async for msg in ws:
                        self.messages.append(json.loads(msg.data))
                        if self.messages[-1]['_type'] == 'WIDone':
                            break
                    done.set()
                    await fetcher
                    async with s.get(self.url + 'image') as r:
                        assert r.status == 200
                        self.final = await r.read()
        except BaseException as e:  # noqa: BLE001 -- reported by join()
            self.errors.append(repr(e))
            self.connected.set()

    async def _fetch_loop(self, s, done):
        while not done.is_set():
            async with s.get(self.url + 'image') as r:
                body = await r.read()
                if r.status == 200:
                    self.sizes.append(Image.open(io.BytesIO(body)).size)
                else:
                    assert r.status == 404
                    await asyncio.sleep(0.002)

    def join(self):
        self._thread.join(60)
        assert not self._thread.is_alive(), 'the client did not finish'
        assert not self.errors, self.errors


def _monitor_threads():
    return [t for t in threading.enumerate() if t.name.startswith('stb-web')]


def _run(st, content, style, kw, web=None):
    trace = []

    def cb(it):
        trace.append(it)
        if web is not None:
            web.put_iterate(it, st)
            if it.i == it.i_max and max(it.w, it.h) == kw['end_scale']:
                web.put_done()

    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        st.stylize(content, [style], callback=cb, **kw)
    return trace


def test_monitor_leaves_the_run_alone(G, vgg_weights):
    from style_transfer_b200 import WebInterface
    content, style = O.synth_image(1, 16, 96, 72), O.synth_image(2, 32, 80, 64)
    kw = dict(min_scale=64, end_scale=96, iterations=5, initial_iterations=6)

    st0 = G.make_st('max', vgg_weights)
    trace0 = _run(st0, content, style, kw)

    with contextlib.redirect_stdout(io.StringIO()):
        web = WebInterface('127.0.0.1', 0)
    try:
        client = Client(web.url)
        st1 = G.make_st('max', vgg_weights)
        trace1 = _run(st1, content, style, kw, web)
    finally:
        web.close()
    client.join()
    assert not _monitor_threads()

    assert [it.loss for it in trace1] == [it.loss for it in trace0]
    np.testing.assert_array_equal(st1.get_image('np_uint16'), st0.get_image('np_uint16'))
    assert st1.model.launch_count() == st0.model.launch_count()

    want = [dict(asdict(it), _type='STIterate') for it in trace1] + [{'_type': 'WIDone'}]
    assert client.messages == want
    scales = {(it.w, it.h) for it in trace1}
    assert client.sizes and set(client.sizes) <= scales, (set(client.sizes), scales)
    assert client.final == _want_jpeg(st1.get_image())
    assert web.snapshots >= len(scales)


def test_put_iterate_does_not_wait_for_the_device(G, vgg_weights):
    from style_transfer_b200 import WebInterface
    with contextlib.redirect_stdout(io.StringIO()):
        web = WebInterface('127.0.0.1', 0)
    pending = []
    box = []

    def cb(it):
        st = box[0]
        if it.i == it.i_max:
            with torch.cuda.stream(st._stream):
                torch.cuda._sleep(200_000_000)   # ~0.1 s of device time queued ahead of the snapshot
            end = torch.cuda.Event()
            end.record(st._stream)
            web.put_iterate(it, st)
            pending.append(end.query())
        else:
            web.put_iterate(it, st)

    try:
        st = G.make_st('max', vgg_weights)
        box.append(st)
        content, style = O.synth_image(1, 16, 256, 192), O.synth_image(2, 32, 200, 160)
        with contextlib.redirect_stdout(io.StringIO()):
            st.stylize(content, [style], min_scale=256, end_scale=256, initial_iterations=3, callback=cb)
        assert pending == [False], 'put_iterate waited for the device'
        assert web.snapshots == 1                       # no client: the scale's last image only

        async def fetch():
            async with aiohttp.ClientSession() as s:
                async with s.get(web.url + 'image') as r:
                    return r.status, await r.read()
        status, body = asyncio.run(fetch())
        assert status == 200 and body == _want_jpeg(st.get_image())
    finally:
        web.close()


def test_banded_scale_serves_the_whole_image(vgg_weights):
    import os
    import style_transfer_b200 as stb
    from style_transfer_b200 import WebInterface
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '20')
    content, style = O.synth_image(1, 16, 512, 384), O.synth_image(2, 32, 296, 216)
    kw = dict(min_scale=512, end_scale=512, initial_iterations=8)

    st0 = stb.StyleTransfer(devices=['cuda:0', 'cuda:0'], pooling='max', vgg_weights=vgg_weights)
    trace0 = _run(st0, content, style, kw)

    with contextlib.redirect_stdout(io.StringIO()):
        web = WebInterface('127.0.0.1', 0)
    banded = []
    try:
        client = Client(web.url)
        st1 = stb.StyleTransfer(devices=['cuda:0', 'cuda:0'], pooling='max', vgg_weights=vgg_weights)
        orig = web.put_iterate

        def put(it, st, **kw_):
            banded.append(st._band is not None)
            orig(it, st, **kw_)
        web.put_iterate = put
        trace1 = _run(st1, content, style, kw, web)
    finally:
        web.close()
    client.join()
    assert all(banded) and len(banded) == 8
    assert [it.loss for it in trace1] == [it.loss for it in trace0]
    np.testing.assert_array_equal(np.asarray(st1.get_image()), np.asarray(st0.get_image()))
    assert client.sizes and all(size == (512, 384) for size in client.sizes), client.sizes
    assert client.final == _want_jpeg(st1.get_image())


class _URLWatch(io.StringIO):
    def __init__(self):
        super().__init__()
        self.url = None
        self.seen = threading.Event()

    def write(self, s):
        m = re.search(r'http://127\.0\.0\.1:\d+/', s)
        if m and self.url is None:
            self.url = m.group(0)
            self.seen.set()
        return super().write(s)


def test_cli_web(vgg_weights, tmp_path, monkeypatch):
    from style_transfer_b200 import cli, web as W
    from style_transfer_b200 import style_transfer as S
    monkeypatch.setattr(S, 'load_vgg19_conv_weights', lambda: vgg_weights)   # no network for the ImageNet weights
    monkeypatch.chdir(tmp_path)
    O.synth_image(1, 16, 96, 72).save('c.png')
    O.synth_image(2, 32, 80, 64).save('s.png')
    out = _URLWatch()
    clients = []

    class Held(W.WebInterface):
        """Starts the client as soon as the URL is printed, and holds the first iteration until it has connected."""
        def __init__(self, host, port):
            super().__init__(host, port)
            assert out.seen.is_set()
            clients.append(Client(out.url))

    monkeypatch.setattr(W, 'WebInterface', Held)
    argv = ['c.png', 's.png', '-s', '96', '-ms', '64', '-i', '3', '-ii', '4', '-o', 'out.png',
            '--web', '--host', '127.0.0.1', '--port', '0']
    with contextlib.redirect_stdout(out):
        cli.main(argv)
    clients[0].join()
    assert not _monitor_threads()
    trace = json.load(open('trace.json'))['iterates']
    assert len(trace) == 7
    assert clients[0].messages == [dict(it, _type='STIterate') for it in trace] + [{'_type': 'WIDone'}]
    assert (tmp_path / 'out.png').exists()
    assert clients[0].final == _want_jpeg(Image.open('out.png').convert('RGB'))


def test_scale_tiled_across_processes_refreshes_at_the_gathers(vgg_weights):
    """Two ranks with no in-process lockstep, as under torchrun: only rank 0 serves, and it may not gather alone.  The
    CLI's pattern: at a save every rank gathers once and rank 0 hands that image to the monitor (`gathered=`); other
    iterations send their message only; the final image goes out with put_done(st) once stylize() has stitched the
    bands.  Every served image is whole, and the last one is the run's image."""
    import os
    import style_transfer_b200 as stb
    from style_transfer_b200 import WebInterface
    from style_transfer_b200 import distributed as D
    os.environ.setdefault('STB_COMM_TIMEOUT_S', '20')
    content, style = O.synth_image(1, 16, 512, 384), O.synth_image(2, 32, 296, 216)
    shared = D.ThreadGroup.Shared(2)
    with contextlib.redirect_stdout(io.StringIO()):
        web = WebInterface('127.0.0.1', 0)
    client = Client(web.url)
    got, errors, saves = {}, [], (3, 6)

    def worker(rank):
        try:
            torch.cuda.set_device(0)
            st = stb.StyleTransfer(devices=['cuda:0'], pooling='max', vgg_weights=vgg_weights,
                                   distributed=D.ThreadGroup(shared, rank))

            def cb(it):
                assert st._band is not None and st._sync is None
                gathered = st.get_image_tensor() if it.i in saves else None   # collective: every rank
                if rank == 0:
                    web.put_iterate(it, st, gathered=gathered)
                    got.setdefault('trace', []).append(it)

            with contextlib.redirect_stdout(io.StringIO()):
                st.stylize(content, [style], min_scale=512, end_scale=512, initial_iterations=8, callback=cb)
            if rank == 0:
                web.put_done(st)
                got['image'] = st.get_image()
        except BaseException as e:  # noqa: BLE001 -- report and release the other rank
            errors.append((rank, repr(e)))
            shared.bar.abort()

    threads = [threading.Thread(target=worker, args=(r,)) for r in range(2)]
    try:
        for t in threads:
            t.start()
        for t in threads:
            t.join(300)
    finally:
        web.close()
    client.join()
    assert not errors, errors
    assert web.snapshots == len(saves) + 1
    assert client.messages == [dict(asdict(it), _type='STIterate') for it in got['trace']] + [{'_type': 'WIDone'}]
    assert all(size == (512, 384) for size in client.sizes), client.sizes
    assert client.final == _want_jpeg(got['image'])
