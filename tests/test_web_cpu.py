"""The live web monitor (style_transfer_b200.WebInterface) without a GPU: routes, wire format, JPEG bytes, the refresh
policy of device snapshots (with a fake snapshot source), shutdown, and the CLI's flags.  Every server binds 127.0.0.1
on an ephemeral port and every client connects there only."""
import asyncio
import io
import json
import re
import socket
import threading
import time

import numpy as np
import pytest
import torch
from PIL import Image, JpegImagePlugin

aiohttp = pytest.importorskip('aiohttp')

import style_transfer_b200 as stb   # noqa: E402
from style_transfer_b200 import STIterate, WebInterface   # noqa: E402
from style_transfer_b200.image_io import srgb_profile   # noqa: E402

KEYS = ['w', 'h', 'i', 'i_max', 'loss', 'time', 'gpu_ram', '_type']


def _it(i, i_max=10, w=56, h=40):
    return STIterate(w=w, h=h, i=i, i_max=i_max, loss=1000.0 / i, time=1.7e9 + 0.01 * i, gpu_ram=123456 * i)


def _get(url):
    async def go():
        async with aiohttp.ClientSession() as s:
            async with s.get(url) as r:
                return r.status, r.headers.get('Content-Type'), await r.read()
    return asyncio.run(go())


def _want_jpeg(tensor):
    buf = io.BytesIO()
    arr = tensor.mul(255).byte().permute(1, 2, 0).numpy()
    Image.fromarray(arr).save(buf, format='jpeg', icc_profile=srgb_profile, quality=95, subsampling=0)
    return buf.getvalue()


def _monitor_threads():
    return [t for t in threading.enumerate() if t.name.startswith('stb-web')]


@pytest.fixture
def wi():
    w = WebInterface('127.0.0.1', 0)
    yield w
    w.close()


def _wait_clients(w, n, timeout=5.0):
    end = time.monotonic() + timeout
    while w.clients != n:
        assert time.monotonic() < end, f'{w.clients} clients connected, expected {n}'
        time.sleep(0.005)


def test_page_and_its_files_are_served(wi):
    status, ctype, body = _get(wi.url)
    assert status == 200 and ctype.startswith('text/html')
    refs = re.findall(r'(?:src|href)="([^"#]+)"', body.decode())
    assert 'main.js' in refs and 'main.css' in refs
    for ref in refs:
        assert _get(wi.url + ref)[0] == 200, ref
    assert _get(wi.url + 'image')[0] == 404


def test_websocket_messages_in_order(wi):
    its = [_it(i, 3) for i in (1, 2, 3)]
    got = []

    async def client():
        async with aiohttp.ClientSession() as s:
            async with s.ws_connect(wi.url + 'websocket') as ws:
                ready.set()
                async for msg in ws:
                    got.append(json.loads(msg.data))
                    if got[-1]['_type'] == 'WIDone':
                        break

    ready = threading.Event()
    t = threading.Thread(target=lambda: asyncio.run(client()))
    t.start()
    assert ready.wait(5)
    _wait_clients(wi, 1)
    for it in its:
        wi.put_iterate(it, torch.rand(3, 40, 56))
    wi.put_done()
    t.join(10)
    assert not t.is_alive()
    assert len(got) == 4
    for msg, it in zip(got, its):
        assert sorted(msg) == sorted(KEYS)
        assert msg['_type'] == 'STIterate'
        assert {k: msg[k] for k in KEYS[:-1]} == {k: getattr(it, k) for k in KEYS[:-1]}
    assert got[3] == {'_type': 'WIDone'}


def test_image_is_the_reference_jpeg(wi):
    g = torch.Generator().manual_seed(3)
    image = torch.rand(3, 37, 53, generator=g)
    image[:, :2] = torch.tensor([0.0, 1.0, 0.5]).view(3, 1, 1)
    wi.put_iterate(_it(1, w=53, h=37), image)
    status, ctype, body = _get(wi.url + 'image')
    assert status == 200 and ctype == 'image/jpeg'
    assert body == _want_jpeg(image)
    im = Image.open(io.BytesIO(body))
    assert im.size == (53, 37)
    assert im.info['icc_profile'] == srgb_profile
    assert JpegImagePlugin.get_sampling(im) == 0          # 4:4:4


def test_latest_image_wins(wi):
    a, b = torch.rand(3, 20, 30), torch.rand(3, 24, 32)
    wi.put_iterate(_it(1, w=30, h=20), a)
    wi.put_iterate(_it(2, w=32, h=24), b)
    assert _get(wi.url + 'image')[2] == _want_jpeg(b)


class _Event:
    def __init__(self):
        self.done = False

    def query(self):
        return self.done

    def synchronize(self):
        while not self.done:
            time.sleep(0.001)


class _FakeST:
    """Stands in for a StyleTransfer: each snapshot is a new solid image, its copy complete when the test says."""
    _band = None
    _sync = None

    def __init__(self):
        self.n = 0

    def _snapshot(self, kind, gathered=None):
        raise AssertionError('the test monitor does not launch device work')


class _Probe(WebInterface):
    def __init__(self):
        self.events = []
        super().__init__('127.0.0.1', 0)

    @staticmethod
    def _new_buffer(hw):
        return torch.empty(*hw, 3, dtype=torch.uint8)

    def _copy_snapshot(self, st, target, gathered):
        st.n += 1
        target.fill_(st.n)
        ev = _Event()
        self.events.append(ev)
        return ev


def _value(body):
    return int(round(float(np.asarray(Image.open(io.BytesIO(body))).mean())))


def test_refresh_policy():
    wi, st = _Probe(), _FakeST()
    try:
        wi.put_iterate(_it(1), st)
        assert wi.snapshots == 0                       # nobody has asked for an image yet
        assert _get(wi.url + 'image')[0] == 404         # ... now a client has
        wi.put_iterate(_it(2), st)
        assert wi.snapshots == 1
        wi.put_iterate(_it(3), st)
        assert wi.snapshots == 1                       # never two in flight

        # /image waits for the snapshot in flight (on the server thread), then serves it
        box = []
        t = threading.Thread(target=lambda: box.append(_get(wi.url + 'image')))
        t.start()
        time.sleep(0.1)
        assert t.is_alive()
        wi.events[0].done = True
        t.join(10)
        assert box[0][0] == 200 and _value(box[0][2]) == 1

        wi.put_iterate(_it(4), st)                     # fetched: the next one is due
        assert wi.snapshots == 2
        wi.events[1].done = True
        for i in (5, 6, 7):
            wi.put_iterate(_it(i), st)
        assert wi.snapshots == 2                       # not fetched yet: no new snapshot
        wi.put_iterate(_it(10), st)                    # the last iteration of a scale always takes one
        assert wi.snapshots == 3
        wi.put_iterate(_it(1, i_max=2, w=80, h=60), st)   # next scale, the last snapshot still in flight
        assert wi.snapshots == 3
        wi.put_iterate(_it(2, i_max=2, w=80, h=60), st)   # its last iteration replaces the one in flight
        assert wi.snapshots == 4
        wi.events[3].done = True                       # the replaced copy's event is never consulted
        status, _, body = _get(wi.url + 'image')
        assert status == 200 and _value(body) == 4
        assert Image.open(io.BytesIO(body)).size == (80, 60)
    finally:
        wi.close()


def test_close_with_a_client_connected():
    wi = WebInterface('127.0.0.1', 0)
    port = wi.port
    stop = threading.Event()
    opened = threading.Event()

    async def client():
        async with aiohttp.ClientSession() as s:
            async with s.ws_connect(wi.url + 'websocket') as ws:
                opened.set()
                while not stop.is_set():   # holds the socket and never closes it itself
                    try:
                        await ws.receive(timeout=0.05)
                    except asyncio.TimeoutError:
                        pass
                    if ws.closed:
                        break

    t = threading.Thread(target=lambda: asyncio.run(client()))
    t.start()
    assert opened.wait(5)
    _wait_clients(wi, 1)
    wi.put_iterate(_it(1, 1), torch.rand(3, 8, 8))
    wi.put_done()
    t0 = time.monotonic()
    wi.close()
    took = time.monotonic() - t0
    stop.set()
    t.join(10)
    assert took < 5.0 + 2.0, f'close() took {took:.1f} s'
    assert not _monitor_threads(), _monitor_threads()
    with socket.socket() as s:
        s.bind(('127.0.0.1', port))
    t0 = time.monotonic()
    wi.close()
    assert time.monotonic() - t0 < 0.1


def test_close_without_put_done_is_prompt():
    wi = WebInterface('127.0.0.1', 0)
    t0 = time.monotonic()
    wi.close()
    assert time.monotonic() - t0 < 2.0
    assert not _monitor_threads()
    wi.put_iterate(_it(1), torch.rand(3, 4, 4))   # after close: ignored
    wi.put_done()


def test_cli_web_flags(monkeypatch, tmp_path):
    from style_transfer_b200 import cli
    ap = cli.build_parser()
    args = ap.parse_args(['c.png', 's.png'])
    # the reference CLI's defaults
    assert (args.web, args.host, args.port, args.browser) == (False, '0.0.0.0', 8080, '')
    assert ap.parse_args(['c.png', 's.png', '--browser']).browser is None
    assert ap.parse_args(['c.png', 's.png', '--browser', 'firefox']).browser == 'firefox'
    args = ap.parse_args(['c.png', 's.png', '--web', '--host', '127.0.0.1', '--port', '0'])
    assert (args.web, args.host, args.port) == (True, '127.0.0.1', 0)

    # --web no longer exits: without a device the CLI gets as far as looking for one
    from oracle import st_oracle as O
    monkeypatch.chdir(tmp_path)
    O.synth_image(1, 16, 24, 16).save('c.png')
    O.synth_image(2, 16, 24, 16).save('s.png')
    monkeypatch.setattr(torch.cuda, 'is_available', lambda: False)
    with pytest.raises(SystemExit) as exc:
        cli.main(['c.png', 's.png', '--web', '--host', '127.0.0.1', '--port', '0'])
    assert 'no CUDA device' in str(exc.value)
    assert not _monitor_threads()


def test_web_is_exported_and_lazy():
    assert stb.WebInterface is WebInterface
    import subprocess
    import sys
    code = ('import sys, style_transfer_b200; from style_transfer_b200 import cli; '
            'print("aiohttp" in sys.modules)')
    from pathlib import Path
    root = Path(__file__).resolve().parent.parent
    out = subprocess.run([sys.executable, '-c', code], cwd=root, capture_output=True, text=True, check=True)
    assert out.stdout.strip() == 'False'


def test_switch_interval_is_lowered_while_open_and_restored():
    import sys
    from style_transfer_b200 import web as W
    before = sys.getswitchinterval()
    wi = WebInterface('127.0.0.1', 0)
    try:
        assert sys.getswitchinterval() == min(before, W.SWITCH_INTERVAL_S)
    finally:
        wi.close()
    assert sys.getswitchinterval() == before
