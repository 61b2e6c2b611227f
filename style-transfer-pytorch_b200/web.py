"""Live web monitor of a stylize() run (the CLI's `--web`): a page that shows the current image and the iteration stats.

Routes and wire format are the reference's, so either front-end works against either server:
  /           the page (web_static/index.html)
  /image      the current image as a JPEG (quality 95, 4:4:4, sRGB profile embedded), 404 before the first one
  /websocket  one JSON message per iteration, the STIterate fields plus "_type": "STIterate", and {"_type": "WIDone"}
              at the end
  /<file>     the page's static files

The server is an aiohttp app on a daemon thread with an event loop of its own: no child process, nothing pickled.
put_iterate() is cheap enough to call on every iteration when it is handed the StyleTransfer itself: the monitor then
takes a device snapshot (stb_snapshot, uint8) only when a browser has asked for a newer image than the one it has, and
at the last iteration of every scale.  An untiled snapshot never synchronises the host: the kernel runs on the
iteration stream, its copy into pinned memory on a side stream, and the monitor's encode thread waits for the copy's
event.
"""
from __future__ import annotations

import asyncio
import concurrent.futures
import contextlib
import io
import json
import sys
import threading
import time
from dataclasses import asdict
from pathlib import Path

import numpy as np
from PIL import Image

from .image_io import srgb_profile

STATIC_DIR = Path(__file__).resolve().parent / 'web_static'
THREAD_NAME = 'stb-web'
GRACE_S = 5.0           # connected clients' time to fetch the final image (as the reference's monitor gives them)
JOIN_S = 12.0           # bound on the whole of close(), grace included (the reference joins its process for 12 s)
# Pillow's JPEG encoder holds the GIL for stretches of several ms, and with the default 5 ms switch interval each
# stretch can delay the stylize thread's next launch past the end of the iteration in flight (measured at 2048^2 on an
# H100: 88 % of the unmonitored it/s at 5 ms, 97 % at 0.5 ms; DESIGN.md section 6b).  While a monitor is open the
# interval is at most this; close() restores it.
SWITCH_INTERVAL_S = 5e-4
STOP_S = 4.0            # the part of JOIN_S kept for closing the websockets and releasing the port
WS_CLOSE_S = 1.0        # how long a websocket close waits for the client's answer


def encode_jpeg(hwc_uint8) -> bytes:
    """The JPEG the monitor serves: quality 95, no chroma subsampling, the sRGB profile embedded."""
    buf = io.BytesIO()
    Image.fromarray(np.asarray(hwc_uint8), 'RGB').save(buf, format='jpeg', icc_profile=srgb_profile, quality=95,
                                                       subsampling=0)
    return buf.getvalue()


def message(obj) -> str:
    """A websocket message: the dataclass's fields plus its class name under "_type"."""
    return json.dumps({**asdict(obj), '_type': type(obj).__name__})


class _Image:
    """One image the monitor can serve: an [H, W, 3] uint8 host array (or a [3, H, W] float tensor to quantise), ready
    once `event` (None: at once) has completed.  `jpeg` is the future of its one encode."""
    __slots__ = ('host', 'event', 'jpeg')

    def __init__(self, host, event=None):
        self.host, self.event, self.jpeg = host, event, None

    def pixels(self):
        import torch
        if self.host.dtype == torch.uint8:
            return self.host.numpy()
        # a [3, H, W] float tensor: quantised as torchvision's to_pil_image does
        return self.host.mul(255).byte().permute(1, 2, 0).numpy()


class WebInterface:
    def __init__(self, host, port):
        from aiohttp import web
        self._web = web
        self._lock = threading.Lock()
        self._current = None         # _Image: the newest image whose pixels are (or will be, by its event) on the host
        self._inflight = None        # _Image: a snapshot whose copy has not been seen complete yet (at most one)
        self._wanted = False         # a client has fetched the current image (or found none): take a new one
        self._reading = set()        # ids of pinned buffers an encode is reading
        self._buffers = {}           # (h, w) -> two reusable pinned uint8 buffers
        self._side = {}              # device -> side stream of the device-to-host copies
        self._done = False
        self._closed = False
        self._wss = set()
        self._busy = 0               # /image requests being answered
        self.snapshots = 0           # snapshots taken from a StyleTransfer
        self.encode_times = []       # seconds per JPEG encode
        self._pool = concurrent.futures.ThreadPoolExecutor(1, thread_name_prefix=THREAD_NAME + '-encode')
        self._switch_was = sys.getswitchinterval()
        sys.setswitchinterval(min(self._switch_was, SWITCH_INTERVAL_S))

        self._loop = asyncio.new_event_loop()
        self._outbox = None
        started = concurrent.futures.Future()
        self._thread = threading.Thread(target=self._run, args=(host, port, started), name=THREAD_NAME, daemon=True)
        self._thread.start()
        try:
            self.host, self.port = host, started.result(JOIN_S)
        except BaseException:
            self._thread.join(JOIN_S)
            self._pool.shutdown()
            sys.setswitchinterval(self._switch_was)
            raise
        print(f'Starting web interface at {self.url}')

    @property
    def url(self):
        return f'http://{self.host}:{self.port}/'

    @property
    def clients(self):
        """Number of connected websocket clients."""
        return len(self._wss)

    # ------------------------------------------------------------------ the stylize thread
    def put_iterate(self, iterate, image, *, gathered=None):
        """Send `iterate` to the connected clients and offer a new image.

        `image` is a [3, H, W] float tensor in [0, 1] (copied to the host here, as the reference does), or the
        StyleTransfer being run: then a snapshot of its averaged image is taken only if a client has fetched the current
        one (or found none) and none is in flight, or if this is the last iteration of a scale.  On a scale tiled across
        processes the StyleTransfer cannot gather its image alone: the snapshot is taken only when the caller passes the
        image it has `gathered` on every rank, and quantises that."""
        if self._closed:
            return
        self._offer(image, iterate.i == iterate.i_max, gathered, (iterate.h, iterate.w))
        self._post(message(iterate))

    def put_done(self, image=None):
        """Tell the clients the run is over.  `image` (a tensor or the StyleTransfer after stylize()): the final image,
        when the last put_iterate() could not offer it (a scale tiled across processes)."""
        if self._closed:
            return
        self._offer(image, True, None, None)
        self._done = True
        self._post(json.dumps({'_type': 'WIDone'}))

    def _offer(self, image, last, gathered, hw):
        if image is None:
            return
        if hasattr(image, '_snapshot'):
            self._offer_snapshot(image, last, gathered, hw)
            return
        entry = _Image(image.detach().cpu())
        with self._lock:
            self._current, self._inflight, self._wanted = entry, None, False

    def _post(self, text):
        self._loop.call_soon_threadsafe(self._outbox.put_nowait, text)

    def _offer_snapshot(self, st, last, gathered, hw):
        tiled_apart = st._band is not None and st._sync is None   # tiled across processes: a gather is collective
        if tiled_apart and gathered is None:
            return
        if hw is None:   # after stylize(): the average is whole again
            hw = tuple(st.average.value.shape[-2:])
        with self._lock:
            self._promote()
            due = last or (self._wanted and self._inflight is None) or tiled_apart
            if not due:
                return
            self._wanted = False
            # a snapshot in flight is replaced in its own buffer (the copies are ordered on the side stream); otherwise
            # the other buffer of this size than the current image's.  Until its event is set, nothing reads it.
            inflight = self._inflight
            if inflight is not None and tuple(inflight.host.shape[:2]) == hw:
                target = inflight.host
            else:
                target = self._free_buffer(hw)
            entry = self._inflight = _Image(target)
        try:
            copied = self._copy_snapshot(st, target, gathered)
        except BaseException:
            with self._lock:
                self._inflight = None
            raise
        with self._lock:
            entry.event = copied
            self.snapshots += 1

    def _copy_snapshot(self, st, target, gathered):
        """Launch st's uint8 snapshot and its copy into the pinned `target`; returns the copy's event.  The host waits
        for neither."""
        import torch
        dev = st._dev
        with torch.cuda.device(dev):
            snap = st._snapshot(0) if gathered is None else st._snapshot(0, gathered)
            side = self._side.get(dev)
            if side is None:
                side = self._side[dev] = torch.cuda.Stream(device=dev)
            ready = torch.cuda.Event()
            ready.record(st._stream)           # the snapshot kernel ran on the iteration stream
            side.wait_event(ready)
            with torch.cuda.stream(side):
                target.copy_(snap, non_blocking=True)
            snap.record_stream(side)
            copied = torch.cuda.Event()
            copied.record(side)
        return copied

    def _free_buffer(self, hw):
        """(lock held) The pinned buffer of size hw that holds neither the current image nor one an encode reads."""
        pair = self._buffers.get(hw)
        if pair is None:   # a new scale: the previous size's buffers go once nothing reads them
            pair = [self._new_buffer(hw) for _ in range(2)]
            self._buffers = {hw: pair}
        cur = self._current.host if self._current is not None else None
        k = 1 if pair[0] is cur else 0
        if id(pair[k]) in self._reading:   # a slow encode of an older image: never overwrite it
            pair[k] = self._new_buffer(hw)
        return pair[k]

    @staticmethod
    def _new_buffer(hw):
        import torch
        return torch.empty(*hw, 3, dtype=torch.uint8, pin_memory=True)

    def _promote(self):
        """(lock held) The snapshot in flight becomes the current image once its copy is complete."""
        inflight = self._inflight
        if inflight is not None and inflight.event is not None and inflight.event.query():
            self._current, self._inflight = inflight, None

    # ------------------------------------------------------------------ shutdown
    def close(self):
        """Give connected clients up to GRACE_S to fetch the final image (if put_done() was called), then close their
        websockets, release the port and join the server thread (bounded).  Idempotent."""
        if self._closed:
            return
        self._closed = True
        end = time.monotonic() + JOIN_S
        if self._thread.is_alive():
            fut = asyncio.run_coroutine_threadsafe(self._shutdown(end), self._loop)
            try:
                fut.result(max(end - time.monotonic(), 0.1))
            except Exception:   # noqa: BLE001 -- a server that does not stop in time is still stopped below
                pass
            self._loop.call_soon_threadsafe(self._loop.stop)
            self._thread.join(max(end - time.monotonic(), 0.5))
        self._pool.shutdown(wait=True, cancel_futures=True)
        sys.setswitchinterval(self._switch_was)

    async def _shutdown(self, end):
        """The grace (after put_done), then the websockets' close and the port's release, all before `end`; the grace
        leaves at least STOP_S of it to the rest."""
        if self._done:
            grace_end = min(time.monotonic() + GRACE_S, end - STOP_S)
            with contextlib.suppress(asyncio.TimeoutError):   # WIDone out to every client that takes it
                await asyncio.wait_for(self._outbox.join(), max(grace_end - time.monotonic(), 0))
            while (self._wss or self._busy) and time.monotonic() < grace_end:
                await asyncio.sleep(0.02)

        async def close_quietly(ws):
            with contextlib.suppress(Exception):   # the client is gone either way
                await ws.close()
        with contextlib.suppress(asyncio.TimeoutError):
            await asyncio.wait_for(asyncio.gather(*map(close_quietly, list(self._wss))),
                                   max(end - STOP_S / 2 - time.monotonic(), 0.1))
        await self._runner.cleanup()

    # ------------------------------------------------------------------ the server thread
    def _run(self, host, port, started):
        loop = self._loop
        asyncio.set_event_loop(loop)
        try:
            loop.run_until_complete(self._start(host, port))
        except BaseException as err:  # noqa: BLE001 -- raised by the constructor
            started.set_exception(err)
            loop.close()
            return
        started.set_result(self._runner.addresses[0][1])
        try:
            loop.run_forever()
        finally:
            tasks = [t for t in asyncio.all_tasks(loop) if not t.done()]
            for t in tasks:
                t.cancel()
            loop.run_until_complete(asyncio.gather(*tasks, return_exceptions=True))
            loop.close()

    async def _start(self, host, port):
        web = self._web
        self._outbox = asyncio.Queue()
        app = web.Application()
        app.router.add_routes([web.get('/', self._index), web.get('/image', self._image),
                               web.get('/websocket', self._websocket), web.static('/', STATIC_DIR)])
        self._runner = web.AppRunner(app, handle_signals=False, shutdown_timeout=1.0)
        await self._runner.setup()
        try:
            await web.TCPSite(self._runner, host, port).start()
        except BaseException:
            await self._runner.cleanup()
            raise
        asyncio.get_running_loop().create_task(self._send_loop())

    async def _send_loop(self):
        while True:
            text = await self._outbox.get()
            try:
                for ws in list(self._wss):
                    try:
                        await ws.send_str(text)
                    except Exception:   # noqa: BLE001 -- a client that cannot take a message is dropped, not the loop
                        self._wss.discard(ws)
            finally:
                self._outbox.task_done()

    async def _index(self, request):
        return self._web.Response(body=(STATIC_DIR / 'index.html').read_bytes(), content_type='text/html')

    async def _websocket(self, request):
        ws = self._web.WebSocketResponse(timeout=WS_CLOSE_S)
        await ws.prepare(request)
        self._wss.add(ws)
        try:
            async for _ in ws:
                pass
        finally:
            self._wss.discard(ws)
        return ws

    async def _image(self, request):
        self._busy += 1
        entry = None
        try:
            entry = await self._newest()
            if entry is None:
                raise self._web.HTTPNotFound()
            body = await asyncio.shield(entry.jpeg)
            return self._web.Response(body=body, content_type='image/jpeg')
        finally:
            self._busy -= 1
            with self._lock:   # the client has the newest image there is (or there is none): the next one is due
                if self._current is entry and self._inflight is None:
                    self._wanted = True

    async def _newest(self):
        """The image to serve, with its encode started (once per image) in the critical section that picks it, so that
        no snapshot can take its buffer in between.  A snapshot whose copy is queued on the device is waited for, on
        the encode thread (the wait releases the GIL; it ends at most one iteration's device time later): so the image
        served after WIDone is the final one.  A snapshot the stylize thread is still launching (on a banded scale, a
        gather) is not waited for: the current image is served, or 404 before the first."""
        loop = asyncio.get_running_loop()
        while True:
            with self._lock:
                self._promote()
                event = self._inflight.event if self._inflight is not None else None
                if event is None:
                    entry = self._current
                    if entry is not None and entry.jpeg is None:
                        self._reading.add(id(entry.host))
                        entry.jpeg = loop.run_in_executor(self._pool, self._encode, entry)
                    return entry
            await loop.run_in_executor(self._pool, event.synchronize)

    def _encode(self, entry):
        try:
            t0 = time.perf_counter()
            body = encode_jpeg(entry.pixels())
            self.encode_times.append(time.perf_counter() - t0)
            return body
        finally:
            with self._lock:
                self._reading.discard(id(entry.host))
