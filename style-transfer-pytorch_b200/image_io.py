"""Image input and output of the CLI: colour-managed loading, 16-bit TIFF writing, and saves kept off the optimisation
loop's critical path (SURVEY.md section 8f, row 3).

Loading follows the reference CLI: an input's embedded ICC profile is honoured (converted to sRGB), and `proof=` soft
proofs it through a CMYK profile first.  `.tif`/`.tiff` outputs are written with 16 bits per channel and tagged with the
sRGB profile.

The reference saves synchronously from inside the per-iteration callback (/root/reference/style_transfer/cli.py:125-133):
at 2048^2 the PNG encode alone stalls the loop for hundreds of iterations' worth of device time.  Here the callback only
launches a device-side snapshot of the averaged iterate (stb_snapshot: uint8, or uint16 for a TIFF) and its copy into
pinned host memory; waiting for the copy, encoding and the file write happen on a worker thread, newest snapshot wins.
"""
from __future__ import annotations

import io
import os
import queue
import struct
import sys
import threading
from pathlib import Path

import numpy as np
from PIL import Image, ImageCms

TIFF_SUFFIXES = ('.tif', '.tiff')

# ICC header dateTimeNumber (bytes 24-35: year, month, day, hours, minutes, seconds as big-endian uint16).  LittleCMS
# stamps the creation time there; a fixed stamp makes every run, and every saved file, carry identical profile bytes.
_ICC_DATE = struct.pack('>6H', 2020, 1, 1, 0, 0, 0)


def _make_srgb_profile() -> bytes:
    prof = bytearray(ImageCms.ImageCmsProfile(ImageCms.createProfile('sRGB')).tobytes())
    prof[24:36] = _ICC_DATE
    # profile ID (MD5 over the header with the date included): LittleCMS leaves it zero ("not computed"), which is what
    # keeps the profile valid with the date pinned; it is written as zero so that it stays so
    prof[84:100] = bytes(16)
    return bytes(prof)


srgb_profile = _make_srgb_profile()


# ---------------------------------------------------------------------------------------------------- loading
def _prof_to_prof(image, src_prof: bytes, dst_prof: bytes, **kwargs):
    return ImageCms.profileToProfile(image, io.BytesIO(src_prof), io.BytesIO(dst_prof), **kwargs)


def load_image(path, proof=None):
    """Open `path` as an sRGB PIL image, as the reference CLI's load_image does.

    An embedded ICC profile is the source profile (otherwise sRGB); a source other than sRGB is converted to sRGB.  With
    `proof` (the path of a CMYK ICC profile) the image is soft-proofed: converted to that profile, then back to sRGB.
    Untagged inputs without `proof` are plain `convert('RGB')`.  Errors exit with `Type: message`."""
    try:
        image = Image.open(path)
        icc = image.info.get('icc_profile')
        src_prof = icc or srgb_profile
        if not icc:
            image = image.convert('RGB')
        if proof is None:
            if src_prof == srgb_profile:
                return image.convert('RGB')
            return _prof_to_prof(image, src_prof, srgb_profile, outputMode='RGB')
        proof_prof = Path(proof).read_bytes()
        cmyk = _prof_to_prof(image, src_prof, proof_prof, outputMode='CMYK')
        return _prof_to_prof(cmyk, proof_prof, srgb_profile, outputMode='RGB')
    except (OSError, ImageCms.PyCMSError) as err:
        sys.exit(f'{type(err).__name__}: {err}')


# ---------------------------------------------------------------------------------------------------- 16-bit TIFF
_SHORT, _LONG, _RATIONAL, _UNDEFINED = 3, 4, 5, 7
_STRIP_BYTES = 64 * 1024


def _tiff_head(tags):
    """Little-endian TIFF header, one IFD and its out-of-line values, for tags (tag, type, count, packed value bytes)
    sorted by tag.  Values longer than 4 bytes follow the IFD, each starting on a word boundary."""
    extra_off = 8 + 2 + 12 * len(tags) + 4
    ifd, extra = [struct.pack('<H', len(tags))], b''
    for tag, typ, count, raw in tags:
        if len(raw) <= 4:
            ifd.append(struct.pack('<HHI', tag, typ, count) + raw.ljust(4, b'\0'))
        else:
            ifd.append(struct.pack('<HHII', tag, typ, count, extra_off + len(extra)))
            extra += raw + b'\0' * (len(raw) & 1)
    return b'II' + struct.pack('<HI', 42, 8) + b''.join(ifd) + struct.pack('<I', 0) + extra


def _tiff16_head(h, w, icc_profile):
    """Everything before the pixels of a baseline RGB TIFF, 16 bits per sample, uncompressed, chunky, in strips of about
    64 KiB.  The strips follow the returned bytes back to back, as one [H, W, 3] little-endian uint16 block."""
    row_bytes = w * 3 * 2
    rows_per_strip = max(1, _STRIP_BYTES // row_bytes)
    strips = -(-h // rows_per_strip)
    counts = [min(rows_per_strip, h - s * rows_per_strip) * row_bytes for s in range(strips)]

    def tags(offsets):
        longs = lambda *v: struct.pack(f'<{len(v)}I', *v)   # noqa: E731
        shorts = lambda *v: struct.pack(f'<{len(v)}H', *v)  # noqa: E731
        return [(256, _LONG, 1, longs(w)), (257, _LONG, 1, longs(h)), (258, _SHORT, 3, shorts(16, 16, 16)),
                (259, _SHORT, 1, shorts(1)),                       # no compression
                (262, _SHORT, 1, shorts(2)),                       # RGB
                (273, _LONG, strips, longs(*offsets)), (277, _SHORT, 1, shorts(3)),
                (278, _LONG, 1, longs(rows_per_strip)), (279, _LONG, strips, longs(*counts)),
                (282, _RATIONAL, 1, longs(72, 1)), (283, _RATIONAL, 1, longs(72, 1)),
                (284, _SHORT, 1, shorts(1)),                       # chunky
                (296, _SHORT, 1, shorts(2)),                       # inch
                (34675, _UNDEFINED, len(icc_profile), icc_profile)]

    # the header's length does not depend on the offsets' values: size it once, then fill them in
    data_off = len(_tiff_head(tags([0] * strips)))
    data_off += -data_off % 16
    if data_off + sum(counts) >= 1 << 32:
        raise ValueError(f'a {w} x {h} 16-bit RGB image does not fit a baseline TIFF (4 GiB)')
    offsets = [data_off + s * counts[0] for s in range(strips)]
    return _tiff_head(tags(offsets)).ljust(data_off, b'\0')


def write_tiff16(path, hwc_uint16, icc_profile):
    """Write an [H, W, 3] uint16 array as a 16-bit RGB TIFF carrying `icc_profile` (tag 34675, InterColorProfile) and
    a 72 dpi resolution, as the reference CLI's save_tiff does.  Written to a `.part` file first, then renamed, so that
    readers never see a half-written file."""
    arr = np.asarray(hwc_uint16)
    if arr.ndim != 3 or arr.shape[2] != 3 or arr.dtype != np.uint16:
        raise ValueError(f'write_tiff16 takes an [H, W, 3] uint16 array, not {arr.dtype} {arr.shape}')
    h, w, _ = arr.shape
    head = _tiff16_head(h, w, bytes(icc_profile))
    path = Path(path)
    tmp = path.with_name(path.stem + '.part' + path.suffix)
    with open(tmp, 'wb') as fp:
        fp.write(head)
        fp.write(np.ascontiguousarray(arr, dtype='<u2').data)
    os.replace(tmp, path)


# ---------------------------------------------------------------------------------------------------- async saves
class AsyncImageWriter:
    def __init__(self):
        self._q: queue.Queue = queue.Queue()
        self._errors: list[BaseException] = []
        self._thread = threading.Thread(target=self._run, name='stb-image-writer', daemon=True)
        self._thread.start()

    # ------------------------------------------------------------------ producer side (the stylize callback)
    def submit_snapshot(self, st, path, gathered=None):
        """Snapshot `st`'s current averaged image on the device and queue it for saving to `path`: 16 bits per channel
        for `.tif`/`.tiff`, 8 otherwise.  On an untiled scale this does not wait for the device.  `gathered`: the image
        st.get_image_tensor() has already returned at this iteration, saved instead of gathering it again."""
        import torch
        path = Path(path)
        snap = st._snapshot(1 if path.suffix.lower() in TIFF_SUFFIXES else 0, gathered)
        stream = st._stream
        host = torch.empty(snap.shape, dtype=snap.dtype, pin_memory=True)
        with torch.cuda.stream(stream):
            stream.wait_stream(torch.cuda.current_stream(snap.device))
            host.copy_(snap, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(stream)
        self._q.put((host, ev, path))

    def submit_array(self, array: np.ndarray, path):
        self._q.put((array, None, Path(path)))

    # ------------------------------------------------------------------ worker
    def _run(self):
        while True:
            item = self._q.get()
            if item is None:
                return
            while True:  # newest snapshot for the same path wins; never fall behind the loop
                try:
                    nxt = self._q.get_nowait()
                except queue.Empty:
                    break
                if nxt is None:
                    self._save(item)
                    return
                if nxt[2] != item[2]:
                    self._save(item)
                item = nxt
            self._save(item)

    def _save(self, item):
        host, ev, path = item
        try:
            if ev is not None:
                ev.synchronize()
            arr = host.numpy() if hasattr(host, 'numpy') else np.asarray(host)
            if path.suffix.lower() in TIFF_SUFFIXES:
                write_tiff16(path, arr, srgb_profile)
                return
            tmp = path.with_name(path.stem + '.part' + path.suffix)
            Image.fromarray(arr).save(tmp)
            os.replace(tmp, path)                                   # readers never see a half-written file
        except BaseException as err:  # noqa: BLE001 - reported by close()
            self._errors.append(err)

    def close(self):
        """Flush pending saves; re-raises the first error of the worker, if any."""
        self._q.put(None)
        self._thread.join()
        if self._errors:
            raise self._errors[0]
