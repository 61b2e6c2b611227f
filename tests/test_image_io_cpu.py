"""Image I/O of the CLI without a GPU: the 16-bit TIFF writer, the pinned sRGB profile, colour-managed loading and
soft proofing (image_io.py), and the CLI's parser."""
from __future__ import annotations

import io
import struct
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
from PIL import Image, ImageCms

import icc_profiles
import style_transfer_b200 as stb
from style_transfer_b200 import cli, image_io
from style_transfer_b200.image_io import load_image, srgb_profile, write_tiff16

ROOT = Path(__file__).resolve().parents[1]
TYPE_SIZE = {1: 1, 2: 1, 3: 2, 4: 4, 5: 8, 7: 1}


def parse_tiff(data):
    """{tag: tuple of values (bytes for UNDEFINED / BYTE)} of the first IFD of a little-endian TIFF."""
    assert data[:4] == b'II*\0'
    (ifd,) = struct.unpack_from('<I', data, 4)
    (n,) = struct.unpack_from('<H', data, ifd)
    tags, last = {}, 0
    for k in range(n):
        tag, typ, count, raw = struct.unpack_from('<HHI4s', data, ifd + 2 + 12 * k)
        assert tag > last, 'IFD entries must be sorted by tag'
        last = tag
        size = TYPE_SIZE[typ] * count
        if size > 4:
            (off,) = struct.unpack('<I', raw)
            assert off % 2 == 0, f'tag {tag}: values must start on a word boundary'
            raw = data[off:off + size]
        raw = raw[:size]
        if typ in (1, 7):
            tags[tag] = bytes(raw)
        elif typ == 3:
            tags[tag] = struct.unpack(f'<{count}H', raw)
        elif typ == 4:
            tags[tag] = struct.unpack(f'<{count}I', raw)
        elif typ == 5:
            tags[tag] = tuple(zip(*[iter(struct.unpack(f'<{2 * count}I', raw))] * 2))
    assert struct.unpack_from('<I', data, ifd + 2 + 12 * n) == (0,)
    return tags


@pytest.mark.parametrize('h,w', [(1, 1), (7, 9), (181, 136), (700, 333)])
def test_write_tiff16_round_trip(tmp_path, h, w):
    rng = np.random.default_rng(h * 1000 + w)
    arr = rng.integers(0, 65536, (h, w, 3), dtype=np.uint16)
    arr.reshape(-1)[:2] = (0, 65535)
    path = tmp_path / 'x.tif'
    write_tiff16(path, arr, srgb_profile)
    assert not (tmp_path / 'x.part.tif').exists()
    data = path.read_bytes()
    tags = parse_tiff(data)
    assert tags[256] == (w,) and tags[257] == (h,)
    assert tags[258] == (16, 16, 16) and tags[259] == (1,) and tags[262] == (2,) and tags[277] == (3,)
    assert tags[284] == (1,) and tags[296] == (2,)
    assert tags[282] == ((72, 1),) and tags[283] == ((72, 1),)
    assert tags[34675] == srgb_profile
    rows = tags[278][0]
    offsets, counts = tags[273], tags[279]
    assert len(offsets) == len(counts) == -(-h // rows)
    assert all(c <= max(64 * 1024, w * 6) for c in counts) and sum(counts) == h * w * 6
    if h == 700:
        assert len(offsets) > 2
    strips = b''.join(data[o:o + c] for o, c in zip(offsets, counts))
    np.testing.assert_array_equal(np.frombuffer(strips, '<u2').reshape(h, w, 3), arr)
    cv2 = pytest.importorskip('cv2')
    back = cv2.imread(str(path), cv2.IMREAD_UNCHANGED)
    assert back is not None and back.dtype == np.uint16
    np.testing.assert_array_equal(back.reshape(h, w, 3)[..., ::-1], arr)


def test_write_tiff16_rejects_other_arrays(tmp_path):
    with pytest.raises(ValueError):
        write_tiff16(tmp_path / 'x.tif', np.zeros((4, 4, 3), np.uint8), srgb_profile)
    with pytest.raises(ValueError):
        write_tiff16(tmp_path / 'x.tif', np.zeros((4, 4), np.uint16), srgb_profile)


def test_srgb_profile():
    assert stb.srgb_profile is srgb_profile
    prof = ImageCms.ImageCmsProfile(io.BytesIO(srgb_profile))
    assert 'sRGB' in ImageCms.getProfileDescription(prof)
    assert srgb_profile[36:40] == b'acsp' and struct.unpack('>I', srgb_profile[:4])[0] == len(srgb_profile)
    assert srgb_profile[84:100] == bytes(16)   # profile ID "not computed": the pinned date leaves it valid
    code = 'import sys; import style_transfer_b200 as s; sys.stdout.write(s.srgb_profile.hex())'
    runs = [subprocess.run([sys.executable, '-c', code], cwd=ROOT, capture_output=True, text=True, check=True).stdout
            for _ in range(2)]
    assert runs[0] == runs[1] == srgb_profile.hex()


def _photo(h=48, w=64):
    y, x = np.mgrid[0:h, 0:w]
    arr = np.stack([x * 255 // (w - 1), y * 255 // (h - 1), (x + y) * 255 // (w + h - 2)], -1).astype(np.uint8)
    arr[:4, :4] = (255, 0, 0)
    arr[-4:, -4:] = (0, 0, 255)
    return arr


def _p2p(image, src, dst, mode):
    return ImageCms.profileToProfile(image, io.BytesIO(src), io.BytesIO(dst), outputMode=mode)


def test_load_image_untagged_is_plain_convert(tmp_path):
    p = tmp_path / 'plain.png'
    Image.fromarray(_photo()).save(p)
    got = load_image(p)
    assert got.mode == 'RGB'
    assert got.tobytes() == Image.open(p).convert('RGB').tobytes()
    p2 = tmp_path / 'pal.png'
    Image.fromarray(_photo()).convert('P').save(p2)
    assert load_image(p2).tobytes() == Image.open(p2).convert('RGB').tobytes()


def test_load_image_converts_tagged_input_to_srgb(tmp_path):
    wide = icc_profiles.wide_gamut_rgb()
    p = tmp_path / 'wide.png'
    Image.fromarray(_photo()).save(p, icc_profile=wide)
    got = load_image(p)
    want = _p2p(Image.open(p), wide, srgb_profile, 'RGB')
    assert got.mode == 'RGB' and got.tobytes() == want.tobytes()
    plain = np.asarray(Image.open(p).convert('RGB'), dtype=int)
    assert np.abs(np.asarray(got, dtype=int) - plain).max() > 20
    # a file tagged with the sRGB profile itself is a plain convert
    p2 = tmp_path / 'srgb.png'
    Image.fromarray(_photo()).save(p2, icc_profile=srgb_profile)
    assert load_image(p2).tobytes() == Image.open(p2).convert('RGB').tobytes()


def test_load_image_soft_proof(tmp_path):
    cmyk = tmp_path / 'narrow.icc'
    cmyk.write_bytes(icc_profiles.narrow_cmyk())
    p = tmp_path / 'plain.png'
    Image.fromarray(_photo()).save(p)
    got = load_image(p, proof=str(cmyk))
    proof = cmyk.read_bytes()
    mid = _p2p(Image.open(p).convert('RGB'), srgb_profile, proof, 'CMYK')
    want = _p2p(mid, proof, srgb_profile, 'RGB')
    assert got.mode == 'RGB' and got.tobytes() == want.tobytes()
    arr = np.asarray(got, dtype=int)
    assert np.abs(arr - _photo()).max() > 20
    assert arr[:4, :4, 1].min() > 0   # pure red leaves the narrow gamut: the proof desaturates it
    # a tagged input goes source profile -> proof -> sRGB
    wide = icc_profiles.wide_gamut_rgb()
    p2 = tmp_path / 'wide.png'
    Image.fromarray(_photo()).save(p2, icc_profile=wide)
    want2 = _p2p(_p2p(Image.open(p2), wide, proof, 'CMYK'), proof, srgb_profile, 'RGB')
    assert load_image(p2, proof=cmyk).tobytes() == want2.tobytes()


def test_load_image_errors_exit_with_the_error(tmp_path):
    with pytest.raises(SystemExit) as e:
        load_image(tmp_path / 'missing.png')
    assert str(e.value).startswith('FileNotFoundError: ') and 'missing.png' in str(e.value)
    bad = tmp_path / 'bad.png'
    bad.write_bytes(b'not an image')
    with pytest.raises(SystemExit) as e:
        load_image(bad)
    assert str(e.value).startswith('UnidentifiedImageError: ')
    good = tmp_path / 'ok.png'
    Image.fromarray(_photo()).save(good)
    with pytest.raises(SystemExit) as e:
        load_image(good, proof=tmp_path / 'missing.icc')
    assert str(e.value).startswith('FileNotFoundError: ')


def test_cli_parser_accepts_tiff_and_proof():
    args = cli.build_parser().parse_args(['c.png', 's.png', '-o', 'x.tif', '--proof', 'p.icc'])
    assert args.output == 'x.tif' and args.proof == 'p.icc'
    assert image_io.TIFF_SUFFIXES == ('.tif', '.tiff')
