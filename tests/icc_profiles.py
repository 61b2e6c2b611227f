"""Small ICC v2 profiles built in the tests, for the colour-managed loading of image_io.load_image.

No ICC profile other than LittleCMS's built-in ones is available to the tests, so the two kinds they need are written
here with numpy and struct:
  * wide_gamut_rgb(): an Adobe RGB (1998)-like display profile, matrix/TRC (rXYZ/gXYZ/bXYZ, curv TRCs, wtpt, desc);
  * narrow_cmyk(): an output ('prtr') profile, CMYK <-> Lab through lut16 tables (A2B0 on a 5-point grid, B2A0 on a
    9-point grid).  Its gamut is sRGB squeezed into [0.05, 0.95] per channel, so a soft proof through it visibly
    flattens the image: no channel of the round trip reaches 255.
"""
from __future__ import annotations

import struct

import numpy as np

D50 = np.array([0.9642, 1.0, 0.8249])
# sRGB primaries adapted to D50 (Bradford), the columns of the linear-RGB -> XYZ(D50) matrix
SRGB_D50 = np.array([[0.4361, 0.3851, 0.1431], [0.2225, 0.7169, 0.0606], [0.0139, 0.0971, 0.7141]])
ADOBE_D50 = np.array([[0.6097, 0.2053, 0.1492], [0.3111, 0.6257, 0.0632], [0.0195, 0.0609, 0.7446]])


def _s15(x):
    return struct.pack('>i', int(round(float(x) * 65536)))


def _xyz_tag(xyz):
    return b'XYZ ' + bytes(4) + b''.join(_s15(v) for v in xyz)


def _desc_tag(text):
    a = text.encode('ascii') + b'\0'
    return b'desc' + bytes(4) + struct.pack('>I', len(a)) + a + struct.pack('>II', 0, 0) + struct.pack('>HB', 0, 0) + bytes(67)


def _text_tag(text):
    return b'text' + bytes(4) + text.encode('ascii') + b'\0'


def _curv_gamma(gamma):
    return b'curv' + bytes(4) + struct.pack('>IH', 1, int(round(gamma * 256))) + bytes(2)


def _lut16(clut, n_in, n_out, grid):
    """lut16Type with identity matrix, identity 2-entry input / output tables and `clut` ([grid]*n_in + [n_out],
    values already in 0..65535, first input channel varying slowest)."""
    eye = b''.join(_s15(1.0 if i == j else 0.0) for i in range(3) for j in range(3))
    head = b'mft2' + bytes(4) + struct.pack('>BBBB', n_in, n_out, grid, 0) + eye + struct.pack('>HH', 2, 2)
    ident = struct.pack('>HH', 0, 65535)
    body = np.clip(np.rint(clut), 0, 65535).astype('>u2').reshape(-1).tobytes()
    return head + ident * n_in + body + ident * n_out


def _profile(cls, space, pcs, tags):
    """Header + tag table + tag data (each tag 4-byte aligned)."""
    table, data = [], b''
    off = 128 + 4 + 12 * len(tags)
    for sig, body in tags:
        table.append(sig.encode('ascii') + struct.pack('>II', off + len(data), len(body)))
        data += body + bytes(-len(body) % 4)
    size = off + len(data)
    header = (struct.pack('>I', size) + bytes(4) + struct.pack('>I', 0x02100000) + cls.encode() + space.encode() +
              pcs.encode() + struct.pack('>6H', 2020, 1, 1, 0, 0, 0) + b'acsp' + bytes(28) +   # platform .. rendering intent
              b''.join(_s15(v) for v in D50) + bytes(4) + bytes(16))                   # illuminant, creator, ID
    header = header.ljust(128, b'\0')
    assert len(header) == 128
    return header + struct.pack('>I', len(tags)) + b''.join(table) + data


def wide_gamut_rgb():
    tags = [('desc', _desc_tag('test wide-gamut RGB')), ('cprt', _text_tag('no copyright')), ('wtpt', _xyz_tag(D50)),
            ('rXYZ', _xyz_tag(ADOBE_D50[:, 0])), ('gXYZ', _xyz_tag(ADOBE_D50[:, 1])),
            ('bXYZ', _xyz_tag(ADOBE_D50[:, 2])),
            ('rTRC', _curv_gamma(2.2)), ('gTRC', _curv_gamma(2.2)), ('bTRC', _curv_gamma(2.2))]
    return _profile('mntr', 'RGB ', 'XYZ ', tags)


# ---------------------------------------------------------------------------------------------------- CMYK <-> Lab
def _srgb_to_lab(rgb):
    lin = np.where(rgb <= 0.04045, rgb / 12.92, ((rgb + 0.055) / 1.055) ** 2.4)
    t = (lin @ SRGB_D50.T) / D50
    f = np.where(t > (6 / 29) ** 3, np.cbrt(t), t / (3 * (6 / 29) ** 2) + 4 / 29)
    return np.stack([116 * f[..., 1] - 16, 500 * (f[..., 0] - f[..., 1]), 200 * (f[..., 1] - f[..., 2])], -1)


def _lab_to_srgb(lab):
    fy = (lab[..., 0] + 16) / 116
    f = np.stack([fy + lab[..., 1] / 500, fy, fy - lab[..., 2] / 200], -1)
    t = np.where(f > 6 / 29, f ** 3, 3 * (6 / 29) ** 2 * (f - 4 / 29))
    lin = np.clip((t * D50) @ np.linalg.inv(SRGB_D50).T, 0, 1)
    return np.where(lin <= 0.0031308, lin * 12.92, 1.055 * lin ** (1 / 2.4) - 0.055)


def _lab_encode(lab):   # ICC v2 16-bit Lab: L 0..100 -> 0..0xFF00, a/b -128..127.996 -> 0..0xFFFF
    return np.stack([lab[..., 0] * 0xFF00 / 100, (lab[..., 1] + 128) * 256, (lab[..., 2] + 128) * 256], -1)


def _lab_decode(v):
    return np.stack([v[..., 0] * 100 / 0xFF00, v[..., 1] / 256 - 128, v[..., 2] / 256 - 128], -1)


LO, HI = 0.05, 0.95   # the CMYK gamut: sRGB channels in [LO, HI]


def narrow_cmyk():
    g = np.linspace(0, 1, 5)
    c, m, y, k = np.meshgrid(g, g, g, g, indexing='ij')
    rgb = LO + (HI - LO) * np.stack([(1 - c) * (1 - k), (1 - m) * (1 - k), (1 - y) * (1 - k)], -1)
    a2b = _lab_encode(_srgb_to_lab(rgb))
    g9 = np.linspace(0, 65535, 9)
    lab = _lab_decode(np.stack(np.meshgrid(g9, g9, g9, indexing='ij'), -1))
    rgb = (np.clip(_lab_to_srgb(lab), LO, HI) - LO) / (HI - LO)
    b2a = np.concatenate([1 - rgb, np.zeros(rgb.shape[:-1] + (1,))], -1) * 65535
    tags = [('desc', _desc_tag('test narrow CMYK')), ('cprt', _text_tag('no copyright')), ('wtpt', _xyz_tag(D50)),
            ('A2B0', _lut16(a2b, 4, 3, 5)), ('B2A0', _lut16(b2a, 3, 4, 9))]
    return _profile('prtr', 'CMYK', 'Lab ', tags)
