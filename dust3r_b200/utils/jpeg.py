"""Header side of the GPU JPEG decoder (csrc/jpeg_ops.cu): a marker parser for SOI ... SOS that fills the `d3r_jpeg_desc` the
kernels read, and decides per file whether the device decoder reproduces Pillow exactly.  Only baseline sequential Huffman files
are accepted (SOF0, or SOF1 at 8 bits), one interleaved scan holding every component, 1 component or 3 YCbCr components at
4:4:4, 4:2:2 or 4:2:0.  Anything else (progressive, arithmetic, 12-bit, CMYK / YCCK, RGB-coded, Adobe transforms other than
YCbCr, other sampling, malformed tables) is reported with the reason, and the caller decodes that file with Pillow.

The EXIF orientation is the one `PIL.ImageOps.exif_transpose` applies: it is read with Pillow's own header parsing (Image.open
reads the markers up to SOS and decodes nothing), so that the EXIF / XMP rules the device path follows cannot differ from
Pillow's."""
from __future__ import annotations

import io
import struct

import numpy as np

from .image import Unsupported, oriented_size

# jutils.c jpeg_natural_order
NATURAL = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                    21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                    60, 61, 54, 47, 55, 62, 63])


def _huff_table(counts, symbols, is_dc):
    """jdhuff.c jpeg_make_d_derived_tbl as (maxcode[18], valoff[18], look[512], val[256]); raises Unsupported on a table
    libjpeg would reject or one with DC categories above 11."""
    if sum(counts) > 256 or len(symbols) != sum(counts):
        raise Unsupported('bad Huffman table')
    if is_dc and any(s > 11 for s in symbols):
        raise Unsupported('DC category above 11')
    maxcode = [-1] * 18
    valoff = [0] * 18
    look = np.zeros(512, dtype=np.uint16)
    code, k = 0, 0
    for length in range(1, 17):
        n = counts[length - 1]
        if n:
            valoff[length] = k - code
            for _ in range(n):
                if length <= 9:
                    shift = 9 - length
                    look[code << shift:(code + 1) << shift] = (length << 8) | symbols[k]
                code += 1
                k += 1
            maxcode[length] = code - 1
        if code >= (1 << length):
            raise Unsupported('bad Huffman table')      # libjpeg: code space overflow
        code <<= 1
    val = np.zeros(256, dtype=np.uint8)
    val[:len(symbols)] = symbols
    return maxcode, valoff, look, val


def parse(data):
    """Marker parser for SOI ... SOS -> dict(width, height, comps [(id, h, v, tq)], scan [(comp index, td, ta)], qt {id: 64
    zig-zag values}, dc / ac {id: table}, restart, scan_begin).  Raises Unsupported for files outside the device decoder's set."""
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise Unsupported('not a JPEG file')
    pos = 2
    qt, dc, ac = {}, {}, {}
    frame = None
    restart = 0
    jfif = adobe = False
    adobe_transform = None
    while True:
        while pos < n and data[pos] != 0xFF:
            pos += 1                                     # libjpeg skips garbage before a marker (with a warning)
        while pos < n and data[pos] == 0xFF:
            pos += 1
        if pos + 2 >= n:
            raise Unsupported('no SOS marker')
        marker = data[pos]
        pos += 1
        if marker in (0x01,) or 0xD0 <= marker <= 0xD7:
            continue
        if marker == 0xD9:
            raise Unsupported('no SOS marker')
        length = struct.unpack('>H', data[pos:pos + 2])[0]
        seg = data[pos + 2:pos + length]
        if length < 2 or len(seg) != length - 2:
            raise Unsupported('truncated marker segment')
        pos += length
        if marker == 0xDB:                               # DQT
            i = 0
            while i < len(seg):
                pq, tq = seg[i] >> 4, seg[i] & 15
                size = 128 if pq else 64
                if tq > 3 or i + 1 + size > len(seg):
                    raise Unsupported('bad DQT')
                vals = np.frombuffer(bytes(seg[i + 1:i + 1 + size]), dtype='>u2' if pq else np.uint8).astype(np.uint16)
                qt[tq] = vals
                i += 1 + size
        elif marker == 0xC4:                             # DHT
            i = 0
            while i < len(seg):
                if i + 17 > len(seg):
                    raise Unsupported('bad DHT')
                tc, th = seg[i] >> 4, seg[i] & 15
                counts = list(seg[i + 1:i + 17])
                total = sum(counts)
                if tc > 1 or th > 3 or i + 17 + total > len(seg):
                    raise Unsupported('bad DHT')
                symbols = list(seg[i + 17:i + 17 + total])
                (ac if tc else dc)[th] = _huff_table(counts, symbols, tc == 0)
                i += 17 + total
        elif marker == 0xDD:                             # DRI
            if len(seg) < 2:
                raise Unsupported('bad DRI')
            restart = struct.unpack('>H', seg[:2])[0]
        elif marker == 0xE0 and seg[:5] == b'JFIF\0':
            jfif = True
        elif marker == 0xEE and seg[:5] == b'Adobe' and len(seg) >= 12:
            adobe, adobe_transform = True, seg[11]
        elif marker in (0xC0, 0xC1):                     # SOF0 / SOF1
            if len(seg) < 6:
                raise Unsupported('bad SOF')
            precision, height, width, nf = seg[0], *struct.unpack('>HH', seg[1:5]), seg[5]
            if precision != 8:
                raise Unsupported(f'{precision}-bit samples')
            if nf not in (1, 3) or len(seg) < 6 + 3 * nf:
                raise Unsupported(f'{nf} components')
            if width == 0 or height == 0:
                raise Unsupported('no frame size (DNL)')
            comps = [(seg[6 + 3 * i], seg[7 + 3 * i] >> 4, seg[7 + 3 * i] & 15, seg[8 + 3 * i]) for i in range(nf)]
            frame = (width, height, comps)
        elif 0xC2 <= marker <= 0xCF and marker not in (0xC4, 0xC8, 0xCC):
            raise Unsupported(f'SOF{marker - 0xC0}: not baseline sequential Huffman')
        elif marker == 0xDA:                             # SOS
            if frame is None:
                raise Unsupported('SOS before SOF')
            width, height, comps = frame
            ns = seg[0] if seg else 0
            if ns != len(comps) or len(seg) != 4 + 2 * ns:
                raise Unsupported('scan does not hold every component')
            ids = [c[0] for c in comps]
            scan = []
            for i in range(ns):
                cid, tables = seg[1 + 2 * i], seg[2 + 2 * i]
                if cid not in ids or ids.index(cid) != i:
                    raise Unsupported('scan components out of frame order')
                scan.append((i, tables >> 4, tables & 15))
            if tuple(seg[1 + 2 * ns:4 + 2 * ns]) != (0, 63, 0):
                raise Unsupported('not a sequential scan')
            if len(comps) == 3:
                if jfif:
                    ycc = True
                elif adobe:
                    ycc = adobe_transform == 1
                else:
                    ycc = tuple(ids) != (82, 71, 66)
                if not ycc:
                    raise Unsupported('colour space is not YCbCr')
                samp = tuple((h, v) for _, h, v, _ in comps)
                if samp not in (((1, 1),) * 3, ((2, 1), (1, 1), (1, 1)), ((2, 2), (1, 1), (1, 1))):
                    raise Unsupported(f'sampling {samp}')
            elif (comps[0][1], comps[0][2]) != (1, 1):
                raise Unsupported('grey sampling other than 1x1')
            for i, (_, _, _, tq) in enumerate(comps):
                if tq not in qt:
                    raise Unsupported('missing quantisation table')
            for _, td, ta in scan:
                if td not in dc or ta not in ac:
                    raise Unsupported('missing Huffman table')
            return dict(width=width, height=height, comps=comps, scan=scan, qt=qt, dc=dc, ac=ac, restart=restart, scan_begin=pos)


def orientation(data):
    """The EXIF orientation exif_transpose would apply (1 when there is none, or an invalid one)."""
    import PIL.Image
    with PIL.Image.open(io.BytesIO(data)) as img:
        o = img.getexif().get(0x0112, 1)
    return int(o) if o in (2, 3, 4, 5, 6, 7, 8) else 1


def descriptor(header, orient=1):
    """dust3r_b200._lib.JpegDesc of a parsed header."""
    from .. import _lib
    d = _lib.JpegDesc()
    d.width, d.height = header['width'], header['height']
    d.n_comp = len(header['comps'])
    d.restart_interval = header['restart']
    d.orientation = orient
    d.scan_begin = header['scan_begin']
    for i, (_, h, v, tq) in enumerate(header['comps']):
        d.h_samp[i], d.v_samp[i] = h, v
        nat = np.zeros(64, dtype=np.uint16)
        nat[NATURAL] = header['qt'][tq]
        d.quant[i][:] = nat.tolist()
    for i, td, ta in header['scan']:
        d.dc_table[i], d.ac_table[i] = td, ta
    for slot, tables in ((0, header['dc']), (4, header['ac'])):
        for tid, (maxcode, valoff, look, val) in tables.items():
            t = d.huff[slot + tid]
            t.maxcode[:] = maxcode
            t.valoff[:] = valoff
            t.look[:] = look.tolist()
            t.val[:] = val.tolist()
    return d


def stage(data):
    """(descriptor, oriented (width, height), payload) of a file the device decoder takes; the payload is the whole file.
    Raises Unsupported for the others."""
    head = parse(data)
    orient = orientation(data)
    return descriptor(head, orient), oriented_size(head, orient), data
