"""Header side of the GPU PNG decoder (csrc/png_ops.cu): a chunk walker that checks every chunk's CRC, collects IHDR, PLTE,
tRNS and the IDAT payloads, fills the `d3r_png_desc` the kernels read, and decides per file whether the device decoder
reproduces Pillow exactly.  Only non-interlaced 8-bit files of colour type 0 (grey), 2 (RGB), 3 (palette), 4 (grey + alpha) or 6
(RGBA) are accepted, with a zlib stream of method 8, a window of at most 32 KiB and no preset dictionary.  Anything else
(Adam7, bit depths 1, 2, 4 and 16, APNG, a CRC mismatch, a missing IEND, IDAT chunks that are not consecutive, an image above
PIL.Image.MAX_IMAGE_PIXELS, a chunk type the walker does not know) is reported with the reason, and the caller decodes that
file with Pillow.

The EXIF orientation is the one `PIL.ImageOps.exif_transpose` applies.  For a PNG, Pillow may load the whole image to find an
eXIf chunk after the pixel data, so it is not asked about the file itself: it reads a stand-in made of the file's ancillary
chunks, in their places, around a 1x1 image.  Pillow's own eXIf, "Raw profile type exif" and XMP rules then give the
orientation, and no pixels of the file are decoded on the host."""
from __future__ import annotations

import ctypes
import io
import struct
import zlib

import numpy as np

from .image import Unsupported, oriented_size

SIGNATURE = b'\x89PNG\r\n\x1a\n'
_BPP = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
# ancillary chunks of the PNG specification; they travel to the orientation stand-in unchanged
_ANCILLARY = {b'cHRM', b'gAMA', b'iCCP', b'sBIT', b'sRGB', b'bKGD', b'hIST', b'pHYs', b'sPLT', b'tIME', b'iTXt', b'tEXt',
              b'zTXt', b'eXIf', b'cICP', b'mDCv', b'cLLi'}


def parse(data):
    """Chunk walker -> dict(width, height, color_type, palette (n, 3) uint8 or None, idat (bytes of the concatenated IDAT
    payloads), before / after (the ancillary chunks before / after the image data, as (type, payload) pairs), trns).
    Raises Unsupported for files outside the device decoder's set."""
    import PIL.Image
    n = len(data)
    if n < 8 or data[:8] != SIGNATURE:
        raise Unsupported('not a PNG file')
    pos = 8
    head = None
    palette = None
    trns = None
    idat = []
    before, after = [], []
    seen_idat = ended_idat = False
    while True:
        if pos + 8 > n:
            raise Unsupported('no IEND chunk')
        length, ctype = struct.unpack('>I4s', data[pos:pos + 8])
        if pos + 12 + length > n:
            raise Unsupported('truncated chunk')
        body = data[pos + 8:pos + 8 + length]
        crc = struct.unpack('>I', data[pos + 8 + length:pos + 12 + length])[0]
        if zlib.crc32(body, zlib.crc32(ctype)) != crc:
            raise Unsupported(f'CRC mismatch in {ctype!r}')
        pos += 12 + length
        if head is None and ctype != b'IHDR':
            raise Unsupported('IHDR is not the first chunk')
        if ctype == b'IHDR':
            if head is not None or length != 13:
                raise Unsupported('bad IHDR')
            width, height, depth, color, method, filt, interlace = struct.unpack('>IIBBBBB', body)
            if interlace != 0:
                raise Unsupported('interlaced (Adam7)')
            if depth != 8:
                raise Unsupported(f'bit depth {depth}')
            if color not in _BPP:
                raise Unsupported(f'colour type {color}')
            if method != 0 or filt != 0 or width == 0 or height == 0:
                raise Unsupported('bad IHDR')
            if PIL.Image.MAX_IMAGE_PIXELS is not None and width * height > PIL.Image.MAX_IMAGE_PIXELS:
                raise Unsupported('more pixels than PIL.Image.MAX_IMAGE_PIXELS')
            if (1 + width * _BPP[color]) * height >= (1 << 31) - 1:
                raise Unsupported('image rows of 2 GiB or more')
            head = (width, height, color)
        elif ctype == b'IDAT':
            if ended_idat:
                raise Unsupported('IDAT chunks are not consecutive')
            seen_idat = True
            idat.append(body)
        elif ctype == b'IEND':
            break
        else:
            ended_idat = seen_idat
            if ctype == b'PLTE':
                if seen_idat or palette is not None or length % 3 or not 3 <= length <= 768:
                    raise Unsupported('bad PLTE')
                palette = np.frombuffer(body, dtype=np.uint8).reshape(-1, 3)
            elif ctype == b'tRNS':
                if seen_idat:
                    raise Unsupported('tRNS after the image data')
                trns = body
            elif ctype in _ANCILLARY:
                (after if seen_idat else before).append((ctype, body))
            else:
                raise Unsupported(f'chunk {ctype!r}')
    if not idat:
        raise Unsupported('no IDAT chunk')
    width, height, color = head
    if color == 3 and palette is None:
        raise Unsupported('palette image without PLTE')
    if trns is not None and not (len(trns) == {0: 2, 2: 6}.get(color) or (color == 3 and len(trns) <= len(palette))):
        raise Unsupported('tRNS of another length than its colour type allows')
    stream = b''.join(idat)
    if len(stream) < 6:
        raise Unsupported('zlib stream too short')
    cmf, flg = stream[0], stream[1]
    if cmf & 15 != 8 or cmf >> 4 > 7 or (cmf * 256 + flg) % 31 or flg & 0x20:
        raise Unsupported('zlib header: not deflate, window above 32 KiB, bad check or preset dictionary')
    return dict(width=width, height=height, color_type=color, palette=palette if color == 3 else None, idat=stream,
                before=before, after=after, trns=trns)


def _chunk(ctype, body):
    return struct.pack('>I', len(body)) + ctype + body + struct.pack('>I', zlib.crc32(body, zlib.crc32(ctype)))


def orientation(header):
    """The EXIF orientation exif_transpose would apply to the file (1 when there is none, or an invalid one), read by Pillow from
    the stand-in: the file's ancillary chunks in their places around a 1x1 grey image.  Raises Unsupported when Pillow cannot
    read those chunks (so that the file itself goes to Pillow, and the caller sees what Pillow does with it)."""
    import PIL.Image
    stand_in = SIGNATURE + _chunk(b'IHDR', struct.pack('>IIBBBBB', 1, 1, 8, 0, 0, 0, 0))
    stand_in += b''.join(_chunk(t, b) for t, b in header['before'])
    stand_in += _chunk(b'IDAT', zlib.compress(b'\0\0'))
    stand_in += b''.join(_chunk(t, b) for t, b in header['after']) + _chunk(b'IEND', b'')
    try:
        with PIL.Image.open(io.BytesIO(stand_in)) as img:
            o = img.getexif().get(0x0112, 1)
    except Exception as e:                                      # noqa: BLE001 -- whatever Pillow raises, Pillow decides
        raise Unsupported(f'ancillary chunks Pillow does not read: {e}') from e
    return int(o) if o in (2, 3, 4, 5, 6, 7, 8) else 1


def descriptor(header, orient=1):
    """dust3r_b200._lib.PngDesc of a parsed header."""
    from .. import _lib
    d = _lib.PngDesc()
    d.width, d.height = header['width'], header['height']
    d.color_type = header['color_type']
    d.orientation = orient
    d.idat_bytes = len(header['idat'])
    pal = header['palette']
    if pal is not None:
        d.palette_len = len(pal)
        flat = np.zeros((256, 3), dtype=np.uint8)
        flat[:len(pal)] = pal
        ctypes.memmove(d.palette, flat.tobytes(), flat.nbytes)
    return d


def stage(data):
    """(descriptor, oriented (width, height), payload) of a file the device decoder takes; the payload is the concatenated
    IDAT data.  Raises Unsupported for the others."""
    head = parse(data)
    orient = orientation(head)
    return descriptor(head, orient), oriented_size(head, orient), head['idat']
