"""GPU PNG decoder (csrc/png_core.h + csrc/png_ops.cu), CPU side: the kernels' per-thread bodies and launch sequence are compiled
for the HOST (tests/native/png_host.cpp, g++) and run over every thread index of every launch on a corpus made here by Pillow
and, for what Pillow cannot emit (forced row filters, zlib strategies and memory levels, 1-byte IDAT chunks, 8-bit palettes
with few entries), by numpy + zlib.  The result must equal np.asarray(exif_transpose(Image.open(f)).convert('RGB')) byte for
byte.  Also: the block chain the decoder follows is the one a sequential inflater walks, corrupt streams set the status word
without reading out of bounds (AddressSanitizer), and files outside the supported set are routed to Pillow by their header.
The `-m gpu` twin is tests/test_png_gpu.py, on the same corpus."""
import ctypes
import io
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

import native_harness

SHORT, ADLER, FAR, FILTER, PALETTE = 4, 8, 2, 16, 32     # D3R_PNG_*


def pixels(h, w, seed, kind='smooth', channels=3):
    rng = np.random.default_rng(seed)
    if kind == 'noise':
        return rng.integers(0, 256, (h, w, channels), dtype=np.uint8)
    if kind == 'flat':
        return np.broadcast_to(rng.integers(0, 256, channels, dtype=np.uint8), (h, w, channels)).copy()
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(x / (37 + 9 * c) + y / (51 + 5 * c) + seed) for c in range(channels)], axis=-1)
    if kind == 'photo':
        img += rng.normal(0, 6, img.shape)
        img[(x // 37 + y // 29) % 3 == 0] *= 0.7
    return np.clip(img, 0, 255).astype(np.uint8)


def pil_png(arr, mode, **kw):
    import PIL.Image
    img = PIL.Image.fromarray(arr[..., 0] if mode in ('L', 'P') else arr, 'L' if mode == 'P' else mode)
    if mode == 'P':
        img = img.convert('P')
    buf = io.BytesIO()
    img.save(buf, 'PNG', **kw)
    return buf.getvalue()


def _chunk(ctype, body):
    return struct.pack('>I', len(body)) + ctype + body + struct.pack('>I', zlib.crc32(body, zlib.crc32(ctype)))


def _filter_rows(arr, bpp, filters):
    """PNG filtering of (h, w * bpp) uint8 rows with the per-row filter types `filters`."""
    h, n = arr.shape
    a = arr.astype(np.int32)
    out = np.zeros((h, n + 1), dtype=np.uint8)
    for y in range(h):
        f = int(filters[y])
        cur = a[y]
        up = a[y - 1] if y else np.zeros(n, np.int32)
        left = np.concatenate([np.zeros(bpp, np.int32), cur[:-bpp]])
        upleft = np.concatenate([np.zeros(bpp, np.int32), up[:-bpp]])
        if f == 0:
            pred = 0
        elif f == 1:
            pred = left
        elif f == 2:
            pred = up
        elif f == 3:
            pred = (left + up) >> 1
        else:
            p = left + up - upleft
            pa, pb, pc = np.abs(p - left), np.abs(p - up), np.abs(p - upleft)
            pred = np.where((pa <= pb) & (pa <= pc), left, np.where(pb <= pc, up, upleft))
        out[y, 0] = f
        out[y, 1:] = (cur - pred) & 255
    return out.tobytes()


def raw_png(arr, color, filters='mixed', level=6, strategy=zlib.Z_DEFAULT_STRATEGY, mem_level=8, split=None, palette=None,
            trns=None, before=(), after=(), stream=None):
    """A PNG written here: arr (h, w, channels) uint8 samples (palette indices for colour type 3), every row filtered with
    `filters` ('mixed' = row % 5, or one type for all rows), deflated by zlib with the given level / strategy / memLevel, the
    stream cut into IDAT chunks of `split` bytes; `stream` replaces the zlib stream."""
    h, w = arr.shape[:2]
    bpp = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[color]
    ftypes = np.arange(h) % 5 if filters == 'mixed' else np.full(h, filters)
    raw = _filter_rows(arr.reshape(h, w * bpp), bpp, ftypes)
    if stream is None:
        c = zlib.compressobj(level, zlib.DEFLATED, 15, mem_level, strategy)
        stream = c.compress(raw) + c.flush()
    out = b'\x89PNG\r\n\x1a\n' + _chunk(b'IHDR', struct.pack('>IIBBBBB', w, h, 8, color, 0, 0, 0))
    if palette is not None:
        out += _chunk(b'PLTE', np.asarray(palette, np.uint8).tobytes())
    if trns is not None:
        out += _chunk(b'tRNS', trns)
    out += b''.join(_chunk(t, b) for t, b in before)
    split = split or max(1, len(stream))
    out += b''.join(_chunk(b'IDAT', stream[i:i + split]) for i in range(0, len(stream), split))
    out += b''.join(_chunk(t, b) for t, b in after)
    return out + _chunk(b'IEND', b'')


def exif_bytes(orientation):
    import PIL.Image
    e = PIL.Image.Exif()
    e[0x0112] = orientation
    return e.tobytes()


def png_corpus(large=True):
    """name -> PNG bytes, every one inside the device decoder's set."""
    c = {}
    rgb = pixels(37, 53, 1, 'photo')
    for mode in ('L', 'RGB', 'P', 'LA', 'RGBA'):
        arr = pixels(37, 53, 2, 'photo', {'L': 1, 'RGB': 3, 'P': 1, 'LA': 2, 'RGBA': 4}[mode])
        c[f'pil_{mode}_53x37'] = pil_png(arr if mode != 'P' else pixels(37, 53, 2, 'photo', 3), mode)
    for level in range(10):
        c[f'pil_level{level}_RGB_53x37'] = pil_png(rgb, 'RGB', compress_level=level)
    c['pil_optimize_RGB_53x37'] = pil_png(rgb, 'RGB', optimize=True)
    for (w, h) in ((1, 1), (2, 3), (7, 9), (33, 17), (255, 1), (1, 300)):
        c[f'size_{w}x{h}'] = pil_png(pixels(h, w, w + h, 'photo'), 'RGB')
    for kind in ('flat', 'smooth', 'noise'):
        c[f'{kind}_RGB_160x120'] = pil_png(pixels(120, 160, 3, kind), 'RGB')
        c[f'{kind}_L_160x120'] = pil_png(pixels(120, 160, 4, kind, 1), 'L')
    for f in range(5):
        c[f'filter{f}_RGB_61x23'] = raw_png(pixels(23, 61, 5, 'photo'), 2, filters=f)
        c[f'filter{f}_RGBA_61x23'] = raw_png(pixels(23, 61, 6, 'photo', 4), 6, filters=f)
        c[f'filter{f}_LA_61x23'] = raw_png(pixels(23, 61, 7, 'photo', 2), 4, filters=f)
    c['mixed_L_61x23'] = raw_png(pixels(23, 61, 8, 'photo', 1), 0)
    for name, strategy in (('fixed', zlib.Z_FIXED), ('huffman', zlib.Z_HUFFMAN_ONLY), ('rle', zlib.Z_RLE),
                           ('filtered', zlib.Z_FILTERED)):
        c[f'zlib_{name}_RGB_200x150'] = raw_png(pixels(150, 200, 9, 'photo'), 2, strategy=strategy)
    for mem in (1, 9):
        c[f'zlib_mem{mem}_RGB_200x150'] = raw_png(pixels(150, 200, 10, 'photo'), 2, mem_level=mem)
    c['idat_1byte_RGB_40x30'] = raw_png(pixels(30, 40, 11, 'photo'), 2, split=1)
    c['idat_100byte_RGB_200x150'] = raw_png(pixels(150, 200, 12, 'photo'), 2, split=100)
    idx = pixels(40, 50, 13, 'noise', 1) % 5
    pal = np.random.default_rng(14).integers(0, 256, (5, 3), dtype=np.uint8)
    c['palette5_50x40'] = raw_png(idx, 3, palette=pal)
    c['palette5_trns_50x40'] = raw_png(idx, 3, palette=pal, trns=b'\x00\x80\xff')
    c['palette256_50x40'] = raw_png(pixels(40, 50, 15, 'noise', 1), 3,
                                    palette=np.random.default_rng(16).integers(0, 256, (256, 3), dtype=np.uint8))
    c['grey_trns_50x40'] = raw_png(pixels(40, 50, 17, 'photo', 1), 0, trns=b'\x00\x10')
    c['rgb_trns_50x40'] = raw_png(pixels(40, 50, 18, 'photo'), 2, trns=b'\x00\x10\x00\x20\x00\x30')
    for o in range(1, 9):
        c[f'exif{o}_RGB_45x31'] = raw_png(pixels(31, 45, 20 + o, 'photo'), 2, before=[(b'eXIf', exif_bytes(o))])
    c['exif6_after_idat_RGB_45x31'] = raw_png(pixels(31, 45, 30, 'photo'), 2, after=[(b'eXIf', exif_bytes(6))])
    hexed = exif_bytes(8).hex()
    raw_profile = f'\nexif\n{len(exif_bytes(8)):8d}\n' + '\n'.join(hexed[i:i + 72] for i in range(0, len(hexed), 72)) + '\n'
    c['rawprofile8_RGB_45x31'] = raw_png(pixels(31, 45, 31, 'photo'), 2,
                                        before=[(b'tEXt', b'Raw profile type exif\0' + raw_profile.encode())])
    c['xmp6_RGB_45x31'] = raw_png(pixels(31, 45, 32, 'photo'), 2, before=[(b'iTXt', b'XML:com.adobe.xmp\0\0\0\0\0'
                                                                             b'<x:xmpmeta tiff:Orientation="6"/>')])
    if large:
        c['photo_RGB_1023x769'] = pil_png(pixels(769, 1023, 40, 'photo'), 'RGB')
        c['smooth_RGB_4032x3024'] = pil_png(pixels(3024, 4032, 41, 'smooth'), 'RGB', compress_level=1)
    return c


def pillow_rgb(data):
    import PIL.Image
    from PIL.ImageOps import exif_transpose
    return np.asarray(exif_transpose(PIL.Image.open(io.BytesIO(data))).convert('RGB'))


@pytest.fixture(scope='module')
def host_png():
    lib = ctypes.CDLL(native_harness.build('png_host'))
    lib.png_host_workspace_bytes.restype = ctypes.c_longlong
    lib.png_host_workspace_bytes.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    lib.png_host_decode.restype = ctypes.c_int
    lib.png_host_decode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p,
                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def parse_desc(data):
    from dust3r_b200.utils import png
    head = png.parse(data)
    o = png.orientation(head)
    return head, png.descriptor(head, o), png.oriented_size(head, o)


def host_decode(lib, stream, desc, size):
    """(RGB array, status, chain block starts, blocks taken from speculative records) from the host-compiled decoder."""
    desc.idat_bytes = len(stream)
    buf = np.frombuffer(stream, dtype=np.uint8).copy()
    ws = np.empty(lib.png_host_workspace_bytes(ctypes.byref(desc), len(stream)), dtype=np.uint8)
    assert ws.size > 0
    w, h = size
    out = np.zeros((h, w, 3), dtype=np.uint8)
    blocks = np.zeros(1 << 16, dtype=np.int64)
    status, nb, spec = ctypes.c_int32(0), ctypes.c_longlong(0), ctypes.c_longlong(0)
    assert lib.png_host_decode(ctypes.byref(desc), buf.ctypes.data, len(stream), out.ctypes.data, ctypes.byref(status),
                               ws.ctypes.data, blocks.ctypes.data, blocks.size, ctypes.byref(nb), ctypes.byref(spec)) == 0
    return out, status.value, blocks[:min(nb.value, blocks.size)].tolist(), spec.value


@pytest.fixture(scope='module')
def corpus():
    return png_corpus()


def test_corpus_is_what_it_claims(corpus):
    import PIL.Image
    modes = set()
    for name, data in corpus.items():
        img = PIL.Image.open(io.BytesIO(data))
        assert img.format == 'PNG' and not img.info.get('interlace'), name
        modes.add(img.mode)
    assert modes == {'L', 'RGB', 'P', 'LA', 'RGBA'}
    orients = {name: pillow_rgb(data).shape[:2] for name, data in corpus.items() if name.startswith(('exif', 'raw', 'xmp'))}
    assert orients['exif6_RGB_45x31'] == (45, 31) and orients['exif3_RGB_45x31'] == (31, 45)
    assert orients['rawprofile8_RGB_45x31'] == (45, 31) and orients['exif6_after_idat_RGB_45x31'] == (45, 31)
    assert orients['xmp6_RGB_45x31'] == (45, 31)


def test_decode_equals_pillow(host_png, corpus):
    """Every file of the corpus, byte for byte, with status 0."""
    for name, data in corpus.items():
        head, desc, size = parse_desc(data)
        got, status, _, _ = host_decode(host_png, head['idat'], desc, size)
        want = pillow_rgb(data)
        assert status == 0, (name, status)
        assert got.shape == want.shape, name
        if not np.array_equal(got, want):
            bad = np.argwhere(got != want)
            pytest.fail(f'{name}: {len(bad)} bytes differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}')


def deflate_block_starts(stream):
    """Bit offsets of the block headers of a zlib stream, found by a plain sequential RFC 1951 decoder written here (bit by
    bit, canonical codes in a dict), independent of the decoder under test."""
    pos = 16

    def bits(n):
        nonlocal pos
        v = 0
        for i in range(n):
            v |= ((stream[(pos + i) >> 3] >> ((pos + i) & 7)) & 1) << i
        pos += n
        return v

    def table(lengths):
        count = [0] * 16
        for l in lengths:
            count[l] += 1
        count[0] = 0
        code, first = 0, [0] * 16
        for l in range(1, 16):
            code = (code + count[l - 1]) << 1
            first[l] = code
        t = {}
        for sym, l in enumerate(lengths):
            if l:
                t[(l, first[l])] = sym
                first[l] += 1
        return t

    def decode(t):
        code = 0
        for l in range(1, 16):
            code = (code << 1) | bits(1)
            if (l, code) in t:
                return t[(l, code)]
        raise ValueError('no code')

    lbase = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
    lextra = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    dextra = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
    starts = []
    while True:
        starts.append(pos)
        final, btype = bits(1), bits(2)
        if btype == 0:
            pos = (pos + 7) // 8 * 8
            n = bits(16)
            bits(16)
            pos += 8 * n
        else:
            if btype == 1:
                lit = table([8] * 144 + [9] * 112 + [7] * 24 + [8] * 8)
                dist = table([5] * 32)
            else:
                nlit, ndist, ncode = bits(5) + 257, bits(5) + 1, bits(4) + 4
                cl = [0] * 19
                for i in range(ncode):
                    cl[[16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15][i]] = bits(3)
                ct, lens = table(cl), []
                while len(lens) < nlit + ndist:
                    sym = decode(ct)
                    if sym < 16:
                        lens.append(sym)
                    elif sym == 16:
                        lens += [lens[-1]] * (3 + bits(2))
                    else:
                        lens += [0] * (3 + bits(3) if sym == 17 else 11 + bits(7))
                lit, dist = table(lens[:nlit]), table(lens[nlit:])
            while True:
                sym = decode(lit)
                if sym == 256:
                    break
                if sym > 256:
                    bits(lextra[sym - 257])
                    bits(dextra[decode(dist)])
        if final:
            return starts


def test_chain_equals_sequential_blocks(host_png, corpus):
    """The blocks the chain accepts are the block boundaries of an independent sequential inflater; dynamic-Huffman streams
    take their blocks from the speculative records, a Z_FIXED stream is finished sequentially (no candidate is a fixed block)."""
    spec_total = checked = 0
    for name, data in corpus.items():
        head, desc, size = parse_desc(data)
        stream = head['idat']
        _, status, chain, spec = host_decode(host_png, stream, desc, size)
        assert status == 0, name
        if len(stream) <= 150000:
            assert chain == deflate_block_starts(stream), name
            checked += 1
        if name == 'zlib_fixed_RGB_200x150':
            assert spec == 0 and len(chain) > 1, (name, len(chain))
        spec_total += spec
    many = corpus['photo_RGB_1023x769']
    head, desc, size = parse_desc(many)
    _, _, chain, spec = host_decode(host_png, head['idat'], desc, size)
    assert len(chain) > 10 and spec == len(chain)
    assert spec_total > 50 and checked > 60


def with_stream(head, stream):
    """The parsed file rebuilt around another zlib stream (valid CRCs), for Pillow to decode."""
    ch = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}[head['color_type']]
    return raw_png(np.zeros((head['height'], head['width'], ch), np.uint8), head['color_type'], stream=stream,
                   palette=head['palette'], trns=head['trns'], before=head['before'], after=head['after'])


def zlib_wrap(raw_deflate, payload):
    """A zlib stream (no preset dictionary) around a raw DEFLATE stream, with the Adler-32 of `payload`."""
    return b'\x78\x9c' + raw_deflate + struct.pack('>I', zlib.adler32(payload))


def _filtered(arr, bpp):
    h, w = arr.shape[:2]
    return _filter_rows(arr.reshape(h, w * bpp), bpp, np.arange(h) % 5)


def corrupt_streams(stream, rng):
    """(stream, must be reported) pairs: truncations, bit flips, a bad Adler-32, trailing data."""
    out = [(stream[:6], True), (stream[:len(stream) // 2], True), (stream[:-1], True), (stream[:-5], True)]
    bad_adler = bytearray(stream)
    bad_adler[-1] ^= 1
    out.append((bytes(bad_adler), True))
    out.append((stream + b'\0', True))
    for _ in range(12):
        b = bytearray(stream)
        for _ in range(int(rng.integers(1, 4))):
            i = int(rng.integers(2, len(stream) - 4))
            b[i] ^= 1 << int(rng.integers(0, 8))
        out.append((bytes(b), False))
    return out


def crafted_streams():
    """name -> (PNG bytes, status bit the kernels must report): a distance before the first byte (a raw DEFLATE stream made
    against a preset dictionary, wrapped without FDICT), a filter type 5, a palette index past the palette, a stream that
    inflates to too few / too many bytes."""
    arr = pixels(20, 30, 50, 'photo')
    raw = _filtered(arr, 3)
    c = zlib.compressobj(9, zlib.DEFLATED, -15, 8, zlib.Z_DEFAULT_STRATEGY, zdict=raw[:2000])
    far = raw_png(arr, 2, stream=zlib_wrap(c.compress(raw) + c.flush(), raw))
    bad_filter = bytearray(raw)
    bad_filter[(1 + 90) * 7] = 5
    filt = raw_png(arr, 2, stream=zlib.compress(bytes(bad_filter)))
    idx = pixels(20, 30, 51, 'noise', 1) % 7
    pal = raw_png(idx, 3, palette=np.zeros((5, 3), np.uint8))
    short = raw_png(arr, 2, stream=zlib.compress(raw[:-10]))
    long = raw_png(arr, 2, stream=zlib.compress(raw + b'\0' * 10))
    return {'far': (far, FAR), 'filter5': (filt, FILTER), 'palette_index': (pal, PALETTE), 'short': (short, SHORT),
            'long': (long, SHORT)}


def test_corrupt_streams_set_the_status_word(host_png, corpus):
    """Truncations, a bad Adler-32 and trailing data are always reported; a bit flip is reported or decodes to exactly what
    Pillow decodes; the crafted streams report their bit."""
    rng = np.random.default_rng(0)
    reported = 0
    for name in ('pil_RGB_53x37', 'zlib_fixed_RGB_200x150', 'pil_level0_RGB_53x37', 'palette5_50x40', 'noise_L_160x120'):
        head, desc, size = parse_desc(corpus[name])
        for i, (stream, must) in enumerate(corrupt_streams(head['idat'], rng)):
            got, status, _, _ = host_decode(host_png, stream, desc, size)
            if must:
                assert status != 0, (name, i)
            if status:
                reported += 1
                continue
            try:
                want = pillow_rgb(with_stream(head, stream))
            except (OSError, SyntaxError, ValueError, zlib.error):
                want = None
            assert want is not None and np.array_equal(got, want), (name, i)
    assert reported > 40
    for name, (data, bit) in crafted_streams().items():
        head, desc, size = parse_desc(data)
        _, status, _, _ = host_decode(host_png, head['idat'], desc, size)
        assert status & bit, (name, status)


def test_corrupt_streams_stay_in_bounds_under_asan(tmp_path, corpus):
    """The same corrupt and crafted streams through the stand-alone harness built with -fsanitize=address: every buffer has
    its exact size, so any read past the stream aborts the run."""
    exe = native_harness.build('png_host', '-O1', '-g', '-fsanitize=address,undefined', '-fno-sanitize-recover=all',
                                '-DPNG_HOST_MAIN', shared=False)
    rng = np.random.default_rng(1)
    args = []
    cases = [(n, corpus[n]) for n in ('pil_RGB_53x37', 'zlib_fixed_RGB_200x150', 'pil_level0_RGB_53x37', 'size_1x1',
                                      'palette5_50x40')]
    for name, data in cases + [(n, d) for n, (d, _) in crafted_streams().items()]:
        head, desc, _ = parse_desc(data)
        dpath = tmp_path / f'{name}.desc'
        dpath.write_bytes(bytes(desc))
        for i, (stream, _) in enumerate([(head['idat'], False)] + corrupt_streams(head['idat'], rng)):
            fpath = tmp_path / f'{name}_{i}.z'
            fpath.write_bytes(stream)
            args += [str(dpath), str(fpath)]
    r = subprocess.run([exe] + args, capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0, r.stderr[-3000:]
    status = [int(v) for v in r.stdout.split()]
    assert len(status) == len(args) // 2
    assert status[0] == 0 and sum(s != 0 for s in status) > 60


def excluded_files():
    """name -> (PNG bytes, reason pattern): every kind of file the header sends to Pillow."""
    import PIL.Image
    arr = pixels(20, 30, 60, 'photo')
    c = {}
    buf = io.BytesIO()
    PIL.Image.fromarray(arr).save(buf, 'PNG')
    good = buf.getvalue()
    c['interlaced'] = (raw_png(arr, 2).replace(_chunk(b'IHDR', struct.pack('>IIBBBBB', 30, 20, 8, 2, 0, 0, 0)),
                                               _chunk(b'IHDR', struct.pack('>IIBBBBB', 30, 20, 8, 2, 0, 0, 1))), 'interlaced')
    for mode, why in (('1', 'bit depth 1'), ('I;16', 'bit depth 16')):
        buf = io.BytesIO()
        PIL.Image.fromarray(arr[..., 0]).convert(mode).save(buf, 'PNG')
        c[f'mode_{mode}'] = (buf.getvalue(), why)
    buf = io.BytesIO()
    PIL.Image.fromarray(arr).quantize(4).save(buf, 'PNG')
    c['palette_2bit'] = (buf.getvalue(), 'bit depth 2')
    buf = io.BytesIO()
    PIL.Image.fromarray(arr).quantize(16).save(buf, 'PNG')
    c['palette_4bit'] = (buf.getvalue(), 'bit depth 4')
    buf = io.BytesIO()
    frames = [PIL.Image.fromarray(pixels(20, 30, s, 'photo')) for s in (1, 2)]
    frames[0].save(buf, 'PNG', save_all=True, append_images=frames[1:])
    c['apng'] = (buf.getvalue(), 'acTL')
    bad = bytearray(good)
    bad[40] ^= 1
    c['crc'] = (bytes(bad), 'CRC')
    c['no_iend'] = (good[:-12], 'IEND')
    arr8 = pixels(8, 8, 61, 'photo')
    raw = _filtered(arr8, 3)
    c['fdict'] = (raw_png(arr8, 2, stream=b'\x78\xbb' + struct.pack('>I', 1) + zlib.compress(raw)[2:]), 'dictionary')
    c['window64k'] = (raw_png(arr8, 2, stream=bytes([0x88, (31 - (0x88 * 256) % 31) % 31]) + zlib.compress(raw)[2:]),
                      'window')
    c['unknown_chunk'] = (raw_png(arr8, 2, before=[(b'prVt', b'x')]), 'prVt')
    c['split_idat'] = (raw_png(arr8, 2, split=10), None)
    split = raw_png(arr8, 2, split=10)
    second = split.index(b'IDAT', split.index(b'IDAT') + 4) - 4
    c['idat_not_consecutive'] = (split[:second] + _chunk(b'tEXt', b'a\0b') + split[second:], 'not consecutive')
    return c


def test_excluded_files_are_routed_by_their_header():
    import PIL.Image
    from dust3r_b200.utils import png
    for name, (data, why) in excluded_files().items():
        if why is None:
            png.parse(data)
            continue
        with pytest.raises(png.Unsupported, match=why):
            png.parse(data)
    head = png.parse(png_corpus(large=False)['size_7x9'])
    old = PIL.Image.MAX_IMAGE_PIXELS
    try:
        PIL.Image.MAX_IMAGE_PIXELS = 62
        with pytest.raises(png.Unsupported, match='MAX_IMAGE_PIXELS'):
            png.parse(png_corpus(large=False)['size_7x9'])
    finally:
        PIL.Image.MAX_IMAGE_PIXELS = old
    assert head['width'] == 7


def test_descriptor_mirror_matches_the_library(corpus):
    """_lib.PngDesc has the size of d3r_png_desc, and the library sizes the workspace of a parsed header as the harness does."""
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    assert ctypes.sizeof(_lib.PngDesc) == lib.d3r_sizeof_png_desc()
    head, desc, _ = parse_desc(corpus['palette5_50x40'])
    assert lib.d3r_png_decode_workspace_bytes(ctypes.byref(desc), len(head['idat'])) > 0
    assert lib.d3r_png_decode_workspace_bytes(ctypes.byref(desc), len(head['idat']) + 1) == 0
    desc.orientation = 9
    assert lib.d3r_png_decode_workspace_bytes(ctypes.byref(desc), len(head['idat'])) == 0


def test_load_images_routes_pngs_by_size(monkeypatch):
    """load_images sends a PNG to the GPU decoder from PNG_DEVICE_MIN_PIXELS pixels on, by its IHDR; smaller ones and files
    outside the set go to Pillow."""
    from dust3r_b200.utils import image
    small = png_corpus(large=False)['pil_RGB_53x37']
    assert image._device_stage(small) is None
    monkeypatch.setattr(image, 'PNG_DEVICE_MIN_PIXELS', 53 * 37)
    launch, staged = image._device_stage(small)
    assert launch is image._png_launch and staged[1] == (53, 37)
    assert image._device_stage(excluded_files()['palette_4bit'][0]) is None
    monkeypatch.setattr(image, 'PNG_DEVICE_MIN_PIXELS', 53 * 37 + 1)
    assert image._device_stage(small) is None
