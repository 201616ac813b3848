"""GPU JPEG decoder (csrc/jpeg_core.h + csrc/jpeg_ops.cu), CPU side: the kernels' per-thread bodies and launch sequence are
compiled for the HOST (tests/native/jpeg_host.cpp, g++) and run over every thread index of every launch on a corpus that Pillow
(libjpeg-turbo) encodes here from seeded pixels; the result must equal np.asarray(exif_transpose(Image.open(f)).convert('RGB'))
byte for byte.  Also: the speculative decode lands on the sequential decoder's state at every subsequence, corrupt and truncated
streams set the status word without reading out of bounds (AddressSanitizer), and files outside the supported set are routed to
Pillow by their header.  The `-m gpu` twin is tests/test_jpeg_gpu.py, on the same corpus."""
import ctypes
import io
import os
import subprocess

import numpy as np
import pytest

import native_harness


def _pixels(h, w, seed, kind='photo'):
    rng = np.random.default_rng(seed)
    if kind == 'noise':
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([128 + 100 * np.sin(x / (7 + 3 * c) + y / (11 + 2 * c) + seed) for c in range(3)], axis=-1)
    img += rng.normal(0, 12, img.shape)
    img[(x // 37 + y // 29) % 3 == 0] *= 0.6                    # edges
    return np.clip(img, 0, 255).astype(np.uint8)


def _pil_jpeg(arr, mode='RGB', orientation=None, **kw):
    import PIL.Image
    img = PIL.Image.fromarray(arr)
    if mode != 'RGB':
        img = img.convert(mode)
    if orientation is not None:
        exif = PIL.Image.Exif()
        exif[0x0112] = orientation
        kw['exif'] = exif
    buf = io.BytesIO()
    img.save(buf, 'JPEG', **kw)
    return buf.getvalue()


def _cv2_jpeg(arr, factor, quality=90):
    import cv2
    ok, enc = cv2.imencode('.jpg', arr[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, quality, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, factor])
    assert ok
    return enc.tobytes()


def jpeg_corpus(large=True):
    """name -> JPEG bytes.  Baseline files the device decodes, 4:4:0 and 4:1:1 (which go to Pillow), noise at quality 100."""
    sub = {'444': 0, '422': 1, '420': 2}
    c = {}
    for q in (30, 75, 90, 100):
        for s in ('444', '422', '420'):
            c[f'q{q}_{s}_64x48'] = _pil_jpeg(_pixels(48, 64, q), quality=q, subsampling=sub[s])
    for s in ('444', '422', '420'):
        c[f'opt_{s}_123x77'] = _pil_jpeg(_pixels(77, 123, 5), quality=85, subsampling=sub[s], optimize=True)
        for r in (1, 7):
            c[f'rst{r}_{s}_100x75'] = _pil_jpeg(_pixels(75, 100, 6), quality=90, subsampling=sub[s], restart_marker_blocks=r)
        for (w, h) in ((1, 1), (7, 9), (17, 33), (2, 3), (3, 2), (4, 5)):
            c[f'size_{s}_{w}x{h}'] = _pil_jpeg(_pixels(h, w, w * h), quality=90, subsampling=sub[s])
    c['grey_q90_53x41'] = _pil_jpeg(_pixels(41, 53, 7), mode='L', quality=90)
    c['grey_rst3_33x17'] = _pil_jpeg(_pixels(17, 33, 8), mode='L', quality=60, restart_marker_blocks=3)
    c['noise_q100_444_96x80'] = _pil_jpeg(_pixels(80, 96, 9, 'noise'), quality=100, subsampling=0)
    c['noise_q100_420_257x130'] = _pil_jpeg(_pixels(130, 257, 10, 'noise'), quality=100, subsampling=2)
    for o in range(1, 9):
        c[f'exif{o}_420_45x31'] = _pil_jpeg(_pixels(31, 45, 20 + o), quality=90, subsampling=2, orientation=o)
    c['cv2_440_70x50'] = _cv2_jpeg(_pixels(50, 70, 11), __import__('cv2').IMWRITE_JPEG_SAMPLING_FACTOR_440)
    c['cv2_411_70x50'] = _cv2_jpeg(_pixels(50, 70, 12), __import__('cv2').IMWRITE_JPEG_SAMPLING_FACTOR_411)
    c['cv2_420_70x50'] = _cv2_jpeg(_pixels(50, 70, 13), __import__('cv2').IMWRITE_JPEG_SAMPLING_FACTOR_420)
    if large:
        c['q90_420_1023x769'] = _pil_jpeg(_pixels(769, 1023, 14), quality=90, subsampling=2)
        c['rst7_422_1023x769'] = _pil_jpeg(_pixels(769, 1023, 15), quality=95, subsampling=1, restart_marker_blocks=7)
        c['q90_420_4032x3024'] = _pil_jpeg(_pixels(3024, 4032, 16), quality=90, subsampling=2)
    return c


# files the device decoder must accept (everything else in the corpus goes to Pillow)
HOST_ONLY = {'cv2_440_70x50', 'cv2_411_70x50'}
RANGE = 16           # D3R_JPEG_RANGE
SYNC_ROUNDS = 8      # jpeg_core.h kSyncRounds; host_decode reports SYNC_ROUNDS + 1 when the sequential finish had work


def pillow_rgb(data):
    import PIL.Image
    from PIL.ImageOps import exif_transpose
    return np.asarray(exif_transpose(PIL.Image.open(io.BytesIO(data))).convert('RGB'))


@pytest.fixture(scope='module')
def host_jpeg():
    lib = ctypes.CDLL(native_harness.build('jpeg_host'))
    lib.jpeg_host_workspace_bytes.restype = ctypes.c_longlong
    lib.jpeg_host_workspace_bytes.argtypes = [ctypes.c_void_p, ctypes.c_longlong]
    lib.jpeg_host_decode.restype = ctypes.c_int
    lib.jpeg_host_decode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p,
                                     ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    lib.jpeg_host_check_sync.restype = ctypes.c_longlong
    lib.jpeg_host_check_sync.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _desc(data):
    from dust3r_b200.utils import jpeg
    head = jpeg.parse(data)
    o = jpeg.orientation(data)
    return jpeg.descriptor(head, o), jpeg.oriented_size(head, o)


def host_decode(lib, data, desc=None):
    """(RGB array, status, subsequences, sync rounds) from the host-compiled decoder."""
    size = None
    if desc is None:
        desc, size = _desc(data)
    buf = np.frombuffer(data, dtype=np.uint8).copy()
    ws = np.empty(lib.jpeg_host_workspace_bytes(ctypes.byref(desc), len(data)), dtype=np.uint8)
    assert ws.size > 0
    w, h = size if size else ((desc.height, desc.width) if desc.orientation >= 5 else (desc.width, desc.height))
    out = np.zeros((h, w, 3), dtype=np.uint8)
    status, nsub, rounds = ctypes.c_int32(0), ctypes.c_longlong(0), ctypes.c_int(0)
    assert lib.jpeg_host_decode(ctypes.byref(desc), buf.ctypes.data, len(data), out.ctypes.data, ctypes.byref(status),
                                ws.ctypes.data, ctypes.byref(nsub), ctypes.byref(rounds)) == 0
    return out, status.value, nsub.value, rounds.value


@pytest.fixture(scope='module')
def corpus():
    return jpeg_corpus()


def test_corpus_is_what_it_claims(corpus):
    import PIL.Image
    for name, data in corpus.items():
        img = PIL.Image.open(io.BytesIO(data))
        assert img.format == 'JPEG' and not img.info.get('progressive'), name
        if name.startswith('rst'):
            assert b'\xff\xdd' in data and b'\xff\xd0' in data, name
        if name.startswith('opt'):
            assert data != _pil_jpeg(_pixels(77, 123, 5), quality=85, subsampling={'444': 0, '422': 1, '420': 2}[name[4:7]])
    assert {n for n in corpus if 'exif' in n} == {f'exif{o}_420_45x31' for o in range(1, 9)}


def test_supported_set_is_chosen_from_the_header(corpus):
    from dust3r_b200.utils import jpeg
    for name, data in corpus.items():
        if name in HOST_ONLY:
            with pytest.raises(jpeg.Unsupported):
                jpeg.parse(data)
        else:
            jpeg.parse(data)
    arr = _pixels(40, 56, 3)
    for data, why in ((_pil_jpeg(arr, progressive=True), 'SOF2'), (_pil_jpeg(arr, mode='CMYK'), 'components'),
                      (_cv2_jpeg(arr, __import__('cv2').IMWRITE_JPEG_SAMPLING_FACTOR_411), 'sampling')):
        with pytest.raises(jpeg.Unsupported, match=why):
            jpeg.parse(data)


def test_decode_equals_pillow(host_jpeg, corpus):
    """Every accepted file of the corpus, byte for byte, with status 0."""
    for name, data in corpus.items():
        if name in HOST_ONLY:
            continue
        got, status, _, _ = host_decode(host_jpeg, data)
        want = pillow_rgb(data)
        assert status == 0, name
        assert got.shape == want.shape, name
        if not np.array_equal(got, want):
            bad = np.argwhere(got != want)
            pytest.fail(f'{name}: {len(bad)} bytes differ, first at {bad[0].tolist()}: {got[tuple(bad[0])]} vs {want[tuple(bad[0])]}')


def test_speculative_decode_equals_sequential(host_jpeg, corpus):
    """The synchronised start state of every subsequence is the sequential decoder's state there; the large files need
    resynchronisation (phase-1 guesses are wrong somewhere) and still converge within the sync rounds."""
    resynced_total = 0
    for name, data in corpus.items():
        if name in HOST_ONLY:
            continue
        desc, _ = _desc(data)
        buf = np.frombuffer(data, dtype=np.uint8).copy()
        ws = np.empty(host_jpeg.jpeg_host_workspace_bytes(ctypes.byref(desc), len(data)), dtype=np.uint8)
        resynced = ctypes.c_longlong(0)
        assert host_jpeg.jpeg_host_check_sync(ctypes.byref(desc), buf.ctypes.data, len(data), ws.ctypes.data,
                                              ctypes.byref(resynced)) == 0, name
        resynced_total += resynced.value
    assert resynced_total > 100
    _, status, nsub, rounds = host_decode(host_jpeg, corpus['q90_420_4032x3024'])
    assert status == 0 and nsub > 1000 and 1 <= rounds <= SYNC_ROUNDS
    # streams without end-of-block codes do not resynchronise within the rounds: the sequential finish completes them
    _, status, _, rounds = host_decode(host_jpeg, corpus['noise_q100_420_257x130'])
    assert status == 0 and rounds == SYNC_ROUNDS + 1


def _corruptions(data, rng):
    """Truncations (inside the scan, right after the header, one byte short) and bit flips in the entropy-coded data."""
    from dust3r_b200.utils import jpeg
    begin = jpeg.parse(data)['scan_begin']
    out = [data[:begin + 1], data[:begin + (len(data) - begin) // 2], data[:-1], data[:-2], data[:-3]]
    for _ in range(12):
        b = bytearray(data)
        for _ in range(int(rng.integers(1, 4))):
            i = int(rng.integers(begin, len(data) - 2))
            b[i] ^= 1 << int(rng.integers(0, 8))
        out.append(bytes(b))
    b = bytearray(data)
    b[begin + 10:begin + 12] = b'\xff\xd3'                     # a stray restart marker
    out.append(bytes(b))
    return out


def test_corrupt_streams_set_the_status_word(host_jpeg, corpus):
    """A decode either reports a non-zero status or equals what Pillow decodes (Pillow raising counts as a difference);
    truncations inside the scan are always reported."""
    rng = np.random.default_rng(0)
    reported = 0
    for name in ('q90_420_64x48', 'rst1_422_100x75', 'rst7_444_100x75', 'grey_q90_53x41', 'noise_q100_444_96x80'):
        desc, _ = _desc(corpus[name])
        for i, data in enumerate(_corruptions(corpus[name], rng)):
            got, status, _, _ = host_decode(host_jpeg, data, desc)
            if i < 2:
                assert status != 0, (name, i)
            if status:
                reported += 1
                continue
            try:
                want = pillow_rgb(data)
            except OSError:
                want = None
            assert want is not None and np.array_equal(got, want), (name, i)
    assert reported > 30


def test_corrupt_streams_stay_in_bounds_under_asan(tmp_path, corpus):
    """The same corrupt streams through the stand-alone harness built with -fsanitize=address: every buffer has its exact size,
    so any read past the compressed bytes aborts the run."""
    exe = native_harness.build('jpeg_host', '-O1', '-g', '-fsanitize=address,undefined', '-fno-sanitize-recover=all',
                                '-DJPEG_HOST_MAIN', shared=False)
    rng = np.random.default_rng(1)
    args = []
    for name in ('q90_420_64x48', 'rst1_422_100x75', 'grey_rst3_33x17', 'size_420_1x1', 'noise_q100_444_96x80'):
        desc, _ = _desc(corpus[name])
        dpath = tmp_path / f'{name}.desc'
        dpath.write_bytes(bytes(desc))
        for i, data in enumerate([corpus[name]] + _corruptions(corpus[name], rng)):
            fpath = tmp_path / f'{name}_{i}.jpg'
            fpath.write_bytes(data)
            args += [str(dpath), str(fpath)]
    r = subprocess.run([exe] + args, capture_output=True, text=True, env=dict(os.environ, ASAN_OPTIONS='detect_leaks=0'))
    assert r.returncode == 0, r.stderr[-3000:]
    status = [int(v) for v in r.stdout.split()]
    assert len(status) == len(args) // 2
    assert status[0] == 0 and sum(s != 0 for s in status) > 20


def test_descriptor_mirror_matches_the_library(corpus):
    """_lib.JpegDesc has the size of d3r_jpeg_desc, and the library sizes the workspace of a parsed header as the harness does."""
    from dust3r_b200 import _lib
    lib = _lib.get_lib()
    assert ctypes.sizeof(_lib.JpegDesc) == lib.d3r_sizeof_jpeg_desc()
    desc, _ = _desc(corpus['rst7_420_100x75'])
    assert lib.d3r_jpeg_decode_workspace_bytes(ctypes.byref(desc), len(corpus['rst7_420_100x75'])) > 0
    desc.orientation = 9
    assert lib.d3r_jpeg_decode_workspace_bytes(ctypes.byref(desc), 1000) == 0


def with_trailer(data, n, seed=0):
    """The file followed by n bytes after EOI, as MPF previews, gain maps and vendor trailers are: random bytes with markers."""
    tail = np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    tail[::997] = 0xFF
    return data + b'\xff\xd8' + tail.tobytes()


def test_bytes_after_eoi_are_not_decoded(host_jpeg, corpus):
    """A 64 KB / 1 MB trailer after EOI changes neither the pixels nor the work: the scan ends at EOI, so the subsequences past
    it are never decoded and the sync rounds needed are those of the bare file."""
    for name in ('q90_420_1023x769', 'rst7_422_1023x769', 'q90_420_64x48'):
        _, _, _, bare_rounds = host_decode(host_jpeg, corpus[name])
        for n in (65536, 1 << 20):
            data = with_trailer(corpus[name], n)
            got, status, nsub, rounds = host_decode(host_jpeg, data)
            assert status == 0 and rounds == bare_rounds, (name, n, status, rounds, bare_rounds)
            assert nsub * 256 >= n
            assert np.array_equal(got, pillow_rgb(data)), (name, n)


def crafted_grey_8x8(dc_quant, dc_coef):
    """A hand-built 8x8 grey baseline file whose single block has only a DC coefficient: the standard luminance DC table, an AC
    table with one code (EOB = '0').  Large dc_quant * dc_coef drive the IDCT output outside [-512, 511]."""
    import struct
    dc_counts = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
    dc_syms = list(range(12))
    q = [dc_quant] + [1] * 63
    seg = lambda m, body: b'\xff' + bytes([m]) + struct.pack('>H', len(body) + 2) + body
    head = b'\xff\xd8' + seg(0xDB, bytes([0]) + bytes(q)) + seg(0xC0, bytes([8, 0, 8, 0, 8, 1, 1, 0x11, 0]))
    head += seg(0xC4, bytes([0x00] + dc_counts + dc_syms)) + seg(0xC4, bytes([0x10, 1] + [0] * 15 + [0]))
    head += seg(0xDA, bytes([1, 1, 0x00, 0, 63, 0]))
    # canonical codes of the standard DC table: category -> (code, length)
    codes, code, k = {}, 0, 0
    for length, cnt in enumerate(dc_counts, 1):
        for _ in range(cnt):
            codes[dc_syms[k]] = (code, length)
            code, k = code + 1, k + 1
        code <<= 1
    cat = int(abs(dc_coef)).bit_length()
    extra = dc_coef if dc_coef >= 0 else dc_coef + (1 << cat) - 1
    c, length = codes[cat]
    bits = format(c, f'0{length}b') + (format(extra, f'0{cat}b') if cat else '') + '0'
    bits += '1' * (-len(bits) % 8)
    scan = bytes(int(bits[i:i + 8], 2) for i in range(0, len(bits), 8)).replace(b'\xff', b'\xff\x00')
    return head + scan + b'\xff\xd9'


RANGE_CASES = [(3, 2047), (2, 2047), (5, 1100), (3, -2047), (5, -1100)]


def test_idct_outputs_outside_the_simd_range_are_reported(host_jpeg):
    """Where libjpeg's C range limit (10-bit wrap) and the saturating SIMD store Pillow runs differ, the decoder reports
    D3R_JPEG_RANGE instead of returning the C result; just inside the range it decodes and equals Pillow."""
    differs = 0
    for dc_quant, dc_coef in RANGE_CASES:
        data = crafted_grey_8x8(dc_quant, dc_coef)
        want = pillow_rgb(data)
        got, status, _, _ = host_decode(host_jpeg, data)
        assert status & RANGE, (dc_quant, dc_coef, status)
        differs += not np.array_equal(got, want)
    assert differs == len(RANGE_CASES)              # the C arithmetic alone would have returned other pixels than Pillow
    for dc_quant, dc_coef in ((1, 1000), (1, -1000), (2, 500)):
        data = crafted_grey_8x8(dc_quant, dc_coef)
        got, status, _, _ = host_decode(host_jpeg, data)
        assert status == 0 and np.array_equal(got, pillow_rgb(data)), (dc_quant, dc_coef)
