"""CPU: the numpy restatement of the PNG encoder (tests/png_oracle.py, whose bytes the sm_90a encoder must write) produces files
that PIL and a zlib chunk walk decode to exactly the input pixels, over sizes that put stripe boundaries and the stored-block
fallback at their edges; its checksums equal zlib's; and on rendered frames its files are no larger than PIL's at
compress_level=1."""
import io
import struct
import zlib

import numpy as np
import pytest
from PIL import Image

from tests import png_oracle as O

SIZES = [(1, 1), (1, 37), (29, 1), (7, 5), (33, 65), (2 * O.stripe_rows(21), 21), (O.stripe_rows(64) + 1, 64),
         (3 * O.stripe_rows(512), 512), (1024, 2048)]
CONTENTS = ['constant', 'gradient', 'render', 'noise']


def golden_renders():
    """The three golden 128x128 renders of the tiny and full-width generators as uint8 HWC, as the scripts convert them."""
    out = []
    for name in ('tiny512_b2', 'full512_b1'):
        for im in np.load(f'tests/golden/{name}.npz')['image_s4']:
            out.append(np.clip(np.round(im.transpose(1, 2, 0) * 127.5 + 128), 0, 255).astype(np.uint8))
    return out


def make_image(content, H, W, seed=0):
    rng = np.random.default_rng(seed)
    if content == 'constant':
        return np.full((H, W, 3), (200, 17, 90), np.uint8)
    if content == 'gradient':
        y, x = np.mgrid[:H, :W]
        return np.stack([(x * 7 + y) % 256, (y * 3) % 256, (x + y * 5) % 256], -1).astype(np.uint8)
    if content == 'render':
        g = golden_renders()[seed % 3]
        reps = (-(-H // 128), -(-W // 128), 1)
        img = np.tile(g, reps)[:H, :W].astype(np.int16) + rng.integers(-2, 3, (H, W, 3))
        return np.clip(img, 0, 255).astype(np.uint8)
    return rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def case_image(content, H, W):
    return make_image(content, H, W, seed=H * 7919 + W)


def walk_chunks(data):
    """Check the signature and every chunk's CRC; -> [(type, payload)]."""
    assert data[:8] == O.SIGNATURE
    out, p = [], 8
    while p < len(data):
        n, = struct.unpack('>I', data[p:p + 4])
        kind, payload = data[p + 4:p + 8], data[p + 8:p + 8 + n]
        crc, = struct.unpack('>I', data[p + 8 + n:p + 12 + n])
        assert crc == zlib.crc32(kind + payload), kind
        out.append((kind, payload))
        p += 12 + n
    assert p == len(data)
    return out


def assert_decodes_to(data, img):
    """PIL, and zlib plus an unfiltering of the rows, both give back the pixels."""
    H, W, _ = img.shape
    np.testing.assert_array_equal(np.asarray(Image.open(io.BytesIO(data)).convert('RGB')), img)
    chunks = walk_chunks(data)
    assert [k for k, _ in chunks] == [b'IHDR', b'IDAT', b'IEND']
    assert chunks[0][1] == struct.pack('>IIBBBBB', W, H, 8, 2, 0, 0, 0)
    raw = zlib.decompress(chunks[1][1])
    ftype, rows = O.filter_rows(img)
    assert raw == rows.tobytes()


@pytest.mark.parametrize('content', CONTENTS)
@pytest.mark.parametrize('H,W', SIZES, ids=[f'{h}x{w}' for h, w in SIZES])
def test_oracle_decodes_to_input(content, H, W):
    img = case_image(content, H, W)
    info = {}
    data = O.encode(img, info)
    assert_decodes_to(data, img)
    assert len(data) <= O.capacity(H, W)
    assert len(info['stored']) == -(-H // O.stripe_rows(W))


@pytest.mark.parametrize('H,W', [(64, 64), (O.stripe_rows(300) * 2 + 3, 300), (1024, 2048)])
def test_noise_takes_the_stored_fallback_within_the_bound(H, W):
    img = make_image('noise', H, W, seed=1)
    info = {}
    data = O.encode(img, info)
    assert all(info['stored'])
    assert len(data) == O.capacity(H, W)                 # every stripe stored: exactly the bound
    assert_decodes_to(data, img)


def test_unfiltered_rows_round_trip():
    """The filtered rows the oracle compresses invert to the image (the filter decision is free, the filters are PNG's)."""
    img = make_image('render', 70, 90)
    ftype, rows = O.filter_rows(img)
    H, W, _ = img.shape
    out = np.zeros((H, 3 * W), np.int64)
    for y in range(H):
        f, r = rows[y, 0], rows[y, 1:].astype(np.int64)
        assert f == ftype[y]
        for x in range(3 * W):
            a = out[y, x - 3] if x >= 3 else 0
            b = out[y - 1, x] if y else 0
            c = out[y - 1, x - 3] if y and x >= 3 else 0
            p = a + b - c
            pr = a if abs(p - a) <= abs(p - b) and abs(p - a) <= abs(p - c) else (b if abs(p - b) <= abs(p - c) else c)
            out[y, x] = (r[x] + [0, a, b, (a + b) // 2, pr][f]) & 0xff
    np.testing.assert_array_equal(out.reshape(H, W, 3), img)


def test_filter_choice_is_least_absolute_sum_with_ties_to_lower():
    img = np.zeros((3, 4, 3), np.uint8)              # all filters give zeros: filter 0
    assert list(O.filter_rows(img)[0]) == [0, 0, 0]
    img = np.tile(np.arange(4, dtype=np.uint8)[None, :, None] * 10, (3, 1, 3))       # horizontal ramp: Sub wins on row 0
    assert O.filter_rows(img)[0][0] == 1 and O.filter_rows(img)[0][1] == 2           # rows below: Up (2) beats Paeth (4)


@pytest.mark.parametrize('n', [0, 1, 5, 4095, 4096, 4097, 3 * 4096 + 17, 100000])
def test_checksums_equal_zlib(n):
    data = np.random.default_rng(n).integers(0, 256, n, dtype=np.uint8).tobytes()
    assert O.crc32(data) == zlib.crc32(data)
    assert O.adler32(data) == zlib.adler32(data)


def test_huffman_lengths_are_limited_and_complete():
    rng = np.random.default_rng(0)
    for limit, n in ((15, 286), (7, 19)):
        for _ in range(20):
            freq = (2.0 ** rng.uniform(0, 24, n)).astype(np.int64) * (rng.random(n) < 0.7)
            ln = O.limited_lengths(freq, limit)
            used = [l for l in ln if l]
            assert max(used) <= limit and len(used) >= 2
            assert sum(2.0 ** -l for l in used) == 1.0                       # a complete prefix code
            assert all((l > 0) == (f > 0) for l, f in zip(ln, freq)) or sum(f > 0 for f in freq) < 2
    assert O.limited_lengths([0, 0, 0, 5], 15) == [1, 0, 0, 1]                  # one used symbol: symbol 0 joins it
    # Fibonacci frequencies give a 20-deep Huffman tree: halving must bring it to 15
    fib = [1, 1]
    while len(fib) < 22:
        fib.append(fib[-1] + fib[-2])
    assert max(O.huffman_lengths(fib)) == 21 and max(O.limited_lengths(fib, 15)) <= 15


def test_rle_of_code_lengths_round_trips():
    seq = [0] * 150 + [5] * 9 + [3, 3] + [0] * 12 + [7] * 4 + [0] * 2 + [8]
    out = []
    for s, e in O.rle_lengths(seq):
        out += [out[-1]] * (e + 3) if s == 16 else [0] * (e + 3) if s == 17 else [0] * (e + 11) if s == 18 else [s]
    assert out == seq


def test_stripes_concatenate_on_byte_boundaries():
    """Every stripe but the last ends in a sync flush (00 00 ff ff on a byte boundary), and the raw deflate data of the first k
    stripes inflates to exactly their rows."""
    img = make_image('render', 3 * O.stripe_rows(256) + 5, 256)
    W, sr = 256, O.stripe_rows(256)
    _, rows = O.filter_rows(img)
    buf, bpr = rows.reshape(-1), O.row_bytes(W)
    data, ends = b'', []
    for r0 in range(0, img.shape[0], sr):
        r1 = min(img.shape[0], r0 + sr)
        part, stored = O.encode_stripe(buf, r0 * bpr, r1 * bpr, O.candidates(W), r1 == img.shape[0])
        assert not stored
        data += part
        ends.append(r1 * bpr)
    for k, end in enumerate(ends[:-1]):
        stripe_end = sum(len(O.encode_stripe(buf, r0 * bpr, min(img.shape[0], r0 + sr) * bpr, O.candidates(W), False)[0])
                         for r0 in range(0, (k + 1) * sr, sr))
        assert data[stripe_end - 4:stripe_end] == b'\x00\x00\xff\xff'
        assert zlib.decompressobj(-15).decompress(data[:stripe_end]) == buf[:end].tobytes()
    d = zlib.decompressobj(-15)
    assert d.decompress(data) == buf.tobytes() and d.eof


def test_renders_no_larger_than_pil_level_1():
    for img in golden_renders():
        buf = io.BytesIO()
        Image.fromarray(img).save(buf, format='png', compress_level=1)
        ours = len(O.encode(img))
        print(f'oracle {ours} bytes, PIL level 1 {len(buf.getvalue())} bytes')
        assert ours <= len(buf.getvalue())


def test_capacity_matches_library():
    """The library's file capacity is the oracle's bound (needs only the host entry point, no device)."""
    from next3d_b200 import png
    for H, W in SIZES + [(1, 20000), (3, 11000)]:
        assert png.check_args(W, H)[1] == O.capacity(H, W)


@pytest.mark.parametrize('name', ['n3d_png_buffer_sizes', 'n3d_png_encode'])
def test_png_entry_points_bound_with_the_header_arity(name):
    import re
    from next3d_b200 import _lib
    src = re.sub(r'/\*.*?\*/', '', open('include/next3d_b200.h').read(), flags=re.S)
    params = re.search(name + r'\s*\(([^)]*)\)', src).group(1).split(',')
    assert len(_lib._SIGNATURES[name][0]) == len(params)
