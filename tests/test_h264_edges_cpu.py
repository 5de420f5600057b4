"""CPU: the H.264 encoder's coding edges.  A case table of the oracle's edge sequences (tests/h264_oracle.py EDGE_SEQUENCES) at
frame sizes the small table never reaches (2-sample crop remainders, one MB column of 66 rows, 65x33 MBs, and the level-6.2
extremes of 1055 MBs along one side), a sweep of every QP 0-51 in both streams, and 20-frame GOPs that wrap frame_num.  A census
counts what the table reaches (every QP, the LEVEL_MAX clamp, the CAVLC tables, every mb_type and coded_block_pattern, skip runs,
quarter-sample vectors, every bS with the deblocking filter on and off, the rate controller's clamps and steps) and fails on any
entry it misses; FFmpeg decodes every stream of the table to its reconstruction; and the largest slice of every case fits the
per-row slot of n3d_h264_buffer_sizes.  tests/test_gpu_h264_edges.py compares the kernels with the oracle on the same table."""
import collections
import functools

import numpy as np
import pytest

from tests import h264_oracle as O
from tests.test_h264_cpu import CASES, FPS, assert_decodes_to, write

SMALL_SIZES = [(2, 2), (18, 18), (16, 1056)]
RC_BPP = 4                     # the edge table's rate-controlled target: bits per pixel, so that the controller starts at QP 0


def cq(name, W, H, n=3, gop=60, qp=0):
    """A case of the constant-QP stream: (name, W, H, frames, gop, qp, bitrate, qp_min, qp_max)."""
    return (name, W, H, n, gop, qp, None, 0, 51)


def rc(name, W, H, n=3, gop=60, bitrate=None, qp_range=(0, 51)):
    """A case of the rate-controlled stream, by default at RC_BPP bits per pixel."""
    return (name, W, H, n, gop, None, bitrate or RC_BPP * W * H * FPS, *qp_range)


def both(name, W, H, n=3):
    """The case in both streams: at QP 0 (the controller starting there), or at QP 24 for the sequences that need P_Skip MBs
    or levels that stay zero."""
    if name in ('static', 'cbp'):
        return [cq(name, W, H, n, qp=24), rc(name, W, H, n, bitrate=10 ** 6, qp_range=(24, 24))]
    return [cq(name, W, H, n), rc(name, W, H, n)]


# Every edge sequence at the small sizes ('motion' with its fourth frame, which moves beyond the search bound); 'cbp' at 8x6 MBs,
# one per coded_block_pattern; at the large sizes the IDR frame and one P frame of the sequences that need the size: 'static'
# (skip runs along 65 and 1055 MB rows, the vector field of the zoom) and 'stripes' (the worst slices, 1055 MBs in one slice;
# 1055 rows of deblocking tickets).
EDGE_CASES = ([c for name in O.EDGE_SEQUENCES for (W, H) in SMALL_SIZES for c in both(name, W, H, 4 if name == 'motion' else 3)]
              + both('cbp', 128, 96) + both('static', 1040, 528, 2) + both('stripes', 16880, 16, 2)
              + both('static', 16880, 16, 2) + both('stripes', 16, 16880, 2))
SWEEP_CASES = [c for q in range(52) for c in (cq('mosaic', 48, 32, 3, 2, q), rc('mosaic', 48, 32, 3, 2, 10 ** 6, (q, q)))]
# frame_num wraps (20 frames, GOP 20); the controller free, starting at QP 51 with a target it cannot reach, and coding an IDR
# frame after an IDR frame (GOP 1)
RUN_CASES = [cq('translate', 48, 32, 20, 20, 18), rc('translate', 48, 32, 20, 20, 2000), rc('cut', 18, 18, 3, 1)]
TABLE = EDGE_CASES + SWEEP_CASES + RUN_CASES


def case_id(c):
    name, W, H, n, gop, qp, bitrate, lo, hi = c
    rate = f'qp{qp}' if bitrate is None else f'rc{bitrate}' + ('' if (lo, hi) == (0, 51) else f'-qp{lo}..{hi}')
    return f'{name}-{W}x{H}-{n}f-gop{gop}-{rate}'


def stream_of(case):
    return 'cq' if case[6] is None else 'rc'


def stream_args(case):
    """H264Writer's / the oracle's stream arguments of a case."""
    _, _, _, _, _, qp, bitrate, lo, hi = case
    return dict(qp=qp) if bitrate is None else dict(bitrate=bitrate, qp_range=(lo, hi))


@functools.lru_cache(maxsize=None)
def edge_run(case):
    """The oracle's stream of a case, with its census: (samples, IDR flags, recon planes per frame, QP per frame, Counter)."""
    name, W, H, n, gop, qp, bitrate, lo, hi = case
    enc = O.Encoder(W, H, qp, gop) if bitrate is None else O.RcEncoder(W, H, bitrate, (FPS, 1), gop, lo, hi)
    census = collections.Counter()
    enc.record(census)
    samples, idr, recon, qps = [], [], [], []
    for f in O.frames(name, W, H, n):
        s, i = enc.encode(f)
        samples.append(s)
        idr.append(i)
        recon.append(enc.recon)
        qps.append(enc.qp)
    return samples, idr, recon, qps, census


# ------------------------------------------------------------------------------------------------ census
def required(stream):
    """(key, what it is) of every entry the table must reach in a stream ('cq' or 'rc')."""
    out = [(('qp', f, q), f'QP {q} in an {f} frame') for f in 'IP' for q in range(52)]
    out += [(('clamp', k), f'a {k} level clamped to LEVEL_MAX') for k in ('I luma DC', 'I chroma DC', 'P chroma DC')]
    out += [(('coeff_token', t), f'coeff_token with {t}') for t in ('nC 0-1', 'nC 2-3', 'nC 4-7', 'nC >= 8', 'chroma DC')]
    out += [(('level_prefix', p), f'level_prefix {p}') for p in (14, 15)]
    out += [(('suffixLength', s), f'a level coded at suffixLength {s}') for s in range(7)]
    out += [(('TotalCoeff', t), f'a 4x4 block with TotalCoeff {t}') for t in range(1, 17)]
    out += [(('total_zeros', '4x4', t), f'total_zeros of a 4x4 block with TotalCoeff {t}') for t in range(1, 16)]
    out += [(('total_zeros', 'chroma DC', t), f'total_zeros of a chroma DC block with TotalCoeff {t}') for t in range(1, 4)]
    out += [(('run_before', z), f'run_before with {z}') for z in [f'zerosLeft {k}' for k in range(1, 7)] + ['zerosLeft > 6']]
    out += [(('I16x16', m, c, l), f'I_16x16 mb_type, {"horizontal" if m == 1 else "DC"} prediction, cbp_c {c}, cbp_l {l}')
            for m in (1, 2) for c in range(3) for l in (0, 15)]
    out += [(('P cbp', l, c), f'a P MB with cbp_l {l}, cbp_c {c}') for l in range(16) for c in range(3)]
    out += [(('skip run', k), f'a skip run at the {k}' if k != 'whole row' else 'a row of skipped MBs')
            for k in ('row start', 'mid-row', 'row end', 'whole row')]
    out += [(('frame_num wrap',), 'frame_num wrapping to 0 inside a GOP')]
    out += [(('idr_pic_id', i), f'idr_pic_id {i}') for i in (0, 1)]
    out += [(('size', s), f'a frame with {s}') for s in ('2-sample crop remainder', 'more than 32 MB rows', 'more than 256 MB rows',
                                                         '1 MB column, several rows', '2 MB columns, several rows',
                                                         'more than 1024 MB columns')]
    if stream == 'rc':
        out += [(('quarter-sample position', x, y), f'a vector at quarter-sample position ({x}, {y})') for y in range(4) for x in range(4)]
        out += [(('vector at the search bound',), 'a vector at the search bound'),
                (('vector refined past the search bound',), 'a vector refined past the search bound')]
        out += [(('bS', p, b, t), f'a {p} line at bS {b} whose sample test {"passes" if t == "filtered" else "fails"}')
                for p in ('luma', 'chroma') for b in range(5) for t in ('filtered', 'not filtered')]
        out += [(('rc', k), f'the rate controller: {k}') for k in ('step -2', 'step +2', 'clamped at qp_min', 'clamped at qp_max',
                                                                    'IDR frame after an IDR frame')]
    return out


def tally(cases):
    """{stream: Counter} over the cases' census (the largest slice's size as a maximum, not a sum)."""
    out = {'cq': collections.Counter(), 'rc': collections.Counter()}
    for c in cases:
        counts = edge_run(c)[4]
        total = out[stream_of(c)]
        big = max(total['slice bytes max'], counts['slice bytes max'])
        total.update(counts)
        total['slice bytes max'] = big
    return out


def missing(counts, stream):
    return [what for key, what in required(stream) if counts[key] == 0]


def test_census_reaches_every_entry():
    counts = tally(TABLE)
    for stream in ('cq', 'rc'):
        c = counts[stream]
        print(f'\n{stream} stream, {sum(1 for x in TABLE if stream_of(x) == stream)} cases:')
        for key, what in required(stream):
            print(f'  {c[key]:9d}  {what}')
        pairs = [k for k in c if k[0] == 'total_zeros pair' and c[k]]
        print(f'  {len(pairs):9d}  (TotalCoeff, total_zeros) pairs of the 135 + 9 the tables hold')
        print(f'  {c["emulation prevention bytes"]:9d}  emulation prevention bytes')
        for kind in ('I luma AC', 'P luma', 'I chroma AC', 'P chroma AC'):    # at most 16 * 255 * 13107 >> 15 = 1632: never clamped
            print(f'  {c["clamp", kind]:9d}  {kind} levels clamped (none can be)')
    for stream in ('cq', 'rc'):
        assert not missing(counts[stream], stream), f'the {stream} stream reaches none of: {missing(counts[stream], stream)}'
        assert counts[stream]['emulation prevention bytes'] >= 100          # the small table inserts 19 in all


def test_census_of_the_small_table_misses_the_edges():
    """The constant-QP cases of tests/test_h264_cpu.py below 512x512 reach none of the QPs but 0, 18 and 40, no clamp, none of
    the sizes and no frame_num wrap: the census tells them from the edge table."""
    cases = [cq(name, W, H, 3, gop, qp) for name, W, H, qp, gop in CASES if W < 512]
    gone = set(missing(tally(cases)['cq'], 'cq'))
    want = {what for key, what in required('cq') if key[0] in ('qp', 'clamp', 'size', 'frame_num wrap') and key[-1] not in (0, 18, 40)}
    assert want <= gone, sorted(want - gone)


@pytest.mark.parametrize('case', TABLE, ids=case_id)
def test_edge_stream_decodes_to_its_reconstruction(tmp_path, case):
    name, W, H, n, gop, qp, bitrate, lo, hi = case
    run = edge_run(case)
    assert len(run[0]) == n and [i for i, x in enumerate(run[1]) if x] == list(range(0, n, gop))
    if bitrate is not None and lo == hi:
        assert run[3] == [lo] * n
    assert_decodes_to(write(tmp_path / 'v.mp4', W, H, run, qp=qp, bitrate=bitrate), run[2], W, H, rgb=W * H <= 1056 * 16)


def slot_capacity(W, H):
    """Bytes of one row's slot (length prefix, NAL header and escaped slice) in n3d_h264_buffer_sizes' buffers."""
    from next3d_b200 import _lib
    out = [_lib.I64() for _ in range(4)]
    assert _lib.lib.n3d_h264_buffer_sizes(W, H, *[_lib.C.byref(x) for x in out]) == 0
    return out[2].value // ((H + 15) // 16)


def slices(sample):
    o, out = 0, []
    while o < len(sample):
        n = int.from_bytes(sample[o:o + 4], 'big')
        out.append(4 + n)
        o += 4 + n
    return out


def test_slices_fit_their_slots():
    """The largest slice (with its length prefix) of every case is within its row's slot, including the worst frames made here:
    noise over 0 / 255 stripes, IDR and P, at QP 0 in one slice of 1055 MBs."""
    worst = (1.0, None)
    for c in TABLE:
        _, W, H = c[:3]
        cap, mbw = slot_capacity(W, H), (W + 15) // 16
        big = max(max(slices(s)) for s in edge_run(c)[0])
        assert big == edge_run(c)[4]['slice bytes max']
        assert big <= cap, (case_id(c), big, cap)
        worst = min(worst, ((cap - big) / cap, case_id(c), big, cap, mbw))
    margin, name, big, cap, mbw = worst
    print(f'\nsmallest slot margin: {name}: largest slice {big} bytes ({big / mbw:.0f} per MB) of a {cap}-byte slot '
          f'({cap / mbw:.0f} per MB): {margin:.1%} free')
    assert np.isfinite(margin)
