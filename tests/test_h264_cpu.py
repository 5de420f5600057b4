"""CPU: the H.264 byte format of both streams, the constant-QP one and the rate-controlled one (quarter-sample motion,
deblocking, a QP per picture from the rate controller).  Streams of the numpy restatement of the encoder (tests/h264_oracle.py,
which the GPU encoder matches byte for byte in tests/test_gpu_h264.py) are written through next3d_b200.mp4 and decoded by
FFmpeg (OpenCV's CAP_FFMPEG backend): the decoder's luma equals the encoder's (deblocked) reconstruction bit for bit, its BGR
output matches the reconstruction converted with BT.601, and the MP4 boxes parse back.  Also the motion searches, the controller
against its targets, the CLI's --encoder n3d and --bitrate paths up to loading the network, and the argument refusals of
next3d_b200.video and of the library."""
import functools
import struct
import sys

import numpy as np
import pytest

from tests import h264_oracle as O

FPS = 30
SIZES = [(16, 16), (48, 32), (40, 24), (512, 512)]
CASES = [(name, W, H, qp, gop) for name in O.SEQUENCES for (W, H) in SIZES for qp in (0, 18, 40) for gop in (1, 3)
         if (W, H) != (512, 512) or gop == 3]            # 512x512: the 3-frame GOP (IDR + P frames) only, to bound the run time
MODES = (0, 18, 40, 'rc')                  # the rate-controlled stream: pinned QPs, and the controller at RC_BPP
RC_BPP = 1.0                               # bits per pixel of the 'rc' mode's target
RC_CASES = [(name, W, H, mode) for name in O.SEQUENCES + ('pan',) for (W, H) in SIZES for mode in MODES
            if (W, H) != (512, 512) or (name in ('translate', 'pan') and mode in (18, 'rc'))]      # 512x512: bounds the run time
RC_FPS, RC_GOP, RC_FRAMES = 60, 60, 240


def oracle(W, H, gop, qp=None, bitrate=None, qp_range=(0, 51), fps=FPS):
    """The oracle of the constant-QP stream at qp, or with a bitrate (bits/s) of the rate-controlled stream, its QP within
    qp_range."""
    return O.Encoder(W, H, qp, gop) if bitrate is None else O.RcEncoder(W, H, bitrate, (fps, 1), gop, *qp_range)


@functools.lru_cache(maxsize=None)
def encoded(name, W, H, qp=None, gop=3, bitrate=None, qp_range=(0, 51), fps=FPS, n=3):
    """Oracle stream of O.frames(name, W, H, n) (see oracle()): (samples, IDR flags, recon planes per frame, (mvs, skip) per
    frame, QP per frame)."""
    enc = oracle(W, H, gop, qp, bitrate, qp_range, fps)
    samples, idr, recon, motion, qps = [], [], [], [], []
    for f in O.frames(name, W, H, n):
        s, i = enc.encode(f)
        samples.append(s)
        idr.append(i)
        recon.append(enc.recon)
        motion.append((enc.mvs, enc.skip))
        qps.append(enc.qp)
    return samples, idr, recon, motion, qps


def rc_args(W, H, mode):
    """encoded()'s rate arguments for a MODES entry."""
    return dict(bitrate=int(RC_BPP * W * H * FPS)) if mode == 'rc' else dict(bitrate=10 ** 6, qp_range=(mode, mode))


def long_run(name, bitrate, qp_min=0, qp_max=51):
    return encoded(name, 64, 48, gop=RC_GOP, bitrate=bitrate, qp_range=(qp_min, qp_max), fps=RC_FPS, n=RC_FRAMES)


def rate(run):
    return 8 * sum(map(len, run[0])) * RC_FPS / RC_FRAMES


def rc_targets(name):
    """Two targets between the stream rates at pinned QP 40 and QP 10."""
    lo, hi = rate(long_run(name, 10 ** 6, 40, 40)), rate(long_run(name, 10 ** 6, 10, 10))
    return [int(lo * (hi / lo) ** f) for f in (0.25, 0.75)]


def write(path, W, H, run, qp=None, bitrate=None, fps=FPS):
    """Writes an encoded() run as an MP4 file: the constant-QP stream's parameter sets at qp, or the rate-controlled stream's
    (pic_init_qp 26) for bitrate."""
    from next3d_b200 import mp4, video
    samples, idr = run[:2]
    mp4.write_mp4(str(path), W, H, fps, video.sps(W, H, fps, bitrate), video.pps(26 if qp is None else qp), samples,
                  [i for i, x in enumerate(idr) if x])
    return path


def decode(path, rgb):
    cv2 = pytest.importorskip('cv2')
    cap = cv2.VideoCapture(str(path), cv2.CAP_FFMPEG, [] if rgb else [cv2.CAP_PROP_CONVERT_RGB, 0])
    assert cap.isOpened()
    out = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        out.append(f)
    cap.release()
    return out


def bt601_bgr(y, cb, cr, W, H):
    """Limited-range BT.601 YCbCr (chroma repeated 2x2) -> BGR uint8 [H, W, 3]."""
    y = y[:H, :W].astype(np.float64) - 16
    u = np.repeat(np.repeat(cb, 2, 0), 2, 1)[:H, :W].astype(np.float64) - 128
    v = np.repeat(np.repeat(cr, 2, 0), 2, 1)[:H, :W].astype(np.float64) - 128
    r = 1.164 * y + 1.596 * v
    g = 1.164 * y - 0.392 * u - 0.813 * v
    b = 1.164 * y + 2.017 * u
    return np.clip(np.rint(np.stack([b, g, r], -1)), 0, 255).astype(np.uint8)


def assert_decodes_to(path, recon, W, H, rgb=True):
    """FFmpeg decodes path to recon: luma bit for bit, and (rgb) BGR within 3 levels of BT.601 where chroma is locally flat."""
    ys = decode(path, rgb=False)
    assert len(ys) == len(recon)
    for t, (y, rec) in enumerate(zip(ys, recon)):
        y = y.reshape(-1)[:W * H].reshape(H, W)
        assert np.array_equal(y, rec[0][:H, :W]), f'frame {t}: decoded luma differs from the reconstruction'
    if not rgb:
        return
    bgr = decode(path, rgb=True)
    assert len(bgr) == len(recon)
    for t, (f, rec) in enumerate(zip(bgr, recon)):
        assert f.shape == (H, W, 3)
        ref = bt601_bgr(*rec, W, H)
        flat = np.ones((H, W), bool)                      # the decoder interpolates chroma: compare where it is locally constant
        for p in rec[1:]:
            up = np.pad(np.repeat(np.repeat(p.astype(int), 2, 0), 2, 1)[:H, :W], 2, mode='edge')
            for dy in range(5):
                for dx in range(5):
                    flat &= up[dy:dy + H, dx:dx + W] == up[2:2 + H, 2:2 + W]
        diff = np.abs(f.astype(int) - ref)[flat]
        # FFmpeg's fixed-point YCbCr -> BGR conversion lands up to 3 levels below the exact BT.601 formula
        assert diff.size == 0 or diff.max() <= 3, f'frame {t}: BGR differs from BT.601 of the reconstruction by {diff.max()}'


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_oracle_stream_decodes_to_its_reconstruction(tmp_path, case):
    name, W, H, qp, gop = case
    run = encoded(*case)
    assert_decodes_to(write(tmp_path / 'v.mp4', W, H, run, qp=qp), run[2], W, H)


@pytest.mark.parametrize('case', RC_CASES, ids=lambda c: '-'.join(map(str, c)))
def test_rc_stream_decodes_to_its_reconstruction(tmp_path, case):
    name, W, H, mode = case
    args = rc_args(W, H, mode)
    run = encoded(name, W, H, **args)
    assert mode == 'rc' or run[4] == [mode] * len(run[4])
    assert_decodes_to(write(tmp_path / 'v.mp4', W, H, run, bitrate=args['bitrate']), run[2], W, H)


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_rate_controlled_long_streams_decode(tmp_path, name):
    """240 frames with QPs that move every frame and IDR frames every 60: FFmpeg's luma equals the reconstruction."""
    t = rc_targets(name)[0]
    run = long_run(name, t)
    assert len(set(run[4])) > 3
    assert_decodes_to(write(tmp_path / 'v.mp4', 64, 48, run, bitrate=t, fps=RC_FPS), run[2], 64, 48, rgb=False)


@pytest.mark.parametrize('name', ['flat', 'gradient'])
@pytest.mark.parametrize('size', SIZES[:3] + [(512, 512)])
def test_psnr_at_qp18_on_smooth_sequences(name, size):
    W, H = size
    _, _, recon, _, _ = encoded(name, W, H, 18, 3)
    for t, (f, rec) in enumerate(zip(O.sequence(name, W, H), recon)):
        y = O.rgb_to_yuv420(f)[0][:H, :W].astype(np.float64)
        mse = np.mean((y - rec[0][:H, :W]) ** 2)
        psnr = 99.0 if mse == 0 else 10 * np.log10(255 ** 2 / mse)
        assert psnr >= 40, f'frame {t}: luma PSNR {psnr:.1f} dB'


@pytest.mark.parametrize('name', O.SEQUENCES)
@pytest.mark.parametrize('size', SIZES)
def test_stream_size_does_not_grow_with_qp(name, size):
    gops = (3,) if size == (512, 512) else (1, 3)
    for gop in gops:
        sizes = [sum(map(len, encoded(name, *size, qp, gop)[0])) for qp in (0, 18, 40)]
        assert sizes[0] >= sizes[1] >= sizes[2], (gop, sizes)


def test_translation_is_found():
    """At QP 18, >= 90% of the P-frame macroblocks of the translated pattern are P_Skip or carry the true motion vector (at
    512x512: in the small sizes most macroblocks touch the border the pattern enters through)."""
    _, idr, _, motion, _ = encoded('translate', 512, 512, 18, 3)
    hit = total = 0
    for (mvs, skip), i in zip(motion, idr):
        if i:
            continue
        hit += int((skip | (mvs == 4 * np.array(O.TRANSLATE)).all(-1)).sum())
        total += skip.size
    assert total > 0 and hit >= 0.9 * total, (hit, total)


def test_quarter_sample_vectors_are_found():
    """At QP 18, most P macroblocks of the sub-sample pan carry its true vector (5, -2) or are skipped.  The refinement is greedy
    (half samples around the integer vector, then quarter samples around the best half sample), and the pattern's elongated SAD
    valley sends some macroblocks to the neighbouring (4, -1) or (6, -3): about 85 % hit at 512x512."""
    _, idr, _, motion, _ = encoded('pan', 512, 512, bitrate=10 ** 6, qp_range=(18, 18))
    hit = total = 0
    for (mvs, skip), i in zip(motion, idr):
        if i:
            continue
        hit += int((skip | (mvs == np.array([4 * O.PAN[0], 4 * O.PAN[1]])).all(-1)).sum())
        total += skip.size
    print(f'pan at 512x512, QP 18: {hit} of {total} P macroblocks carry (5, -2) or are skipped ({hit / total:.1%})')
    assert total > 0 and hit >= 0.8 * total, (hit, total)


@pytest.mark.parametrize('size', [(48, 32), (512, 512)])
def test_quarter_sample_motion_pays(size):
    """At equal QP, the new stream's P frames of the sub-sample pan are smaller than the constant-QP stream's."""
    W, H = size
    new, idr, *_ = encoded('pan', W, H, bitrate=10 ** 6, qp_range=(18, 18))
    old = encoded('pan', W, H, 18, 3)[0]
    p_new, p_old = sum(len(s) for s, i in zip(new, idr) if not i), sum(len(s) for s, i in zip(old, idr) if not i)
    print(f'pan {W}x{H} QP 18: P frames {p_new} bytes with quarter-sample motion and deblocking, {p_old} without ({p_new / p_old:.2f}x)')
    assert p_new < p_old


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_rate_control_hits_its_target(name):
    """Over 240 frames (64x48, 60 frames/s, an IDR frame every 60), the stream is within 10 % of bitrate x duration for targets
    between the pinned-QP-40 and pinned-QP-10 rates, and consecutive P frames' QPs differ by at most 2."""
    for t in rc_targets(name):
        run = long_run(name, t)
        got, qps, idr = rate(run), run[4], run[1]
        print(f'{name}: target {t} bits/s, got {got:.0f} ({got / t:.3f}x), QP {min(qps)}..{max(qps)}')
        assert abs(got - t) <= 0.1 * t, (t, got)
        pq = [q for q, i in zip(qps, idr) if not i]
        assert max(abs(a - b) for a, b in zip(pq[1:], pq[:-1])) <= 2


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_rate_control_saturates_at_its_bounds(name):
    low, high = long_run(name, 1000), long_run(name, 5 * 10 ** 8)
    assert rate(low) > 1000 and low[4][-RC_GOP:] == [51] * RC_GOP
    assert rate(high) < 5 * 10 ** 8 and high[4][-RC_GOP:] == [0] * RC_GOP


def test_constant_qp_stream_is_unchanged_by_the_new_one():
    """The oracle's constant-QP stream is the one the existing tests pin, whatever the rate-controlled oracle did before."""
    encoded('translate', 48, 32, bitrate=10 ** 6, qp_range=(18, 18))
    enc = O.Encoder(48, 32, 18, 3)
    assert [enc.encode(f)[0] for f in O.sequence('translate', 48, 32)] == encoded('translate', 48, 32, 18, 3)[0]


def _children(data, start, end):
    from next3d_b200 import mp4
    return {k: (s, e) for k, s, e in mp4.parse_boxes(data, start, end)}


def test_mp4_boxes(tmp_path):
    from next3d_b200 import mp4, video
    run = encoded('translate', 40, 24, 18, 2)
    samples = run[0]
    path = write(tmp_path / 'v.mp4', 40, 24, run, qp=18)
    data = path.read_bytes()
    assert [k for k, _, _ in mp4.parse_boxes(data)] == [b'ftyp', b'mdat', b'moov']
    top = _children(data, 0, len(data))
    s, e = top[b'mdat']
    assert data[s:e] == b''.join(samples)
    trak = _children(data, *_children(data, *top[b'moov'])[b'trak'])
    mdia = _children(data, *trak[b'mdia'])
    timescale, duration = struct.unpack('>II', data[mdia[b'mdhd'][0] + 12:mdia[b'mdhd'][0] + 20])
    stbl = _children(data, *_children(data, *mdia[b'minf'])[b'stbl'])
    s, _ = stbl[b'stts']
    assert struct.unpack('>IIII', data[s:s + 16]) == (0, 1, len(samples), timescale // FPS)
    assert duration == len(samples) * timescale // FPS
    s, _ = stbl[b'stsz']
    _, zero, n = struct.unpack('>III', data[s:s + 12])
    assert zero == 0 and n == len(samples)
    assert list(struct.unpack(f'>{n}I', data[s + 12:s + 12 + 4 * n])) == [len(x) for x in samples]
    s, _ = stbl[b'stco']
    offs = struct.unpack(f'>{n}I', data[s + 8:s + 8 + 4 * n])
    assert [data[o:o + len(x)] for o, x in zip(offs, samples)] == samples
    for x in samples:                                        # each sample is length-prefixed NAL units, one slice per MB row
        o, nals = 0, 0
        while o < len(x):
            o += 4 + struct.unpack('>I', x[o:o + 4])[0]
            nals += 1
        assert o == len(x) and nals == 24 // 16 + 1
    s, _ = stbl[b'stss']
    k = struct.unpack('>I', data[s + 4:s + 8])[0]
    assert list(struct.unpack(f'>{k}I', data[s + 8:s + 8 + 4 * k])) == [1, 3]           # frames 0 and 2 (gop 2) are IDR
    s, e = stbl[b'stsd']
    avc1 = _children(data, s + 8, e)[b'avc1']
    avcc = _children(data, avc1[0] + 78, avc1[1])[b'avcC']
    rec = data[avcc[0]:avcc[1]]
    sps, pps = video.sps(40, 24, FPS), video.pps(18)
    assert rec[0] == 1 and rec[1:4] == sps[1:4] and rec[4] == 0xff and rec[5] == 0xe1
    assert struct.unpack('>H', rec[6:8])[0] == len(sps) and rec[8:8 + len(sps)] == sps
    o = 8 + len(sps)
    assert rec[o] == 1 and struct.unpack('>H', rec[o + 1:o + 3])[0] == len(pps) and rec[o + 3:] == pps
    assert sps[1] == 66 and sps[2] == 0xc0 and sps[3] == 10                              # Constrained Baseline, level 1


def test_levels_and_refusals():
    from next3d_b200 import video
    assert video.level_idc(16, 16, 30) == 10
    assert video.level_idc(512, 512, 60) == 31
    assert video.level_idc(2048, 1024, 60) == 42
    assert video.level_idc(8192, 4320, 60) == 61
    for args in [(17, 16, 30, 18, 60), (16, 15, 30, 18, 60), (16, 16, 30, 52, 60), (16, 16, 30, -1, 60), (16, 16, 30, 18, 0),
                 (16896 + 16, 1024, 30, 18, 60), (8192, 8192, 30, 18, 60)]:
        with pytest.raises(ValueError):
            video.check_args(*args)


def test_library_refuses_bad_sizes():
    from next3d_b200 import _lib
    out = [_lib.I64() for _ in range(4)]
    ref = [_lib.C.byref(x) for x in out]
    assert _lib.lib.n3d_h264_buffer_sizes(64, 48, *ref) == 0 and out[0].value == 64 * 48 * 3 // 2
    for w, h in [(17, 16), (16, 15), (0, 16), (16, 16 * 1056), (16 * 400, 16 * 400)]:
        assert _lib.lib.n3d_h264_buffer_sizes(w, h, *ref) == -1 and b'n3d_h264' in _lib.lib.n3d_last_error()


@pytest.mark.parametrize('command', ['gen_videos', 'reenact'])
def test_cli_n3d_encoder_gets_past_the_imageio_refusal(tmp_path, monkeypatch, command):
    """With --encoder n3d and imageio blocked, the run fails only on the missing --network file."""
    from next3d_b200.__main__ import main
    from tests.test_legacy_cpu import _demo_args
    monkeypatch.setitem(sys.modules, 'imageio', None)
    argv = [command, '--seeds', '0', '--outdir', str(tmp_path / 'o'), '--lms_cond', 'True', '--encoder', 'n3d',
            '--network', str(tmp_path / 'missing.pkl')]
    argv += ['--drive_root', 'd'] if command == 'reenact' else _demo_args(tmp_path)
    with pytest.raises(FileNotFoundError, match='missing.pkl'):
        main(argv)
    with pytest.raises(SystemExit, match='qp'):
        main(argv + ['--qp', '52'])


def test_bitrate_parsing_levels_and_refusals():
    from next3d_b200 import video
    assert video.parse_bitrate('10M') == 10 ** 7 and video.parse_bitrate('800k') == 800000 and video.parse_bitrate(12345) == 12345
    assert video.parse_bitrate('1.5M') == 1500000
    for bad in ['0', '-1M', 'fast', '10Mb', '', 0, -5, 1.5, None, True]:
        with pytest.raises(ValueError):
            video.parse_bitrate(bad)
    assert video.level_idc(512, 512, 60) == 31 and video.level_idc(512, 512, 60, 12 * 10 ** 6) == 31
    assert video.level_idc(512, 512, 60, 15 * 10 ** 6) == 32
    assert video.level_idc(16, 16, 30, 100000) == 11
    with pytest.raises(ValueError):
        video.level_idc(512, 512, 60, 900 * 10 ** 6)
    with pytest.raises(ValueError):
        video.check_args(16, 16, 30, 18, 60, 10 ** 9)


def test_library_refuses_bad_rc_arguments():
    from next3d_b200 import _lib
    st = (_lib.C.c_int64 * (_lib.H264_RC_STATE_BYTES // 8))()
    p = _lib.C.addressof(st)
    for args, msg in [((None, 64, 48, 10 ** 6, 30, 1, 0, 51), b'null state'), ((p, 63, 48, 10 ** 6, 30, 1, 0, 51), b'even'),
                      ((p, 64, 48, 0, 30, 1, 0, 51), b'bits_per_second'), ((p, 64, 48, 1 << 32, 30, 1, 0, 51), b'bits_per_second'),
                      ((p, 64, 48, 10 ** 6, 0, 1, 0, 51), b'frame rate'), ((p, 64, 48, 10 ** 6, 30, 0, 0, 51), b'frame rate'),
                      ((p, 64, 48, 10 ** 6, 30, 1, 20, 19), b'qp bounds'), ((p, 64, 48, 10 ** 6, 30, 1, -1, 51), b'qp bounds'),
                      ((p, 64, 48, 10 ** 6, 30, 1, 0, 52), b'qp bounds')]:
        assert _lib.lib.n3d_h264_rc_init(*args, None) == -1, args                    # refused before any launch
        assert msg in _lib.lib.n3d_last_error(), (args, _lib.lib.n3d_last_error())
    assert _lib.lib.n3d_h264_encode_rc(None, 64, 48, None, 1, 0, 0, None, None, None, None, None, None, None, None) == -1
    assert b'null state' in _lib.lib.n3d_last_error()


def test_writer_refuses_bad_rates():
    from next3d_b200.video import H264Writer
    for kw in [dict(bitrate=0), dict(bitrate='-2M'), dict(bitrate='ten'), dict(bitrate='10M', qp_range=(30, 20)),
               dict(bitrate='10M', qp_range=(0, 52)), dict(bitrate='900M')]:
        with pytest.raises(ValueError):
            H264Writer('unused.mp4', 512, 512, 60, device='cuda', **kw)


@pytest.mark.parametrize('command', ['gen_videos', 'reenact'])
def test_cli_bitrate(tmp_path, monkeypatch, command):
    """--bitrate needs --encoder n3d, a valid rate and no --qp; with those it gets as far as the missing --network file."""
    from next3d_b200.__main__ import main
    from tests.test_legacy_cpu import _demo_args
    monkeypatch.setitem(sys.modules, 'imageio', None)
    argv = [command, '--seeds', '0', '--outdir', str(tmp_path / 'o'), '--lms_cond', 'True', '--network', str(tmp_path / 'missing.pkl')]
    argv += ['--drive_root', 'd'] if command == 'reenact' else _demo_args(tmp_path)
    for rate in ['script', '8M']:
        with pytest.raises(FileNotFoundError, match='missing.pkl'):
            main(argv + ['--encoder', 'n3d', '--bitrate', rate])
    with pytest.raises(SystemExit, match='--encoder n3d'):
        main(argv + ['--bitrate', '8M'])
    with pytest.raises(SystemExit, match='--bitrate'):
        main(argv + ['--encoder', 'n3d', '--bitrate', 'fast'])
    with pytest.raises(SystemExit, match='--qp'):
        main(argv + ['--encoder', 'n3d', '--bitrate', '8M', '--qp', '18'])
    with pytest.raises(FileNotFoundError, match='missing.pkl'):
        main(argv + ['--encoder', 'n3d', '--qp', '18'])
