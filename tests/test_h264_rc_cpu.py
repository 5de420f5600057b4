"""CPU: the rate-controlled H.264 stream (quarter-sample motion, deblocking, a QP per picture from the rate controller).  Streams
of its numpy restatement (tests/h264_rc_oracle.py, which the kernels match byte for byte in tests/test_gpu_h264_rc.py) are
decoded by FFmpeg (OpenCV's CAP_FFMPEG backend): the decoder's luma equals the oracle's deblocked reconstruction bit for bit.
Also the quarter-sample search, the controller against its targets, the writer's and the CLI's refusals, and the level."""
import functools
import sys

import numpy as np
import pytest

from tests import h264_oracle as O
from tests import h264_rc_oracle as R
from tests.test_h264_cpu import FPS, SIZES, bt601_bgr, decode, encoded

MODES = (0, 18, 40, 'rc')                  # pinned QPs, and the controller at RC_BPP
RC_BPP = 1.0                               # bits per pixel of the 'rc' mode's target
CASES = [(name, W, H, mode) for name in O.SEQUENCES + ('pan',) for (W, H) in SIZES for mode in MODES
         if (W, H) != (512, 512) or (name in ('translate', 'pan') and mode in (18, 'rc'))]      # 512x512: bounds the run time
RC_FPS, RC_GOP, RC_FRAMES = 60, 60, 240


def rc_args(W, H, mode):
    """(bitrate, qp_min, qp_max) of a MODES entry."""
    return (int(RC_BPP * W * H * FPS), 0, 51) if mode == 'rc' else (10 ** 6, mode, mode)


@functools.lru_cache(maxsize=None)
def rc_encoded(name, W, H, bitrate, qp_min, qp_max, fps=FPS, gop=3, n=3):
    """Oracle stream: (samples, IDR flags, recon planes per frame, (mvs, skip) per frame, QP per frame)."""
    enc = R.RcEncoder(W, H, bitrate, (fps, 1), gop, qp_min, qp_max)
    samples, idr, recon, motion = [], [], [], []
    for f in R.frames(name, W, H, n):
        s, i = enc.encode(f)
        samples.append(s)
        idr.append(i)
        recon.append(enc.recon)
        motion.append((enc.mvs, enc.skip))
    return samples, idr, recon, motion, list(enc.qps)


def long_run(name, bitrate, qp_min=0, qp_max=51):
    return rc_encoded(name, 64, 48, bitrate, qp_min, qp_max, RC_FPS, RC_GOP, RC_FRAMES)


def rate(run):
    return 8 * sum(map(len, run[0])) * RC_FPS / RC_FRAMES


def rc_targets(name):
    """Two targets between the stream rates at pinned QP 40 and QP 10."""
    lo, hi = rate(long_run(name, 10 ** 6, 40, 40)), rate(long_run(name, 10 ** 6, 10, 10))
    return [int(lo * (hi / lo) ** f) for f in (0.25, 0.75)]


def write_and_decode(tmp_path, W, H, fps, samples, idr, bitrate):
    from next3d_b200 import mp4, video
    path = tmp_path / 'v.mp4'
    mp4.write_mp4(str(path), W, H, fps, video.sps(W, H, fps, bitrate), video.pps(26), samples, [i for i, x in enumerate(idr) if x])
    return path


def assert_decodes_to(path, recon, W, H, rgb=True):
    ys = decode(path, rgb=False)
    assert len(ys) == len(recon)
    for t, (y, rec) in enumerate(zip(ys, recon)):
        y = y.reshape(-1)[:W * H].reshape(H, W)
        assert np.array_equal(y, rec[0][:H, :W]), f'frame {t}: decoded luma differs from the deblocked reconstruction'
    if not rgb:
        return
    for t, (f, rec) in enumerate(zip(decode(path, rgb=True), recon)):
        ref = bt601_bgr(*rec, W, H)
        flat = np.ones((H, W), bool)                      # the decoder interpolates chroma: compare where it is locally constant
        for p in rec[1:]:
            up = np.pad(np.repeat(np.repeat(p.astype(int), 2, 0), 2, 1)[:H, :W], 2, mode='edge')
            for dy in range(5):
                for dx in range(5):
                    flat &= up[dy:dy + H, dx:dx + W] == up[2:2 + H, 2:2 + W]
        diff = np.abs(f.astype(int) - ref)[flat]
        assert diff.size == 0 or diff.max() <= 3, f'frame {t}: BGR differs from BT.601 of the reconstruction by {diff.max()}'


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_rc_stream_decodes_to_its_reconstruction(tmp_path, case):
    name, W, H, mode = case
    bitrate, lo, hi = rc_args(W, H, mode)
    samples, idr, recon, _, qps = rc_encoded(name, W, H, bitrate, lo, hi)
    assert mode == 'rc' or qps == [mode] * len(qps)
    assert_decodes_to(write_and_decode(tmp_path, W, H, FPS, samples, idr, bitrate), recon, W, H)


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_rate_controlled_long_streams_decode(tmp_path, name):
    """240 frames with QPs that move every frame and IDR frames every 60: FFmpeg's luma equals the reconstruction."""
    t = rc_targets(name)[0]
    samples, idr, recon, _, qps = long_run(name, t)
    assert len(set(qps)) > 3
    assert_decodes_to(write_and_decode(tmp_path, 64, 48, RC_FPS, samples, idr, t), recon, 64, 48, rgb=False)


def test_quarter_sample_vectors_are_found():
    """At QP 18, most P macroblocks of the sub-sample pan carry its true vector (5, -2) or are skipped.  The refinement is greedy
    (half samples around the integer vector, then quarter samples around the best half sample), and the pattern's elongated SAD
    valley sends some macroblocks to the neighbouring (4, -1) or (6, -3): about 85 % hit at 512x512."""
    _, idr, _, motion, _ = rc_encoded('pan', 512, 512, 10 ** 6, 18, 18)
    hit = total = 0
    for (mvs, skip), i in zip(motion, idr):
        if i:
            continue
        hit += int((skip | (mvs == np.array([4 * R.PAN[0], 4 * R.PAN[1]])).all(-1)).sum())
        total += skip.size
    print(f'pan at 512x512, QP 18: {hit} of {total} P macroblocks carry (5, -2) or are skipped ({hit / total:.1%})')
    assert total > 0 and hit >= 0.8 * total, (hit, total)


@pytest.mark.parametrize('size', [(48, 32), (512, 512)])
def test_quarter_sample_motion_pays(size):
    """At equal QP, the new stream's P frames of the sub-sample pan are smaller than the constant-QP stream's."""
    W, H = size
    new, idr, *_ = rc_encoded('pan', W, H, 10 ** 6, 18, 18)
    enc = O.Encoder(W, H, 18, 3)
    old = [enc.encode(f)[0] for f in R.frames('pan', W, H)]
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
    rc_encoded('translate', 48, 32, 10 ** 6, 18, 18)
    enc = O.Encoder(48, 32, 18, 3)
    assert [enc.encode(f)[0] for f in O.sequence('translate', 48, 32)] == encoded('translate', 48, 32, 18, 3)[0]


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
