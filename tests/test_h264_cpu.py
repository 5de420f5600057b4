"""CPU: the H.264 byte format.  Streams of the numpy restatement of the encoder (tests/h264_oracle.py, which the GPU encoder
matches byte for byte in tests/test_gpu_h264.py) are written through next3d_b200.mp4 and decoded by FFmpeg (OpenCV's
CAP_FFMPEG backend): the decoder's luma equals the encoder's reconstruction bit for bit, its BGR output matches the
reconstruction converted with BT.601, and the MP4 boxes parse back.  Also the CLI's --encoder n3d path up to loading the
network, and the argument refusals of next3d_b200.video."""
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


@functools.lru_cache(maxsize=None)
def encoded(name, W, H, qp, gop):
    """Oracle stream: (samples, IDR flags, recon planes per frame, (mvs, skip) per frame)."""
    enc = O.Encoder(W, H, qp, gop)
    samples, idr, recon, motion = [], [], [], []
    for f in O.sequence(name, W, H):
        s, i = enc.encode(f)
        samples.append(s)
        idr.append(i)
        recon.append(enc.recon)
        motion.append((enc.mvs, enc.skip))
    return samples, idr, recon, motion


def write(path, case):
    from next3d_b200 import mp4, video
    name, W, H, qp, gop = case
    samples, idr, _, _ = encoded(*case)
    mp4.write_mp4(str(path), W, H, FPS, video.sps(W, H, FPS), video.pps(qp), samples, [i for i, x in enumerate(idr) if x])
    return samples


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


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_oracle_stream_decodes_to_its_reconstruction(tmp_path, case):
    name, W, H, qp, gop = case
    path = tmp_path / 'v.mp4'
    write(path, case)
    _, _, recon, _ = encoded(*case)
    ys = decode(path, rgb=False)
    assert len(ys) == len(recon)
    for t, (y, rec) in enumerate(zip(ys, recon)):
        y = y.reshape(-1)[:W * H].reshape(H, W) if y.size != W * H else y.reshape(H, W)
        assert np.array_equal(y, rec[0][:H, :W]), f'frame {t}: decoded luma differs from the reconstruction'
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


@pytest.mark.parametrize('name', ['flat', 'gradient'])
@pytest.mark.parametrize('size', SIZES[:3] + [(512, 512)])
def test_psnr_at_qp18_on_smooth_sequences(name, size):
    W, H = size
    _, _, recon, _ = encoded(name, W, H, 18, 3)
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
    _, idr, _, motion = encoded('translate', 512, 512, 18, 3)
    hit = total = 0
    for (mvs, skip), i in zip(motion, idr):
        if i:
            continue
        hit += int((skip | (mvs == np.array(O.TRANSLATE)).all(-1)).sum())
        total += skip.size
    assert total > 0 and hit >= 0.9 * total, (hit, total)


def _children(data, start, end):
    from next3d_b200 import mp4
    return {k: (s, e) for k, s, e in mp4.parse_boxes(data, start, end)}


def test_mp4_boxes(tmp_path):
    from next3d_b200 import mp4, video
    case = ('translate', 40, 24, 18, 2)
    path = tmp_path / 'v.mp4'
    samples = write(path, case)
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
