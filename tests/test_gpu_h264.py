"""GPU: the sm_90a H.264 encoder (csrc/h264.cu through next3d_b200.video.H264Writer) writes, in both streams, the same bytes as
its numpy restatement (tests/h264_oracle.py, whose streams FFmpeg decodes to their reconstruction in tests/test_h264_cpu.py),
the same reconstruction and, under rate control, the same QP sequence, for the CPU suite's cases and for rendered frames; the
rate-controlled stream hits its targets on a rendered orbit; the entry points refuse bad arguments; and the CLI's --encoder n3d
writes a playable file at a QP and at the scripts' bitrates."""
import struct

import numpy as np
import pytest
import torch

from tests import h264_oracle as O
from tests.test_h264_cpu import (CASES, FPS, RC_CASES, RC_FPS, RC_FRAMES, RC_GOP, encoded, long_run, oracle, rc_args,
                                 rc_targets)

pytestmark = pytest.mark.gpu
DEV = 'cuda'
STREAMS = {'cq': dict(qp=18), 'rc': dict(bitrate=12 * 10 ** 6)}       # the rendered frames' stream arguments


def read_samples(path):
    """(samples, 0-based IDR indices) of the one video track of an MP4 written by next3d_b200.mp4."""
    from next3d_b200 import mp4
    data = open(path, 'rb').read()
    kids = lambda s, e: {k: (a, b) for k, a, b in mp4.parse_boxes(data, s, e)}
    top = kids(0, len(data))
    stbl = kids(*kids(*kids(*kids(*kids(*top[b'moov'])[b'trak'])[b'mdia'])[b'minf'])[b'stbl'])
    s, _ = stbl[b'stsz']
    n = struct.unpack('>I', data[s + 8:s + 12])[0]
    sizes = struct.unpack(f'>{n}I', data[s + 12:s + 12 + 4 * n])
    s, _ = stbl[b'stco']
    offs = struct.unpack(f'>{n}I', data[s + 8:s + 8 + 4 * n])
    s, _ = stbl[b'stss']
    k = struct.unpack('>I', data[s + 4:s + 8])[0]
    return [data[o:o + z] for o, z in zip(offs, sizes)], [i - 1 for i in struct.unpack(f'>{k}I', data[s + 8:s + 8 + 4 * k])]


def gpu_encode(path, frames, W, H, gop, fps=FPS, batch=2, keep_recon=True, **stream):
    """Encode frame by frame from CUDA tensors with H264Writer(..., **stream) (qp=, or bitrate= and qp_range=); returns (samples,
    IDR indices, recon planes per frame, or [] without keep_recon)."""
    from next3d_b200.video import H264Writer
    recon = []
    with H264Writer(str(path), W, H, fps, gop=gop, batch=batch, **stream) as w:
        for f in frames:
            w.write(torch.as_tensor(f).to(DEV))
            if keep_recon:
                recon.append(tuple(p.cpu().numpy() for p in w.recon))
    return (*read_samples(path), recon)


def oracle_encode(frames, W, H, gop, fps=FPS, **stream):
    enc = oracle(W, H, gop, fps=fps, **stream)
    samples, idr, recon = [], [], []
    for i, f in enumerate(frames):
        s, k = enc.encode(f)
        samples.append(s)
        recon.append(enc.recon)
        if k:
            idr.append(i)
    return samples, idr, recon


def assert_same(got, want):
    """The same samples and IDR frames, and the same reconstructions unless got has none."""
    (gs, gi, gr), (ws, wi, wr) = got, want
    assert len(gs) == len(ws) and gi == wi
    for t in range(len(ws)):
        if gr:
            for p, (a, b) in enumerate(zip(gr[t], wr[t])):
                assert np.array_equal(a, b), f'frame {t}: reconstruction plane {p} differs ({int((a != b).sum())} samples)'
        assert gs[t] == ws[t], f'frame {t}: {len(gs[t])} bytes, the oracle {len(ws[t])}'


def idr_indices(run):
    return [i for i, x in enumerate(run[1]) if x]


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_gpu_stream_equals_oracle(tmp_path, case):
    name, W, H, qp, gop = case
    run = encoded(*case)
    got = gpu_encode(tmp_path / 'v.mp4', O.sequence(name, W, H), W, H, gop, qp=qp)
    assert_same(got, (run[0], idr_indices(run), run[2]))


@pytest.mark.parametrize('case', RC_CASES, ids=lambda c: '-'.join(map(str, c)))
def test_gpu_rc_stream_equals_oracle(tmp_path, case):
    name, W, H, mode = case
    args = rc_args(W, H, mode)
    run = encoded(name, W, H, **args)
    got = gpu_encode(tmp_path / 'v.mp4', O.frames(name, W, H), W, H, 3, **args)
    assert_same(got, (run[0], idr_indices(run), run[2]))


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_gpu_rc_long_streams_equal_oracle(tmp_path, name):
    """240 frames under the controller, at both targets and at the saturating ones: the same bytes, so the same QP sequence."""
    frames = O.frames(name, 64, 48, RC_FRAMES)
    for t in rc_targets(name) + [1000, 5 * 10 ** 8]:
        run = long_run(name, t)
        got = gpu_encode(tmp_path / 'v.mp4', frames, 64, 48, RC_GOP, fps=RC_FPS, batch=8, keep_recon=False, bitrate=t)
        assert_same(got, (run[0], idr_indices(run), []))


def test_numpy_batches_and_deferred_copies(tmp_path):
    """A numpy batch, copied to the device by the writer, with several frames per host copy: the same bytes."""
    from next3d_b200.video import H264Writer
    frames = O.sequence('translate', 48, 32, 7)
    with H264Writer(str(tmp_path / 'v.mp4'), 48, 32, FPS, qp=18, gop=4, batch=3) as w:
        w.write(np.stack(frames[:5]))
        w.write(frames[5])
        w.write(frames[6])
    samples, idr = read_samples(tmp_path / 'v.mp4')
    want = oracle_encode(frames, 48, 32, 4, qp=18)
    assert idr == want[1] == [0, 4] and samples == want[0]


def _rendered(tiny, kind):
    from next3d_b200 import drivers, weights
    cfg, G = tiny
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device=DEV)
    if kind == 'orbit':
        rk = G.rendering_kwargs
        ws = drivers.grid_keyframes(G, [3], (1, 1), truncation_psi=0.7)[0, 0]
        cams = drivers.orbit_camera_params(16, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
        return list(drivers.render_orbit(G, ws[:1], cams, v, seed=0))
    ws_grid = drivers.grid_keyframes(G, [0, 1, 2, 3], (2, 1), truncation_psi=0.7)
    return list(drivers.render_grid_frames(G, ws_grid, v, 8, seed=0))


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    return cfg, G


@pytest.mark.parametrize('stream', list(STREAMS))
@pytest.mark.parametrize('kind', ['orbit', 'grid2x1'])
def test_rendered_frames_equal_oracle(tmp_path, tiny, kind, stream):
    frames = _rendered(tiny, kind)
    assert len(frames) == 16
    H, W, _ = frames[0].shape
    got = gpu_encode(tmp_path / 'v.mp4', frames, W, H, 60, fps=60, batch=8, **STREAMS[stream])
    assert_same(got, oracle_encode(frames, W, H, 60, fps=60, **STREAMS[stream]))
    try:
        import cv2
    except ImportError:
        pytest.skip('cv2 is not importable here: the decode of these streams rests on the oracle, which FFmpeg decodes in '
                    'tests/test_h264_cpu.py')
    cap = cv2.VideoCapture(str(tmp_path / 'v.mp4'), cv2.CAP_FFMPEG, [cv2.CAP_PROP_CONVERT_RGB, 0])
    n = 0
    while True:
        ok, y = cap.read()
        if not ok:
            break
        assert np.array_equal(y.reshape(-1)[:W * H].reshape(H, W), got[2][n][0][:H, :W]), f'frame {n}'
        n += 1
    assert n == len(frames)


def test_rendered_orbit_hits_its_targets(tmp_path, tiny):
    """240 rendered orbit frames at 512x512, 60 frames/s: within 10 % of targets between the pinned-QP-40 and QP-10 rates."""
    from next3d_b200 import drivers, weights
    cfg, G = tiny
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device=DEV)
    rk = G.rendering_kwargs
    ws = drivers.grid_keyframes(G, [3], (1, 1), truncation_psi=0.7)[0, 0]
    cams = drivers.orbit_camera_params(240, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    frames = [torch.as_tensor(f).to(DEV) for f in drivers.render_orbit(G, ws[:1], cams, v, seed=0)]
    H, W, _ = frames[0].shape

    def rate(bitrate, qp_range):
        s, _, _ = gpu_encode(tmp_path / 'o.mp4', frames, W, H, 60, fps=60, batch=16, keep_recon=False, bitrate=bitrate,
                             qp_range=qp_range)
        return 8 * sum(map(len, s)) * 60 / len(s)
    lo, hi = rate(10 ** 6, (40, 40)), rate(10 ** 6, (10, 10))
    for f in (0.25, 0.75):
        t = int(lo * (hi / lo) ** f)
        got = rate(t, (0, 51))
        print(f'orbit {W}x{H}: target {t} bits/s, got {got:.0f} ({got / t:.3f}x); pinned QP 40: {lo:.0f}, QP 10: {hi:.0f}')
        assert abs(got - t) <= 0.1 * t, (t, got)


@pytest.mark.parametrize('stream', list(STREAMS))
def test_encode_refuses_bad_arguments(stream):
    """n3d_h264_encode (a P frame at QP 18) and n3d_h264_encode_rc (an IDR frame under a fresh controller) write a frame, then
    refuse each bad argument; n3d_h264_rc_init refuses bad rates and bounds."""
    from next3d_b200 import _lib
    rc = stream == 'rc'
    sizes = [_lib.I64() for _ in range(4)]
    assert _lib.lib.n3d_h264_buffer_sizes(32, 32, *[_lib.C.byref(s) for s in sizes]) == 0
    plane, scratch, slices, sample = (torch.zeros(s.value, dtype=torch.uint8, device=DEV) for s in sizes)
    rgb, ref, out_len = torch.zeros(32 * 32 * 3, dtype=torch.uint8, device=DEV), torch.zeros_like(plane), torch.zeros(1, dtype=torch.int64, device=DEV)
    cur = torch.zeros_like(plane)
    st = torch.zeros(_lib.H264_RC_STATE_BYTES // 8, dtype=torch.int64, device=DEV)
    cuda_stream = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    if rc:
        assert _lib.lib.n3d_h264_rc_init(p(st), 32, 32, 10 ** 6, 30, 1, 0, 51, cuda_stream) == 0
        for args in [(None, 32, 32, 10 ** 6, 30, 1, 0, 51), (p(st), 31, 32, 10 ** 6, 30, 1, 0, 51), (p(st), 32, 32, 0, 30, 1, 0, 51),
                     (p(st), 32, 32, 10 ** 6, 30, 0, 0, 51), (p(st), 32, 32, 10 ** 6, 30, 1, 30, 29)]:
            assert _lib.lib.n3d_h264_rc_init(*args, cuda_stream) == -1, args                  # N3D_ERR_INVALID_ARG

    def call(**kw):
        a = dict(rgb=p(rgb), w=32, h=32, qp=18, st=p(st), idr=int(rc), fn=int(not rc), idr_id=0, cur=p(cur), ref=p(ref), rec=p(plane),
                 scratch=p(scratch), slices=p(slices), sample=p(sample), n=p(out_len))
        a.update(kw)
        entry, qp_or_state = (_lib.lib.n3d_h264_encode_rc, a['st']) if rc else (_lib.lib.n3d_h264_encode, a['qp'])
        return entry(a['rgb'], a['w'], a['h'], qp_or_state, a['idr'], a['fn'], a['idr_id'], a['cur'], a['ref'], a['rec'], a['scratch'],
                     a['slices'], a['sample'], a['n'], cuda_stream)
    assert call() == 0
    torch.cuda.synchronize()
    assert out_len.item() > 0
    if rc:
        assert st[5].item() == 0          # 32 bits per pixel: the first QP is 0, kept after the first IDR frame
    refusals = [(dict(rgb=None), b'null'), (dict(sample=None), b'null'), (dict(idr=0, ref=None), b'null ref'),
                (dict(rec=p(ref)), b'different'), (dict(w=31), b'even'), (dict(h=30, w=33), b'even'),
                (dict(w=16 * 400, h=16 * 400), b'level 6.2'), (dict(fn=16), b'frame_num')]
    refusals += [(dict(st=None), b'null state')] if rc else [(dict(qp=52), b'qp 52'), (dict(qp=-1), b'qp')]
    for kw, msg in refusals:
        assert call(**kw) == -1, kw                                     # N3D_ERR_INVALID_ARG
        assert msg in _lib.lib.n3d_last_error(), (kw, _lib.lib.n3d_last_error())
    torch.cuda.synchronize()


@pytest.mark.parametrize('args', [['--qp', '24'], ['--bitrate', 'script']], ids=list(STREAMS))
def test_cli_gen_videos_n3d_grid(tmp_path, monkeypatch, args):
    import sys
    from next3d_b200 import config, mp4, weights
    from next3d_b200.__main__ import main
    from tests.test_gpu_legacy import _mask
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    cfg = config.tiny_config(512)
    net = tmp_path / 'tiny.pkl'
    net.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    monkeypatch.setitem(sys.modules, 'imageio', None)                  # the n3d encoder never imports imageio
    out = tmp_path / 'out'
    main(['gen_videos', '--network', str(net), '--seeds', '0-3', '--grid', '2x1', '--w-frames', '2', '--outdir', str(out),
          '--lms_cond', 'True', '--encoder', 'n3d', *args, *_demo_args(tmp_path)])
    samples, idr = read_samples(out / 'interpolation.mp4')
    assert len(samples) == 2 * 2 and idr == [0]                            # 2 keyframes per cell x 2 frames each
    data = (out / 'interpolation.mp4').read_bytes()
    assert [k for k, _, _ in mp4.parse_boxes(data)] == [b'ftyp', b'mdat', b'moov']
    try:
        import cv2
    except ImportError:
        return
    cap = cv2.VideoCapture(str(out / 'interpolation.mp4'), cv2.CAP_FFMPEG)
    n = 0
    while cap.read()[0]:
        n += 1
    assert n == 4
