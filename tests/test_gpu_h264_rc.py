"""GPU: the rate-controlled stream of the sm_90a H.264 encoder (n3d_h264_encode_rc through H264Writer(bitrate=...)) writes the
same bytes, reconstructions and QP sequence as its numpy restatement (tests/h264_rc_oracle.py, whose streams FFmpeg decodes to
their reconstruction in tests/test_h264_rc_cpu.py), for the CPU suite's cases and for rendered frames; it hits its targets on a
rendered orbit; the entry points refuse bad arguments; and `--bitrate script` writes a playable file."""
import numpy as np
import pytest
import torch

from tests import h264_rc_oracle as R
from tests.test_gpu_h264 import DEV, _rendered, read_samples, tiny  # noqa: F401  (tiny: fixture)
from tests.test_h264_cpu import FPS
from tests.test_h264_rc_cpu import CASES, RC_FPS, RC_FRAMES, RC_GOP, long_run, rc_args, rc_encoded, rc_targets

pytestmark = pytest.mark.gpu


def gpu_encode(path, frames, W, H, bitrate, qp_range, gop, fps=FPS, batch=2, keep_recon=True):
    """Encode frame by frame from CUDA tensors; returns (samples, IDR indices, recon planes per frame)."""
    from next3d_b200.video import H264Writer
    recon = []
    with H264Writer(str(path), W, H, fps, gop=gop, batch=batch, bitrate=bitrate, qp_range=qp_range) as w:
        for f in frames:
            w.write(torch.as_tensor(f).to(DEV))
            if keep_recon:
                recon.append(tuple(p.cpu().numpy() for p in w.recon))
    return (*read_samples(path), recon)


def oracle_encode(frames, W, H, bitrate, qp_range, gop, fps):
    enc = R.RcEncoder(W, H, bitrate, (fps, 1), gop, *qp_range)
    samples, idr, recon = [], [], []
    for i, f in enumerate(frames):
        s, k = enc.encode(f)
        samples.append(s)
        recon.append(enc.recon)
        if k:
            idr.append(i)
    return samples, idr, recon


def assert_same(got, want):
    (gs, gi, gr), (ws, wi, wr) = got, want
    assert len(gs) == len(ws) and gi == wi
    for t in range(len(ws)):
        if gr:
            for p, (a, b) in enumerate(zip(gr[t], wr[t])):
                assert np.array_equal(a, b), f'frame {t}: reconstruction plane {p} differs ({int((a != b).sum())} samples)'
        assert gs[t] == ws[t], f'frame {t}: {len(gs[t])} bytes, the oracle {len(ws[t])}'


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_gpu_rc_stream_equals_oracle(tmp_path, case):
    name, W, H, mode = case
    bitrate, lo, hi = rc_args(W, H, mode)
    samples, idr, recon, _, _ = rc_encoded(name, W, H, bitrate, lo, hi)
    got = gpu_encode(tmp_path / 'v.mp4', R.frames(name, W, H), W, H, bitrate, (lo, hi), 3)
    assert_same(got, (samples, [i for i, x in enumerate(idr) if x], recon))


@pytest.mark.parametrize('name', ['translate', 'pan'])
def test_gpu_rc_long_streams_equal_oracle(tmp_path, name):
    """240 frames under the controller, at both targets and at the saturating ones: the same bytes, so the same QP sequence."""
    frames = R.frames(name, 64, 48, RC_FRAMES)
    for t in rc_targets(name) + [1000, 5 * 10 ** 8]:
        samples, idr, recon, _, _ = long_run(name, t)
        got = gpu_encode(tmp_path / 'v.mp4', frames, 64, 48, t, (0, 51), RC_GOP, fps=RC_FPS, batch=8, keep_recon=False)
        assert_same(got, (samples, [i for i, x in enumerate(idr) if x], []))


@pytest.mark.parametrize('kind', ['orbit', 'grid2x1'])
def test_rendered_frames_equal_oracle(tmp_path, tiny, kind):
    frames = _rendered(tiny, kind)
    H, W, _ = frames[0].shape
    bitrate = 12 * 10 ** 6
    got = gpu_encode(tmp_path / 'v.mp4', frames, W, H, bitrate, (0, 51), 60, fps=60, batch=8)
    assert_same(got, oracle_encode(frames, W, H, bitrate, (0, 51), 60, 60))
    try:
        import cv2
    except ImportError:
        pytest.skip('cv2 is not importable here: the decode of these streams rests on the oracle, which FFmpeg decodes in '
                    'tests/test_h264_rc_cpu.py')
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
        s, _, _ = gpu_encode(tmp_path / 'o.mp4', frames, W, H, bitrate, qp_range, 60, fps=60, batch=16, keep_recon=False)
        return 8 * sum(map(len, s)) * 60 / len(s)
    lo, hi = rate(10 ** 6, (40, 40)), rate(10 ** 6, (10, 10))
    for f in (0.25, 0.75):
        t = int(lo * (hi / lo) ** f)
        got = rate(t, (0, 51))
        print(f'orbit {W}x{H}: target {t} bits/s, got {got:.0f} ({got / t:.3f}x); pinned QP 40: {lo:.0f}, QP 10: {hi:.0f}')
        assert abs(got - t) <= 0.1 * t, (t, got)


def test_rc_entry_points_refuse_bad_arguments():
    from next3d_b200 import _lib
    sizes = [_lib.I64() for _ in range(4)]
    assert _lib.lib.n3d_h264_buffer_sizes(32, 32, *[_lib.C.byref(s) for s in sizes]) == 0
    plane, scratch, slices, sample = (torch.zeros(s.value, dtype=torch.uint8, device=DEV) for s in sizes)
    rgb, ref, out_len = torch.zeros(32 * 32 * 3, dtype=torch.uint8, device=DEV), torch.zeros_like(plane), torch.zeros(1, dtype=torch.int64, device=DEV)
    cur = torch.zeros_like(plane)
    st = torch.zeros(_lib.H264_RC_STATE_BYTES // 8, dtype=torch.int64, device=DEV)
    stream = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()
    assert _lib.lib.n3d_h264_rc_init(p(st), 32, 32, 10 ** 6, 30, 1, 0, 51, stream) == 0
    for args in [(None, 32, 32, 10 ** 6, 30, 1, 0, 51), (p(st), 31, 32, 10 ** 6, 30, 1, 0, 51), (p(st), 32, 32, 0, 30, 1, 0, 51),
                 (p(st), 32, 32, 10 ** 6, 30, 0, 0, 51), (p(st), 32, 32, 10 ** 6, 30, 1, 30, 29)]:
        assert _lib.lib.n3d_h264_rc_init(*args, stream) == -1, args                      # N3D_ERR_INVALID_ARG

    def call(**kw):
        a = dict(rgb=p(rgb), w=32, h=32, st=p(st), idr=1, fn=0, idr_id=0, cur=p(cur), ref=p(ref), rec=p(plane), scratch=p(scratch),
                 slices=p(slices), sample=p(sample), n=p(out_len))
        a.update(kw)
        return _lib.lib.n3d_h264_encode_rc(a['rgb'], a['w'], a['h'], a['st'], a['idr'], a['fn'], a['idr_id'], a['cur'], a['ref'],
                                           a['rec'], a['scratch'], a['slices'], a['sample'], a['n'], stream)
    assert call() == 0
    torch.cuda.synchronize()
    assert out_len.item() > 0 and st[5].item() == 0          # 32 bits per pixel: the first QP is 0, kept after the first IDR frame
    for kw, msg in [(dict(st=None), b'null state'), (dict(rgb=None), b'null'), (dict(idr=0, ref=None), b'null ref'),
                    (dict(rec=p(ref)), b'different'), (dict(w=31), b'even'), (dict(w=16 * 400, h=16 * 400), b'level 6.2'),
                    (dict(fn=16), b'frame_num')]:
        assert call(**kw) == -1, kw
        assert msg in _lib.lib.n3d_last_error(), (kw, _lib.lib.n3d_last_error())
    torch.cuda.synchronize()


def test_cli_gen_videos_bitrate_script(tmp_path, monkeypatch):
    import sys
    from next3d_b200.__main__ import main
    from tests.test_gpu_legacy import _mask
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    from next3d_b200 import config, weights
    cfg = config.tiny_config(512)
    net = tmp_path / 'tiny.pkl'
    net.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    monkeypatch.setitem(sys.modules, 'imageio', None)
    out = tmp_path / 'out'
    main(['gen_videos', '--network', str(net), '--seeds', '0-3', '--grid', '2x1', '--w-frames', '2', '--outdir', str(out),
          '--lms_cond', 'True', '--encoder', 'n3d', '--bitrate', 'script', *_demo_args(tmp_path)])
    samples, idr = read_samples(out / 'interpolation.mp4')
    assert len(samples) == 2 * 2 and idr == [0]
    from next3d_b200 import mp4
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
