"""GPU: the sm_90a H.264 encoder (csrc/h264.cu through next3d_b200.video.H264Writer) writes the same bytes as its numpy
restatement (tests/h264_oracle.py, whose streams FFmpeg decodes to their reconstruction in tests/test_h264_cpu.py) and the same
reconstruction, for the CPU suite's sequences and for rendered frames; argument refusals; and the CLI's --encoder n3d."""
import struct

import numpy as np
import pytest
import torch

from tests import h264_oracle as O
from tests.test_h264_cpu import CASES, FPS, encoded

pytestmark = pytest.mark.gpu
DEV = 'cuda'


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


def gpu_encode(path, frames, W, H, qp, gop, fps=FPS, batch=2):
    """Encode frame by frame from CUDA tensors; returns (samples, IDR indices, recon planes per frame)."""
    from next3d_b200.video import H264Writer
    recon = []
    with H264Writer(str(path), W, H, fps, qp=qp, gop=gop, batch=batch) as w:
        for f in frames:
            w.write(torch.as_tensor(f).to(DEV))
            recon.append(tuple(p.cpu().numpy() for p in w.recon))
    return (*read_samples(path), recon)


def oracle_encode(frames, W, H, qp, gop):
    enc = O.Encoder(W, H, qp, gop)
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
        for p, (a, b) in enumerate(zip(gr[t], wr[t])):
            assert np.array_equal(a, b), f'frame {t}: reconstruction plane {p} differs'
        assert gs[t] == ws[t], f'frame {t}: {len(gs[t])} bytes, the oracle {len(ws[t])}'


@pytest.mark.parametrize('case', CASES, ids=lambda c: '-'.join(map(str, c)))
def test_gpu_stream_equals_oracle(tmp_path, case):
    name, W, H, qp, gop = case
    samples, idr, recon, _ = encoded(*case)
    got = gpu_encode(tmp_path / 'v.mp4', O.sequence(name, W, H), W, H, qp, gop)
    assert_same(got, (samples, [i for i, x in enumerate(idr) if x], recon))


def test_numpy_batches_and_deferred_copies(tmp_path):
    """A numpy batch, copied to the device by the writer, with several frames per host copy: the same bytes."""
    from next3d_b200.video import H264Writer
    frames = O.sequence('translate', 48, 32, 7)
    with H264Writer(str(tmp_path / 'v.mp4'), 48, 32, FPS, qp=18, gop=4, batch=3) as w:
        w.write(np.stack(frames[:5]))
        w.write(frames[5])
        w.write(frames[6])
    samples, idr = read_samples(tmp_path / 'v.mp4')
    want = oracle_encode(frames, 48, 32, 18, 4)
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


@pytest.mark.parametrize('kind', ['orbit', 'grid2x1'])
def test_rendered_frames_equal_oracle(tmp_path, tiny, kind):
    frames = _rendered(tiny, kind)
    assert len(frames) == 16
    H, W, _ = frames[0].shape
    got = gpu_encode(tmp_path / 'v.mp4', frames, W, H, 18, 60, fps=60, batch=8)
    assert_same(got, oracle_encode(frames, W, H, 18, 60))
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


def test_encode_refuses_bad_arguments():
    from next3d_b200 import _lib
    sizes = [_lib.I64() for _ in range(4)]
    assert _lib.lib.n3d_h264_buffer_sizes(32, 32, *[_lib.C.byref(s) for s in sizes]) == 0
    plane, scratch, slices, sample = (torch.zeros(s.value, dtype=torch.uint8, device=DEV) for s in sizes)
    rgb, ref, out_len = torch.zeros(32 * 32 * 3, dtype=torch.uint8, device=DEV), torch.zeros_like(plane), torch.zeros(1, dtype=torch.int64, device=DEV)
    cur = torch.zeros_like(plane)
    stream = torch.cuda.current_stream().cuda_stream
    p = lambda t: t.data_ptr()

    def call(**kw):
        a = dict(rgb=p(rgb), w=32, h=32, qp=18, idr=0, fn=1, idr_id=0, cur=p(cur), ref=p(ref), rec=p(plane), scratch=p(scratch),
                 slices=p(slices), sample=p(sample), n=p(out_len))
        a.update(kw)
        return _lib.lib.n3d_h264_encode(a['rgb'], a['w'], a['h'], a['qp'], a['idr'], a['fn'], a['idr_id'], a['cur'], a['ref'], a['rec'],
                                        a['scratch'], a['slices'], a['sample'], a['n'], stream)
    assert call() == 0
    torch.cuda.synchronize()
    assert out_len.item() > 0
    for kw, msg in [(dict(rgb=None), b'null'), (dict(sample=None), b'null'), (dict(ref=None), b'null ref'), (dict(rec=p(ref)), b'different'),
                    (dict(w=31), b'even'), (dict(h=30, w=33), b'even'), (dict(qp=52), b'qp 52'), (dict(qp=-1), b'qp'),
                    (dict(w=16 * 400, h=16 * 400), b'level 6.2'), (dict(fn=16), b'frame_num')]:
        assert call(**kw) == -1, kw                                     # N3D_ERR_INVALID_ARG
        assert msg in _lib.lib.n3d_last_error(), (kw, _lib.lib.n3d_last_error())
    torch.cuda.synchronize()


def test_cli_gen_videos_n3d_grid(tmp_path, monkeypatch):
    import sys
    from next3d_b200.__main__ import main
    from tests.test_gpu_legacy import _mask
    from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle
    from next3d_b200 import config, weights
    cfg = config.tiny_config(512)
    net = tmp_path / 'tiny.pkl'
    net.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    monkeypatch.setitem(sys.modules, 'imageio', None)                  # the n3d encoder never imports imageio
    out = tmp_path / 'out'
    main(['gen_videos', '--network', str(net), '--seeds', '0-3', '--grid', '2x1', '--w-frames', '2', '--outdir', str(out),
          '--lms_cond', 'True', '--encoder', 'n3d', '--qp', '24', *_demo_args(tmp_path)])
    samples, idr = read_samples(out / 'interpolation.mp4')
    assert len(samples) == 2 * 2 and idr == [0]                            # 2 keyframes per cell x 2 frames each
