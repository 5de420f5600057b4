"""GPU: the CLI's video path split over ranks.  H264Encoder segments that start at a multiple of the GOP (`first_frame`) concatenate
to the constant-QP stream of one encoder, and a segment of either stream is the oracle started at its first frame; two
rate-controlled halves of a rendered orbit hit their target.  `python -m next3d_b200` under a torchrun-style environment at world
2 and 3 (gloo, every rank on the same GPU, or on separate GPUs when two are visible) writes byte for byte the files of the
one-process run of the same command -- PNG and MRC sheets, grid, orbit and depth videos, reenactment -- also when a rank owns no
frames; with --bitrate the file decodes to every frame with IDR frames exactly at the GOP starts.  And the one-process
--encoder n3d file is H264Writer's over the driver's frames."""
import os
import socket
import subprocess
import sys

import pytest
import torch

from tests import h264_oracle as O
from tests.test_gpu_h264 import oracle_encode, read_samples
from tests.test_legacy_cpu import _demo_args, generator_fields, persistence_pickle

pytestmark = pytest.mark.gpu
DEV = 'cuda'
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _encode(frames, W, H, gop, first=0, **stream):
    from next3d_b200.video import H264Encoder
    enc = H264Encoder(W, H, 30, gop=gop, batch=2, first_frame=first, **stream)
    out = []
    for f in frames:
        out += enc.write(torch.as_tensor(f).to(DEV))
    return out + enc.flush()


@pytest.mark.parametrize('gop,cuts', [(3, [3]), (3, [3, 6]), (1, [1, 2, 5]), (4, [8])])
def test_cq_segments_concatenate_to_the_whole_stream(gop, cuts):
    frames = O.sequence('translate', 48, 32, 9)
    whole = _encode(frames, 48, 32, gop, qp=18)
    bounds = [0, *cuts, len(frames)]
    parts = sum((_encode(frames[a:b], 48, 32, gop, a, qp=18) for a, b in zip(bounds, bounds[1:])), [])
    assert [k for _, k in parts] == [i % gop == 0 for i in range(len(frames))]
    assert parts == whole
    samples, idr, _ = oracle_encode(frames, 48, 32, gop, qp=18)
    assert [s for s, _ in whole] == samples and idr == [i for i, (_, k) in enumerate(whole) if k]


def test_first_frame_must_start_a_gop():
    from next3d_b200.video import H264Encoder
    for first in (1, 5, -3):
        with pytest.raises(ValueError, match='first_frame'):
            H264Encoder(48, 32, 30, gop=3, first_frame=first)


def _oracle_from(enc, first):
    """The oracle `enc` started at frame `first` of a longer video: its frame counter sets frame_num and idr_pic_id, as
    H264Encoder's first_frame does; the rate controller of an RcEncoder starts afresh, as each segment's does."""
    enc.n = first
    return enc


@pytest.mark.parametrize('first', [0, 3, 6])
@pytest.mark.parametrize('stream', ['cq', 'rc'])
def test_segment_equals_the_oracle(stream, first):
    frames = O.frames('pan', 48, 32, 9)[first:]
    if stream == 'cq':
        got = _encode(frames, 48, 32, 3, first, qp=18)
        enc = _oracle_from(O.Encoder(48, 32, 18, 3), first)
    else:
        got = _encode(frames, 48, 32, 3, first, bitrate=48 * 32 * 30)
        enc = _oracle_from(O.RcEncoder(48, 32, 48 * 32 * 30, (30, 1), 3), first)
    assert got == [enc.encode(f) for f in frames]


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config
    from tests.test_gpu_views import _generator
    cfg = config.tiny_config(512)
    _, G = _generator(cfg, 6)
    return cfg, G


def test_two_rc_segments_hit_their_target(tiny):
    """A 240-frame rendered orbit at 512x512, 60 frames/s, encoded as two rate-controlled halves of two GOPs each: within 10 % of
    targets between the pinned-QP-40 and QP-10 rates, as one encoder is."""
    from next3d_b200 import drivers, weights
    from next3d_b200.video import H264Encoder
    cfg, G = tiny
    *_, v = weights.demo_inputs(cfg, 1, seed=0, device=DEV)
    rk = G.rendering_kwargs
    ws = drivers.grid_keyframes(G, [3], (1, 1), truncation_psi=0.7)[0, 0]
    cams = drivers.orbit_camera_params(240, torch.tensor(rk['avg_camera_pivot']), rk['avg_camera_radius'])
    frames = torch.stack([torch.as_tensor(f) for f in drivers.render_orbit(G, ws[:1], cams, v, seed=0)]).to(DEV)

    def rate(bitrate, qp_range, cuts=(0, 120, 240)):
        n = 0
        for a, b in zip(cuts, cuts[1:]):
            enc = H264Encoder(512, 512, 60, gop=60, batch=16, bitrate=bitrate, qp_range=qp_range, first_frame=a)
            n += sum(len(s) for s, _ in enc.write(frames[a:b]) + enc.flush())
        return 8 * n * 60 / 240
    lo, hi = rate(10 ** 6, (40, 40)), rate(10 ** 6, (10, 10))
    for f in (0.25, 0.75):
        t = int(lo * (hi / lo) ** f)
        got = rate(t, (0, 51))
        print(f'two halves: target {t} bits/s, got {got:.0f} ({got / t:.3f}x)')
        assert abs(got - t) <= 0.1 * t, (t, got)


# ------------------------------------------------------------------------------------------------ the CLI at world 1, 2 and 3
@pytest.fixture(scope='module')
def inputs(tmp_path_factory):
    """(network pickle, demo mesh arguments, driving directory) of the tiny generator."""
    from next3d_b200 import config, weights
    from tests.test_gpu_legacy import _drive_root, _mask
    d = tmp_path_factory.mktemp('inputs')
    cfg = config.tiny_config(512)
    net = d / 'tiny.pkl'
    net.write_bytes(persistence_pickle(cfg, weights.make_state_dict(cfg, seed=9), generator_fields(cfg, _mask(10))))
    demo = _demo_args(d)
    return str(net), demo, _drive_root(d / 'drive', demo, n=7)


def _port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _cli(argv, world, devices=False):
    """Run `python -m next3d_b200 argv` as `world` ranks in a torchrun environment (world 1: in this process, as a user runs
    it without torchrun); -> the ranks' (exit code, stderr)."""
    if world == 1:
        from next3d_b200.__main__ import main
        main(argv)
        return [(0, '')]
    port = _port()
    procs = []
    for r in range(world):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE=str(world), LOCAL_RANK=str(r if devices else 0), LOCAL_WORLD_SIZE=str(world),
                   MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), PYTHONPATH=ROOT)
        procs.append(subprocess.Popen([sys.executable, '-m', 'next3d_b200', *argv], cwd=ROOT, env=env, stdout=subprocess.DEVNULL,
                                      stderr=subprocess.PIPE, text=True))
    out = []
    for p in procs:
        try:
            _, err = p.communicate(timeout=900)
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
        out.append((p.returncode, err))
    for r, (code, err) in enumerate(out):
        assert code == 0, f'rank {r}: exit {code}\n{err[-3000:]}'
    return out


def _files(d):
    return {name: open(os.path.join(d, name), 'rb').read() for name in sorted(os.listdir(d))}


def _same_files_at(worlds, make_argv, tmp_path, devices=False):
    """The output directory of make_argv(outdir) at every world size holds the same files, byte for byte."""
    want = None
    for w in (1, *worlds):
        out = str(tmp_path / f'w{w}')
        _cli(make_argv(out), w, devices)
        got = _files(out)
        assert got, f'world {w}: no output'
        if want is None:
            want = got
        else:
            assert sorted(got) == sorted(want), w
            for name in want:
                assert got[name] == want[name], f'world {w}: {name} differs'
    return want


def _videos(net, demo, extra):
    return lambda out: ['gen_videos', '--network', net, '--outdir', out, '--lms_cond', 'True', '--encoder', 'n3d', *demo, *extra]


def test_cli_gen_samples_at_world_2_and_3(inputs, tmp_path):
    """7 seeds in calls of 3 heads: ranks of 2 + 1 calls, and of one call each."""
    net, demo, _ = inputs
    files = _same_files_at((2, 3), lambda out: ['gen_samples', '--network', net, '--seeds', '0-6', '--outdir', out, '--shapes', 'True',
                                                '--shape-res', '32', '--lms_cond', 'True', *demo], tmp_path)
    assert len(files) == 14


GRID = ['--seeds', '0-3', '--grid', '2x1', '--w-frames', '4']                         # 8 frames of 2 cells, calls of 8 images


@pytest.mark.parametrize('gop', [3, 4])                                               # gop 4: two GOPs, rank 2 of 3 owns nothing
def test_cli_grid_video_at_world_2_and_3(inputs, tmp_path, gop):
    net, demo, _ = inputs
    files = _same_files_at((2, 3), _videos(net, demo, [*GRID, '--gop', str(gop)]), tmp_path)
    samples, idr = read_samples(tmp_path / 'w1' / 'interpolation.mp4')
    assert list(files) == ['interpolation.mp4'] and len(samples) == 8 and idr == list(range(0, 8, gop))


def test_cli_orbit_depth_videos_at_world_2_and_3(inputs, tmp_path):
    net, demo, _ = inputs
    files = _same_files_at((2, 3), _videos(net, demo, ['--seeds', '4,5', '--interpolate', 'False', '--w-frames', '5',
                                                       '--sample_mult', '1', '--nrr', '32', '--image_mode', 'image_depth',
                                                       '--gop', '2']), tmp_path)
    assert list(files) == ['4.mp4', '5.mp4']


def test_cli_reenact_at_world_2_and_3(inputs, tmp_path):
    net, _, drive = inputs
    _same_files_at((2, 3), lambda out: ['reenact', '--network', net, '--drive_root', drive, '--grid', '2x1', '--seeds', '6',
                                        '--outdir', out, '--num_frames', '5', '--lms_cond', 'True', '--encoder', 'n3d', '--gop', '2'],
                   tmp_path)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='one GPU visible: the ranks share it in the other tests')
def test_cli_grid_video_on_separate_gpus(inputs, tmp_path):
    net, demo, _ = inputs
    _same_files_at((2,), _videos(net, demo, [*GRID, '--gop', '3']), tmp_path, devices=True)


def test_cli_bitrate_video_at_world_3_decodes(inputs, tmp_path):
    """Each rank's share runs its own rate controller: not the one-process bytes, but a file with every frame and IDR frames at
    multiples of the GOP."""
    net, demo, _ = inputs
    out = str(tmp_path / 'w3')
    _cli(_videos(net, demo, [*GRID, '--gop', '3', '--bitrate', 'script'])(out), 3)
    samples, idr = read_samples(os.path.join(out, 'interpolation.mp4'))
    assert len(samples) == 8 and idr == [0, 3, 6]
    cv2 = pytest.importorskip('cv2')
    cap = cv2.VideoCapture(os.path.join(out, 'interpolation.mp4'), cv2.CAP_FFMPEG)
    n = 0
    while cap.read()[0]:
        n += 1
    assert n == 8


def test_cli_world_1_is_h264writer_over_the_driver_frames(inputs, tmp_path):
    from next3d_b200 import drivers, inputs as I
    from next3d_b200.video import H264Writer
    from tests.test_gpu_legacy import _load
    net, demo, _ = inputs
    out = str(tmp_path / 'out')
    _cli(_videos(net, demo, [*GRID, '--qp', '24'])(out), 1)
    G, v = _load(net), I.load_frame(demo[1], demo[3]).to(DEV)
    for k in ('depth_resolution', 'depth_resolution_importance'):                     # --sample_mult 2
        G.rendering_kwargs[k] *= 2
    ws = drivers.grid_keyframes(G, [0, 1, 2, 3], (2, 1), truncation_psi=1, truncation_cutoff=14)
    frames = list(drivers.render_grid_frames(G, ws, v, 4, seed=0))
    H, W, _ = frames[0].shape
    with H264Writer(str(tmp_path / 'want.mp4'), W, H, 60, qp=24) as w:
        for f in frames:
            w.write(f)
    assert open(os.path.join(out, 'interpolation.mp4'), 'rb').read() == (tmp_path / 'want.mp4').read_bytes()
