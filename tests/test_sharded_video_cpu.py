"""CPU: the sharded video path of the CLI without a GPU.  Each rank's schedule (drivers.call_plan, gop_span, head_plan) makes
exactly the single-process run's calls for its own outputs -- same item ids, tail padding and sampler seed -- and the ranks' own
frames, in rank order, are the single-process frames, at world sizes 1 to 5 (the drivers run on the recording stub generator of
tests/test_driver_calls_cpu.py, one rank after another in this process).  Under gloo with spawned ranks, write_video_sharded
muxes fake coded samples into the MP4 that mp4.write_mp4 writes for their concatenation, and a rank that fails makes every rank
raise an error naming it, without a file and without a hang.  And the CLI refuses its torchrun and --gop misuses before loading
the network."""
import os
import socket
import sys

import pytest
import torch
import torch.multiprocessing as mp

from next3d_b200 import distributed as D, drivers, mp4
from tests.test_driver_calls_cpu import _StubG, _drive_root, _interp_on_host
from tests.test_legacy_cpu import _demo_args

WORLDS = (1, 2, 3, 4, 5)


# ------------------------------------------------------------------------------------------------ schedule maths
@pytest.mark.parametrize('n,batch', [(1, 4), (7, 3), (24, 8), (25, 8), (60, 6)])
def test_call_plans_reproduce_the_single_process_calls(n, batch):
    """Every own range, cut anywhere: the rank's calls are the local_plan calls overlapping it, with their ids and step ids, and
    the kept outputs are exactly the range."""
    local = drivers.local_plan(n, batch)
    for a in range(n + 1):
        for b in range(a, n + 1):
            plan = drivers.call_plan(n, batch, (a, b))
            want = [k for k in range(local.steps) if k * batch < b and (k + 1) * batch > a] if a < b else []
            assert [plan.step_id(k) for k in range(plan.steps)] == want
            kept = []
            for k in range(plan.steps):
                assert plan.frames(k) == local.frames(plan.step_id(k))
                lo, hi = plan.keep(k)
                kept += plan.frames(k)[lo:hi]
            assert kept == list(range(a, b))


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('F,gop', [(1, 60), (8, 3), (16, 4), (240, 60), (240, 30), (59, 7)])
def test_gop_spans_own_every_frame_once(F, gop, world):
    spans = [drivers.gop_span(F, gop, r, world) for r in range(world)]
    assert spans[0][0] == 0 and spans[-1][1] == F
    for (a, b), (c, _) in zip(spans, spans[1:]):
        assert b == c
    for a, b in spans:
        assert a <= b and (a == b or a % gop == 0) and (b % gop == 0 or b == F)
    owners = sum(b > a for a, b in spans)
    assert owners == min(world, -(-F // gop))                     # a rank may own nothing only when there are fewer GOPs


@pytest.mark.parametrize('world', WORLDS)
@pytest.mark.parametrize('S,batch', [(1, 9), (5, 9), (7, 6), (10, 3), (4, 1)])
def test_head_plans_are_whole_calls(S, batch, world):
    B = max(1, batch // 3)
    plans = [drivers.head_plan(S, B, r, world) for r in range(world)]
    assert plans[0].own[0] == 0 and plans[-1].own[1] == S
    for p, q in zip(plans, plans[1:]):
        assert p.own[1] == q.own[0]
    for p in plans:
        (a, b), call = p.own, p.first
        assert (a == b or a == B * call) and (b % B == 0 or b == S)
        assert all(p.keep(k)[0] == 0 for k in range(p.steps))               # every call starts at one of the rank's own heads


# ------------------------------------------------------------------------------------------------ the drivers, rank by rank
def _run(make, world):
    """[(span, frames [n, H, W, 3] uint8, calls)] of every rank of `world`: make(G, rank, world) -> drivers.*_video_shard(...)."""
    out = []
    for r in range(world):
        G = make.G()
        span, frames = make(G, r, world)
        f = [t for t in frames]
        out.append((span, torch.cat(f) if f else None, G.calls))
    return out


def _check_ranks(make, world, F, gop, single_frames, single_calls):
    runs = _run(make, world)
    assert [s for s, _, _ in runs] == [drivers.gop_span(F, gop, r, world) for r in range(world)]
    got = torch.cat([f for _, f, _ in runs if f is not None])
    assert torch.equal(got, single_frames)
    n_render = [c for c in single_calls if c[0] != 'grid']
    for (a, b), f, calls in runs:
        assert (f is None and a == b and calls == []) or f.shape[0] == b - a
        if calls:                                                     # a contiguous run of the single-process calls
            render = [c for c in calls if not c[2]]                  # not the backbone-caching calls
            want = [c for c in n_render if not c[2]]
            i = want.index(render[0])
            assert render == want[i:i + len(render)], (a, b)
    return runs


class _Maker:
    def __init__(self, fn, res=4):
        self.fn, self.res = fn, res

    def G(self):
        return _StubG(self.res)

    def __call__(self, G, rank, world):
        return self.fn(G, rank, world)


@pytest.mark.parametrize('world', WORLDS)
def test_grid_video_shards_are_the_single_process_video(monkeypatch, world):
    """2x2 grid (items are cells, 4 per frame) of 2 keyframes x 5 frames in calls of 6 images: calls straddle frames and ranks;
    gop 3 gives 4 GOPs, so world 5 leaves a rank without frames."""
    monkeypatch.setattr(drivers, 'interpolate_ws_device', _interp_on_host)
    torch.manual_seed(0)
    ws = torch.randn(2, 2, 2, 3, 512)
    v = torch.randn(1, 11, 3)
    G1 = _StubG()
    single = torch.stack([torch.as_tensor(f) for f in drivers.render_grid_frames(G1, ws, v, 5, batch=6, seed=7)])
    make = _Maker(lambda G, r, w: drivers.grid_video_shard(G, ws, v, 5, 3, r, w, batch=6, seed=7))
    runs = _check_ranks(make, world, 10, 3, single, G1.calls)
    if world == 5:
        assert runs[-1][0] == (10, 10) and runs[-1][2] == []


@pytest.mark.parametrize('world', WORLDS)
def test_orbit_video_shards_are_the_single_process_video(world):
    torch.manual_seed(1)
    ws, v = torch.randn(1, 3, 512), torch.randn(1, 11, 3)
    cams = drivers.orbit_camera_params(11, torch.tensor([0, 0, 0.2]), 2.7)
    G1 = _StubG()
    single = torch.stack([torch.as_tensor(f) for f in drivers.render_orbit(G1, ws, cams, v, batch=4, seed=3)])
    make = _Maker(lambda G, r, w: drivers.orbit_video_shard(G, ws, cams, v, 2, r, w, batch=4, seed=3))
    _check_ranks(make, world, 11, 2, single, G1.calls)


@pytest.mark.parametrize('world', WORLDS)
def test_reenact_grid_video_shards_are_the_single_process_video(tmp_path, world):
    """Items are driving frames of S = 2 heads (calls of 3 frames at batch 6); every rank caches the backbones on its first call."""
    root = _drive_root(str(tmp_path), n=9)                                 # frames 1 .. 7
    torch.manual_seed(2)
    ws = torch.randn(2, 3, 512)
    G1 = _StubG(512)
    single = torch.stack([torch.as_tensor(f) for f in drivers.reenact_grid_frames(G1, ws, root, 10, (3, 1), batch=6, seed=5,
                                                                                    workers=1)])
    make = _Maker(lambda G, r, w: drivers.reenact_grid_video_shard(G, ws, root, 10, (3, 1), 2, r, w, batch=6, seed=5, workers=1), 512)
    runs = _check_ranks(make, world, 7, 2, single, G1.calls)
    for (a, b), _, calls in runs:
        if a < b:
            assert calls[0][2] and not calls[0][3] and all(c[3] for c in calls[1:])          # cache once, then reuse


@pytest.mark.parametrize('world', WORLDS)
def test_sheet_head_plans_are_the_single_process_sheets(world):
    """render_sample_sheets over each rank's head_plan: the single process's seeds, sheets and calls."""
    torch.manual_seed(3)
    ws, v = torch.randn(7, drivers.NUM_WS, 512), torch.randn(1, 11, 3)
    G1 = _StubG()
    single = [s for _, s, _ in drivers.render_sample_sheets(G1, ws, v, batch=6, seed=4)]
    ids, sheets, calls = [], [], []
    for r in range(world):
        G = _StubG()
        got = list(drivers.render_sample_sheets(G, ws, v, batch=6, seed=4, plan=drivers.head_plan(7, 2, r, world)))
        ids += [i for i, _, _ in got]
        sheets += [s for _, s, _ in got]
        calls += G.calls
    assert ids == list(range(7))
    assert len(sheets) == len(single) and all((x == y).all() for x, y in zip(sheets, single))
    assert calls == G1.calls


# ------------------------------------------------------------------------------------------------ gather, mux and failure under gloo
class _FakeEncoder:
    """Stands in for video.H264Encoder: sample i of a frame is its bytes' sum and index, IDR every gop frames of the video."""
    fps = 60

    def __init__(self, width, height, first, gop):
        self.width, self.height, self.n, self.gop = width, height, first, gop
        self.sps, self.pps = b'\x67\x42\xc0\x1e', b'\x68\xce'

    def write(self, frames):
        out = []
        for f in frames:
            out.append((fake_sample(self.n, f), self.n % self.gop == 0))
            self.n += 1
        return out

    def flush(self):
        return []


def fake_sample(i, frame):
    return int(i).to_bytes(4, 'big') + int(frame.sum()).to_bytes(8, 'big') * (1 + i % 3)


def _frame(i):
    return torch.full((1, 4, 6, 3), i % 251, dtype=torch.uint8)


def _port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _mux_worker(rank, world, port, path, F, gop, fail, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    D.init_from_env('gloo')
    try:
        def shard():
            a, b = drivers.gop_span(F, gop, rank, world)

            def frames():
                for i in range(a, b):
                    if rank == fail and i == a + 1:
                        raise ValueError('the stub renderer failed')
                    yield _frame(i)
            return (a, b), frames()
        try:
            drivers.write_video_sharded(path, shard, lambda w, h, first: _FakeEncoder(w, h, first, gop))
            q.put((rank, None))
        except D.RankError as e:
            q.put((rank, (e.rank, str(e))))
    finally:
        torch.distributed.destroy_process_group()


def _spawn(world, *args):
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _port()
    procs = [ctx.Process(target=_mux_worker, args=(r, world, port, *args, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=120) for _ in range(world))
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
    assert [p.exitcode for p in procs] == [0] * world
    return got


@pytest.mark.parametrize('world,F,gop', [(2, 10, 3), (3, 7, 1), (3, 4, 2)])           # (3, 4, 2): rank 2 owns nothing
def test_gather_and_mux_equal_write_mp4(tmp_path, world, F, gop):
    path = str(tmp_path / 'v.mp4')
    assert set(_spawn(world, path, F, gop, -1).values()) == {None}
    want = str(tmp_path / 'want.mp4')
    enc = _FakeEncoder(6, 4, 0, gop)
    samples = [enc.write(_frame(i))[0] for i in range(F)]
    mp4.write_mp4(want, 6, 4, 60, enc.sps, enc.pps, [s for s, _ in samples], [i for i, (_, k) in enumerate(samples) if k])
    data = open(path, 'rb').read()
    assert data == open(want, 'rb').read()
    assert [k for k, _, _ in mp4.parse_boxes(data)] == [b'ftyp', b'mdat', b'moov']


def test_a_failing_rank_stops_every_rank(tmp_path):
    """Rank 1 raises after its first frame: every rank raises RankError naming rank 1 and its message, no file is written, and
    the processes end (the queue read has a timeout)."""
    path = tmp_path / 'v.mp4'
    got = _spawn(3, str(path), 12, 2, 1)
    for r in range(3):
        assert got[r] is not None and got[r][0] == 1 and 'rank 1' in got[r][1] and 'the stub renderer failed' in got[r][1], got
    assert not path.exists()


def test_one_process_raises_the_error_itself(tmp_path):
    def shard():
        def frames():
            yield _frame(0)
            raise ValueError('stub failure')
        return (0, 2), frames()
    with pytest.raises(ValueError, match='stub failure'):
        drivers.write_video_sharded(str(tmp_path / 'v.mp4'), shard, lambda w, h, first: _FakeEncoder(w, h, first, 2))
    assert not (tmp_path / 'v.mp4').exists()


# ------------------------------------------------------------------------------------------------ CLI refusals
@pytest.mark.parametrize('world', ['1', '2'])
@pytest.mark.parametrize('cmd,extra,match', [
    ('gen_videos', ['--encoder', 'imageio', '--gop', '30'], 'gop'),
    ('gen_videos', ['--encoder', 'n3d', '--gop', '0'], 'gop 0'),
    ('reenact', ['--encoder', 'n3d', '--gop', '-3'], 'gop -3'),
    ('reenact', ['--gop', '30'], 'gop'),
])
def test_cli_refuses_gop_misuse(tmp_path, monkeypatch, world, cmd, extra, match):
    _refuses(tmp_path, monkeypatch, world, cmd, extra, match)


@pytest.mark.parametrize('cmd', ['gen_videos', 'reenact'])
def test_cli_refuses_imageio_under_torchrun(tmp_path, monkeypatch, cmd):
    _refuses(tmp_path, monkeypatch, '2', cmd, ['--encoder', 'imageio'], 'torchrun')
    _refuses(tmp_path, monkeypatch, '2', cmd, [], 'torchrun')                             # imageio is the default


def _refuses(tmp_path, monkeypatch, world, cmd, extra, match):
    """The refusal comes before the process group and the network: the --network file does not exist, and no MASTER_ADDR is set."""
    from next3d_b200.__main__ import main
    monkeypatch.setitem(sys.modules, 'imageio', None)
    for k in ('MASTER_ADDR', 'MASTER_PORT'):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv('WORLD_SIZE', world)
    monkeypatch.setenv('RANK', '0')
    argv = [cmd, '--seeds', '0', '--outdir', str(tmp_path / 'o'), '--lms_cond', 'True', '--network', str(tmp_path / 'missing.pkl'),
            *extra]
    argv += ['--drive_root', 'd'] if cmd == 'reenact' else _demo_args(tmp_path)
    with pytest.raises(SystemExit, match=match):
        main(argv)
    assert not torch.distributed.is_initialized()
