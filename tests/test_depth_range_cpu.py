"""CPU: the per-image depth range (N3DRender.depth_range_per_image, n3d_depth_clamp_images, the `depth_range` keyword) is checked
before anything reaches the device, and the sharded drivers' frame split (drivers.shard_plan, FramePack slices) in a gloo world of 2.
The render calls carry ray_end < ray_start, which the library checks after the depth-range flag: a call whose flag passes gets the
ray-setup error, and nothing is launched either way."""
import ctypes as C
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from next3d_b200 import config

ENTRIES = ['n3d_render_rays', 'n3d_render_rays_normals']


def _call(entry, flag, depth_minmax=None):
    from next3d_b200 import _lib, kernels
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, ray_start=2.0, ray_end=1.0)
    planes = torch.zeros(1, 3, 4, 4, 32)
    cam, intr = torch.zeros(1, 16), torch.zeros(1, 9)
    dec = (torch.zeros(64, 32), torch.zeros(64), torch.zeros(33, 64), torch.zeros(33))
    out = torch.zeros(4 * 4 * 32)
    p = kernels._render_full_desc(planes, cam, intr, 4, opts, dec, out, out, out, depth_minmax, None, None, 0, None,
                                  depth_range_per_image=flag)
    if entry == 'n3d_render_rays':
        rc = _lib.lib.n3d_render_rays(C.byref(p), None)
    else:
        rc = _lib.lib.n3d_render_rays_normals(C.byref(p), kernels.ptr(out), kernels.ptr(out), None)
    return rc, _lib.lib.n3d_last_error().decode()


@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('flag', [2, -1, 7])
def test_depth_range_flag_other_than_0_or_1_is_refused(entry, flag):
    rc, msg = _call(entry, flag, torch.zeros(2))
    assert rc == -1 and f'depth_range_per_image = {flag}' in msg, (rc, msg)


@pytest.mark.parametrize('entry', ENTRIES)
def test_per_image_range_needs_depth_minmax(entry):
    rc, msg = _call(entry, 1)
    assert rc == -1 and 'needs depth_minmax' in msg, (rc, msg)


@pytest.mark.parametrize('entry', ENTRIES)
@pytest.mark.parametrize('flag,mm', [(0, None), (0, 2), (1, 2)])
def test_depth_range_flags_0_and_1_pass_the_check(entry, flag, mm):
    rc, msg = _call(entry, flag, None if mm is None else torch.zeros(mm))
    assert rc == -1 and 'bad ray setup' in msg, (rc, msg)


def test_depth_clamp_images_refuses_bad_arguments():
    from next3d_b200 import _lib, kernels
    depth, mm = torch.zeros(6), torch.zeros(4)
    fn = _lib.lib.n3d_depth_clamp_images
    for args in [(None, 2, 3, kernels.ptr(mm)), (kernels.ptr(depth), 2, 3, None), (kernels.ptr(depth), -1, 3, kernels.ptr(mm)),
                 (kernels.ptr(depth), 2, -3, kernels.ptr(mm))]:
        assert fn(*args, None) == -1, args
        assert 'n3d_depth_clamp_images: bad args' in _lib.lib.n3d_last_error().decode()
    assert fn(kernels.ptr(depth), 0, 3, kernels.ptr(mm), None) == 0            # nothing to clamp: no launch
    with pytest.raises(RuntimeError, match=r'depth_minmax must be \[2, 2\]'):
        kernels.depth_clamp_images(depth.view(2, 3), torch.zeros(2))


def test_depth_range_keyword_is_checked():
    from next3d_b200 import engine
    assert engine._depth_range('batch') == 'batch' and engine._depth_range('image') == 'image'
    with pytest.raises(ValueError, match='depth_range'):
        engine._depth_range('frame')


def test_frame_pack_slices(tmp_path):
    from next3d_b200 import inputs
    rng = np.random.RandomState(0)
    verts, cams = rng.randn(7, 5, 3).astype(np.float32), rng.randn(7, 25).astype(np.float32)
    path = str(tmp_path / 'clip.n3dpack')
    inputs.write_frame_pack(path, verts, cams, ids=[f'{k:04d}' for k in range(7)])
    pack = inputs.FramePack(path, pin=False)
    part = pack[2:5]
    assert len(part) == 3 and part.ids == ['0002', '0003', '0004'] and np.array_equal(part.cams, cams[2:5])
    assert [t.shape for t in part] == [(1, 5, 3)] * 3
    assert all(np.array_equal(t[0].numpy(), verts[2 + i]) for i, t in enumerate(part))
    assert len(pack[6:9]) == 1 and len(pack[4:4]) == 0 and len(pack) == 7
    with pytest.raises(TypeError):
        pack[0:6:2]


def test_shard_plan_world_1():
    from next3d_b200 import drivers
    p = drivers.shard_plan(30, 8)
    assert (p.rank, p.world, p.batch, p.steps) == (0, 1, 6, 5)                  # 5 batches of 6, not 4 of 8
    assert p.frames(0) == list(range(6)) and p.frames(4) == list(range(24, 30))
    p = drivers.shard_plan(5, 2)
    assert p.batch == 1 and p.steps == 5
    p = drivers.shard_plan(7, 4)
    assert (p.batch, p.steps) == (4, 2) and p.frames(1) == [4, 5, 6, 6]          # the tail repeats the last frame
    assert [p.valid(k) for k in range(2)] == [4, 3] and [p.step_id(k) for k in range(2)] == [0, 1]
    p = drivers.local_plan(7, 3)                                                # the single-process run: exactly `batch` per step
    assert (p.rank, p.world, p.batch, p.steps) == (0, 1, 3, 3) and p.frames(2) == [6, 6, 6] and p.valid(2) == 1
    assert drivers.local_plan(0, 3).steps == 0


def _worker(rank, world, port, F, batch, pack, q):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from next3d_b200 import distributed as D, drivers, inputs
    r, w, _ = D.init_from_env('gloo')
    p = drivers.shard_plan(F, batch)
    steps = [torch.zeros(1, dtype=torch.int64) for _ in range(w)]
    torch.distributed.all_gather(steps, torch.tensor([p.steps]))
    frames = [p.frames(k) for k in range(p.steps)]
    a, b = p.spans[r]
    first = frames[0][0] if frames else a
    part = inputs.FramePack(pack, pin=False)[first:max(b, first + 1)]
    read = [int(t[0, 0, 0].item()) for t in part]                               # vertex 0 of frame f holds f
    q.put((r, p.spans, p.batch, [int(s.item()) for s in steps], frames, read))
    torch.distributed.destroy_process_group()


@pytest.mark.parametrize('F,batch', [(8, 4), (7, 3), (1, 2)])
def test_shard_plan_and_pack_slices_two_ranks_gloo(tmp_path, F, batch):
    """Every rank derives the same split and the same step count, renders exactly its own frames (padding repeats its last one; a
    rank without frames repeats the previous rank's last) and reads only those frames from the pack."""
    from next3d_b200 import inputs
    verts = np.zeros((F, 4, 3), np.float32)
    verts[:, 0, 0] = np.arange(F)
    pack = str(tmp_path / 'clip.n3dpack')
    inputs.write_frame_pack(pack, verts, np.zeros((F, 25), np.float32))
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, F, batch, pack, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict((x[0], x[1:]) for x in (q.get(timeout=120), q.get(timeout=120)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    spans = res[0][0]
    assert spans == res[1][0] and spans[0][0] == 0 and spans[0][1] == spans[1][0] and spans[1][1] == F
    assert res[0][1] == res[1][1] and res[0][2] == res[1][2] and res[0][2][0] == res[0][2][1]
    covered = []
    for r in (0, 1):
        (a, b), frames, read = res[r][0][r], res[r][3], res[r][4]
        flat = [i for f in frames for i in f]
        assert len(frames) == res[r][2][0] and all(len(f) == res[r][1] for f in frames)
        if b > a:
            assert sorted(set(flat)) == list(range(a, b)) and read == list(range(a, b))
            covered += list(range(a, b))
        else:
            assert set(flat) == {a - 1} and read == [a - 1]
    assert covered == list(range(F))
