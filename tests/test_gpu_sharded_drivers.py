"""GPU: depth frames of the batched drivers (one depth range per frame, as the scripts' one frame per call) and the sharded drivers
(reenact_frames_sharded, render_orbit_sharded) against the single-GPU ones; a spawned NCCL world of 2 when two GPUs are visible."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _generator():
    from next3d_b200 import config, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    cfg = config.tiny_config(512)
    return cfg, TriPlaneGenerator.from_config(cfg, weights.make_state_dict(cfg, seed=9), device=DEV)


@pytest.fixture(scope='module')
def tiny():
    return _generator()


def _head(cfg, G, seed=3, dev=DEV):
    from next3d_b200 import weights
    z, cc, c, v = weights.demo_inputs(cfg, 1, seed=seed)
    return G.mapping(z.to(dev), cc.to(dev), truncation_psi=0.7, truncation_cutoff=14), c, v


def _noise(G, F, seed):
    R = G.neural_rendering_resolution
    D, Df = G.rendering_kwargs['depth_resolution'], G.rendering_kwargs['depth_resolution_importance']
    g = torch.Generator().manual_seed(seed)
    return torch.rand(F, R * R, D, 1, generator=g).to(DEV), torch.rand(F, R * R, Df, generator=g).to(DEV)


def _drive_dir(root, v, c, n):
    """A driving directory of n labels (dataset.json + NNNN.png / .obj / _kpt2d.txt): n - 2 frames."""
    rng = np.random.RandomState(1)
    labels = []
    for k in range(n):
        name = f'{k:04d}'
        (root / f'{name}.png').write_bytes(b'')
        vk = v[0].numpy() + rng.randn(*v[0].shape).astype(np.float32) * 1e-4
        (root / f'{name}.obj').write_text(''.join(f'v {float(a)!r} {float(b)!r} {float(c_)!r}\n' for a, b, c_ in vk[:5023]))
        (root / f'{name}_kpt2d.txt').write_text('\n'.join(f'{float(a)!r} {float(b)!r} {float(c_)!r}' for a, b, c_ in vk[5023:]) + '\n')
        cam = c[0].numpy().astype(np.float64)
        cam[3] += 0.01 * k
        labels.append([f'{name}.png', cam.tolist()])
    (root / 'dataset.json').write_text(json.dumps({'labels': labels}))
    return str(root)


def _per_frame(G, ws, cams, verts, noise, f, mode):
    from next3d_b200 import drivers
    u_c, u_f = noise
    out = G.synthesis(ws, cams[f:f + 1].to(DEV), verts.to(DEV), noise_mode='const', sampler_noise=(u_c[f:f + 1], u_f[f]))
    return drivers._frames_u8(out, mode)[0].cpu().numpy()


def _assert_frames(got, want):
    torch.cuda.synchronize()                       # the sharded drivers fill their host tensor in stream order
    assert len(got) == len(want)
    for f, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a), np.asarray(b)
        assert a.shape == b.shape and np.array_equal(a, b), f'frame {f}: max |diff| {np.abs(a.astype(int) - b.astype(int)).max()}'


# ------------------------------------------------------------------------------------------------ depth frames
def test_render_frames_and_orbit_depth_equal_per_frame_calls(tiny):
    """image_mode 'image_depth' in batches of 2 (last one padded) == one synthesis call per frame, pixel for pixel."""
    from next3d_b200 import drivers
    cfg, G = tiny
    ws, _, v = _head(cfg, G)
    F = 5
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    noise = _noise(G, F, 12)
    want = [_per_frame(G, ws, cams, v, noise, f, 'image_depth') for f in range(F)]
    wsf = ws.cpu().expand(F, -1, -1)
    _assert_frames(list(drivers.render_frames(G, wsf, cams, v, batch=2, image_mode='image_depth', sampler_noise=noise)), want)
    _assert_frames(list(drivers.render_orbit(G, ws, cams, v, batch=2, image_mode='image_depth', sampler_noise=noise)), want)


def test_reenact_frames_depth_equal_per_frame_calls(tiny, tmp_path):
    from next3d_b200 import drivers, inputs
    cfg, G = tiny
    ws, c, v = _head(cfg, G)
    root = _drive_dir(tmp_path, v, c, 7)
    sch = drivers.reenact_schedule(root, 100)
    F = len(sch['ks'])
    noise = _noise(G, F, 4)
    want = []
    for f in range(F):
        vf = inputs.load_frame(sch['obj_paths'][f], sch['lms_paths'][f])
        want.append(_per_frame(G, ws, sch['cams'], vf, noise, f, 'image_depth'))
    _assert_frames(list(drivers.reenact_frames(G, ws, root, 100, batch=2, sampler_noise=noise, image_mode='image_depth')), want)


# ------------------------------------------------------------------------------------------------ sharded drivers, world size 1
@pytest.mark.parametrize('image_mode', ['image', 'image_depth'])
def test_reenact_frames_sharded_equals_reenact_frames(tiny, tmp_path, image_mode):
    """From a directory and from a pack; the launch counts show the backbones are skipped after the first batch."""
    from next3d_b200 import drivers, inputs
    from tests.test_gpu_views import _backbone_launches
    cfg, G = tiny
    ws, c, v = _head(cfg, G)
    root = _drive_dir(tmp_path, v, c, 8)
    sch = drivers.reenact_schedule(root, 100)
    F = len(sch['ks'])
    assert F == 6
    noise = _noise(G, F, 5)
    want = list(drivers.reenact_frames(G, ws, root, 100, batch=2, sampler_noise=noise, image_mode=image_mode))
    launches, synthesis = [], G.synthesis

    def counting(*a, **kw):
        out = synthesis(*a, **kw)
        launches.append(G._get_engine().launches)
        return out
    G.synthesis = counting
    try:
        got = drivers.reenact_frames_sharded(G, ws, root, 100, batch=2, sampler_noise=noise, image_mode=image_mode)
    finally:
        del G.synthesis
    res = cfg.img_resolution if image_mode == 'image' else G.neural_rendering_resolution
    assert got.shape == (F, res, res, 3) and got.dtype == torch.uint8
    _assert_frames(list(got.numpy()), want)
    bb = _backbone_launches(G, cfg)
    assert len(launches) == 3 and launches[1:] == [launches[0] - bb] * 2, (launches, bb)
    pack = str(tmp_path / 'clip.n3dpack')
    inputs.write_frame_pack(pack, np.stack([inputs.load_frame(o, l)[0].numpy() for o, l in zip(sch['obj_paths'], sch['lms_paths'])]),
                            sch['cams'].numpy(), ids=sch['ids'])
    _assert_frames(list(drivers.reenact_frames_sharded(G, ws, pack, 100, batch=2, sampler_noise=noise, image_mode=image_mode).numpy()),
                   want)


@pytest.mark.parametrize('image_mode', ['image', 'image_depth'])
def test_render_orbit_sharded_equals_render_orbit(tiny, image_mode):
    from next3d_b200 import drivers
    cfg, G = tiny
    ws, _, v = _head(cfg, G)
    F = 6
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    noise = _noise(G, F, 6)
    want = list(drivers.render_orbit(G, ws, cams, v, batch=3, image_mode=image_mode, sampler_noise=noise))
    got = drivers.render_orbit_sharded(G, ws, cams, v, batch=3, image_mode=image_mode, sampler_noise=noise)
    _assert_frames(list(got.numpy()), want)
    seeded = drivers.render_orbit_sharded(G, ws, cams, v, batch=3, seed=4)           # in-kernel RNG: right shape, frames differ
    assert seeded.shape == (F, cfg.img_resolution, cfg.img_resolution, 3) and not torch.equal(seeded[0], seeded[2])


def test_render_frames_sharded_global_noise_rows(tiny):
    """sampler_noise rows are global frame ids: render_frames_sharded == render_frames with the same rows."""
    from next3d_b200 import drivers
    cfg, G = tiny
    ws, _, v = _head(cfg, G)
    F = 4
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    noise = _noise(G, F, 7)
    wsf = ws.cpu().expand(F, -1, -1)
    want = list(drivers.render_frames(G, wsf, cams, v, batch=2, sampler_noise=noise))
    _assert_frames(list(drivers.render_frames_sharded(G, wsf, cams, v, batch=2, sampler_noise=noise).numpy()), want)


# ------------------------------------------------------------------------------------------------ NCCL world of 2
def _rank(rank, world, port, pack, cams_path, noise_path, out_dir):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    from next3d_b200 import distributed as D, drivers
    r, _, local = D.init_from_env('nccl')
    try:
        dev = f'cuda:{local}'
        torch.cuda.set_device(dev)
        cfg, G = _generator()
        G = G.to(dev)
        ws, _, v = _head(cfg, G, dev=dev)
        noise = tuple(t.to(dev) for t in torch.load(noise_path))
        cams = torch.load(cams_path)
        reen = drivers.reenact_frames_sharded(G, ws, pack, 100, batch=4, sampler_noise=noise, image_mode='image_depth')
        orbit = drivers.render_orbit_sharded(G, ws, cams, v, batch=4, sampler_noise=noise)
        torch.cuda.synchronize()
        if r == 0:
            np.save(os.path.join(out_dir, 'reenact.npy'), reen.numpy())
            np.save(os.path.join(out_dir, 'orbit.npy'), orbit.numpy())
    finally:
        torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs two GPUs')
def test_sharded_drivers_world_of_two_equal_world_of_one(tiny, tmp_path):
    """8 frames over 2 ranks (batches of 4 on both world sizes): the gathered frames equal world size 1's."""
    from next3d_b200 import drivers, inputs
    cfg, G = tiny
    ws, c, v = _head(cfg, G)
    F = 8
    rng = np.random.RandomState(3)
    verts = np.stack([v[0].numpy() + rng.randn(*v[0].shape).astype(np.float32) * 1e-4 for _ in range(F)])
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    pack = str(tmp_path / 'clip.n3dpack')
    inputs.write_frame_pack(pack, verts, cams.numpy())
    noise = _noise(G, F, 8)
    torch.save(tuple(t.cpu() for t in noise), str(tmp_path / 'noise.pt'))
    torch.save(cams, str(tmp_path / 'cams.pt'))
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    procs = [ctx.Process(target=_rank, args=(r, 2, port, pack, str(tmp_path / 'cams.pt'), str(tmp_path / 'noise.pt'), str(tmp_path)))
             for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=600)
    codes = [p.exitcode for p in procs]
    for p in procs:
        if p.is_alive():
            p.kill()
            p.join()
    assert codes == [0, 0], codes
    want_reen = drivers.reenact_frames_sharded(G, ws, pack, 100, batch=4, sampler_noise=noise, image_mode='image_depth')
    want_orbit = drivers.render_orbit_sharded(G, ws, cams, v, batch=4, sampler_noise=noise)
    _assert_frames(list(np.load(str(tmp_path / 'reenact.npy'))), list(want_reen.numpy()))
    _assert_frames(list(np.load(str(tmp_path / 'orbit.npy'))), list(want_orbit.numpy()))
