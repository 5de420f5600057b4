"""CPU: the host side of the sample-sheet drivers (gen_samples_next3d.py) against the script's own expressions.  The cameras are
compared with the reference's camera_utils, whose results on these inputs are stored in tests/golden/reference_samples.npz
(tests.helpers.ReferenceVectors); the seed latents, the sheet layout, the batching, padding and sampler-noise rows of
render_sample_sheets (with a stub generator), the argument checks, and the sharded twin gathering 512 x 1536 sheets over two ranks
under gloo."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from next3d_b200 import drivers
from tests.helpers import ReferenceVectors
from tests.test_drivers_cpu import _camera_utils

REF = ReferenceVectors('reference_samples')
RIGS = {'default': {}, 'ffhq': dict(avg_camera_pivot=[0, 0, 0.2], avg_camera_radius=2.7),
        'off_axis': dict(avg_camera_pivot=[0.05, -0.1, 0.15], avg_camera_radius=3.2)}
FOVS = {'18.837': 18.837, '18': 18, '12': 12, '30': 30}


def _script_cameras(rk, fov_deg):
    """(camera_params of the three yaws [3, 25], conditioning_params [1, 25]) as gen_samples_next3d.py:162, 186-196 builds them."""
    cu = _camera_utils()
    intrinsics = cu.FOV_to_intrinsics(fov_deg)
    cams = []
    angle_p = -0.2
    for angle_y, angle_p in [(.4, angle_p), (0, angle_p), (-.4, angle_p)]:
        cam_pivot = torch.tensor(rk.get('avg_camera_pivot', [0, 0, 0]))
        cam_radius = rk.get('avg_camera_radius', 2.7)
        cam2world_pose = cu.LookAtPoseSampler.sample(np.pi / 2 + angle_y, np.pi / 2 + angle_p, cam_pivot, radius=cam_radius)
        conditioning_cam2world_pose = cu.LookAtPoseSampler.sample(np.pi / 2, np.pi / 2, cam_pivot, radius=cam_radius)
        cams.append(torch.cat([cam2world_pose.reshape(-1, 16), intrinsics.reshape(-1, 9)], 1))
        conditioning_params = torch.cat([conditioning_cam2world_pose.reshape(-1, 16), intrinsics.reshape(-1, 9)], 1)
    return torch.cat(cams), conditioning_params


class _Rig(torch.nn.Module):
    def __init__(self, rk):
        super().__init__()
        self.rendering_kwargs = rk


@pytest.mark.parametrize('rig', list(RIGS))
@pytest.mark.parametrize('fov', list(FOVS))
def test_cameras_are_the_script_s(rig, fov):
    cams, cond = drivers.sample_sheet_cameras(_Rig(RIGS[rig]), FOVS[fov])
    assert cams.dtype == cond.dtype == torch.float32 and cams.shape == (3, 25) and cond.shape == (1, 25)
    assert torch.equal(cams, REF.get(f'cams_{rig}_{fov}', lambda: _script_cameras(RIGS[rig], FOVS[fov])[0]))
    assert torch.equal(cond, REF.get(f'cond_{rig}_{fov}', lambda: _script_cameras(RIGS[rig], FOVS[fov])[1]))


def test_default_fov_is_18_837():
    G = _Rig(RIGS['ffhq'])
    assert torch.equal(drivers.sample_sheet_cameras(G)[0], drivers.sample_sheet_cameras(G, 18.837)[0])
    assert not torch.equal(drivers.sample_sheet_cameras(G, 18)[0], drivers.sample_sheet_cameras(G, 18.837)[0])


class _StubMapG(_Rig):
    z_dim = 7

    def __init__(self):
        super().__init__(dict(RIGS['ffhq']))
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.calls = []

    def mapping(self, z, c, truncation_psi=1, truncation_cutoff=None):
        self.calls.append((z, c, truncation_psi, truncation_cutoff))
        return z.float()[:, None].repeat(1, 28, 1)


def test_seed_latents_and_mapping_inputs():
    seeds = [0, 1, 4, 5, 6, 10720, 2 ** 32 - 1]
    z = drivers.seed_latents(seeds, 512)
    assert z.dtype == torch.float64 and z.shape == (len(seeds), 512)
    for s, seed in enumerate(seeds):
        assert np.array_equal(z[s].numpy(), np.random.RandomState(seed).randn(1, 512)[0])     # gen_samples_next3d.py:184
    G = _StubMapG()
    ws = drivers.sample_sheet_ws(G, seeds[:3], truncation_psi=0.7, truncation_cutoff=10, fov_deg=12)
    zc, c, psi, cutoff = G.calls[0]
    assert torch.equal(zc, drivers.seed_latents(seeds[:3], G.z_dim)) and (psi, cutoff) == (0.7, 10)
    assert torch.equal(c, REF.get('cond_ffhq_12', lambda: _script_cameras(RIGS['ffhq'], 12)[1]).expand(3, -1))
    assert ws.shape == (3, 28, G.z_dim)
    with pytest.raises(ValueError, match='seeds'):
        drivers.sample_sheet_ws(G, [])


def _script_sheet(imgs):
    """gen_samples_next3d.py:201-206: the uint8 image of each yaw, concatenated along the width, sample 0."""
    out = []
    for img in imgs:
        img = (img.permute(0, 2, 3, 1) * 127.5 + 128).clamp(0, 255).to(torch.uint8)
        out.append(img)
    img = torch.cat(out, dim=2)
    return img[0].cpu().numpy()


def test_sheet_layout_is_the_script_s():
    g = torch.Generator().manual_seed(5)
    B, H, W = 3, 6, 5
    front = torch.randn(B, 3, H, W, generator=g) * 1.5
    views = torch.randn(2 * B, 3, H, W, generator=g) * 1.5
    got = drivers.sheet_u8(front, views)
    assert got.shape == (B, H, 3 * W, 3) and got.dtype == torch.uint8
    for b in range(B):
        assert np.array_equal(got[b].numpy(), _script_sheet([front[b:b + 1], views[2 * b:2 * b + 1], views[2 * b + 1:2 * b + 2]]))


# ------------------------------------------------------------------------------------------------ the drivers with a stub generator
def _image(ws, c, noise, res):
    """A deterministic image per (ws, camera, sampler noise) row, values past [-1, 1] included."""
    s = ws.mean(dim=(1, 2)) * 3 + c.mean(dim=1)
    if noise is not None:
        s = s + noise[0].mean(dim=(1, 2, 3)) + noise[1].reshape(ws.shape[0], -1).mean(1)
    ramp = torch.linspace(-1.5, 1.5, 3 * res * res).reshape(1, 3, res, res)
    return torch.tanh(s)[:, None, None, None] * 2 + ramp


class _StubSheetG(torch.nn.Module):
    """The generator interface the sample-sheet drivers use: synthesis with cache_backbone, render_views of the cached heads and the
    engine's cached_sigma_grid; records every call."""
    w_dim = 512

    def __init__(self, res=8):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.img_resolution = res
        self.rendering_kwargs = dict(RIGS['ffhq'])
        self.calls, self.cached = [], None

    def synthesis(self, ws, c, v, noise_mode='random', cache_backbone=False, seed=None, sampler_noise=None):
        assert noise_mode == 'const' and cache_backbone and v.shape[0] == ws.shape[0] == c.shape[0]
        self.calls.append(('synthesis', ws.shape[0], seed))
        self.cached = ws.clone()
        return {'image': _image(ws, c, sampler_noise, self.img_resolution)}

    def render_views(self, c, seed=None, sampler_noise=None):
        self.calls.append(('render_views', c.shape[0], seed))
        ws = self.cached.repeat_interleave(c.shape[0] // self.cached.shape[0], 0)
        return {'image': _image(ws, c, sampler_noise, self.img_resolution)}

    def _get_engine(self):
        return self

    def cached_sigma_grid(self, b, shape_res, sigma):
        self.calls.append(('grid', b))
        sigma.copy_(self.cached[b].mean() + torch.arange(float(shape_res ** 3)).reshape((shape_res,) * 3))


def _sheet_inputs(S, res=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    ws = torch.randn(S, 28, 512, generator=g)
    v = torch.randn(1, 9, 3, generator=g)
    M = 4
    noise = (torch.rand(3 * S, M, 3, 1, generator=g), torch.rand(3 * S, M, 2, generator=g))
    return ws, v, noise


def _expected(G, ws, i, noise, shape_res):
    """Seed i as the script renders it: one call per yaw, rows 3 i + yaw of the noise; and its stub grid."""
    cams, _ = drivers.sample_sheet_cameras(G)
    imgs = [_image(ws[i:i + 1], cams[j:j + 1], (noise[0][3 * i + j:3 * i + j + 1], noise[1][3 * i + j]), G.img_resolution) for j in range(3)]
    return _script_sheet(imgs), (ws[i].mean() + torch.arange(float(shape_res ** 3)).reshape((shape_res,) * 3)).numpy()


@pytest.mark.parametrize('S,batch', [(1, 3), (4, 6), (7, 9), (5, 2)])
def test_sheets_batching_padding_and_noise_rows(S, batch):
    ws, v, noise = _sheet_inputs(S)
    G = _StubSheetG()
    got = list(drivers.render_sample_sheets(G, ws, v, batch=batch, shapes=True, shape_res=3, sampler_noise=noise))
    B = max(1, batch // 3)
    steps = -(-S // B)
    assert [i for i, _, _ in got] == list(range(S))
    for i, sheet, sig in got:
        want_sheet, want_sig = _expected(G, ws, i, noise, 3)
        assert sheet.dtype == np.uint8 and np.array_equal(sheet, want_sheet), i
        assert sig.dtype == np.float32 and np.array_equal(sig, want_sig), i
    calls = [c for c in G.calls if c[0] != 'grid']
    assert calls == [('synthesis', B, None), ('render_views', 2 * B, None)] * steps
    assert [c[1] for c in G.calls if c[0] == 'grid'] == [b for k in range(steps) for b in range(min(B, S - k * B))]


def test_sheets_without_shapes_and_seeds():
    ws, v, _ = _sheet_inputs(4)
    G = _StubSheetG()
    got = list(drivers.render_sample_sheets(G, ws, v, batch=6, seed=10))
    assert all(sig is None for _, _, sig in got) and len(got) == 4
    assert G.calls == [('synthesis', 2, 10), ('render_views', 4, 11), ('synthesis', 2, 12), ('render_views', 4, 13)]


@pytest.mark.parametrize('what,kw,match', [
    ('ws', dict(ws=torch.zeros(0, 28, 512)), 'ws holds no seed'),
    ('ws', dict(ws=torch.zeros(2, 14, 512)), r'ws must be \[S, 28, 512\]'),
    ('ws', dict(ws=torch.zeros(28, 512)), r'ws must be \[S, 28, 512\]'),
    ('batch', dict(batch=0), 'batch must be at least 1'),
    ('shape_res', dict(shape_res=1), 'shape_res must be at least 2'),
    ('v', dict(v=torch.zeros(2, 9, 3)), 'v must be one mesh'),
    ('v', dict(v=torch.zeros(9, 3)), 'v must be one mesh'),
])
def test_refusals_name_the_argument(what, kw, match):
    ws, v, _ = _sheet_inputs(2)
    args = dict(ws=ws, v=v, batch=3, shape_res=8)
    args.update(kw)
    def meshes(G, ws, v, batch, shapes, shape_res):
        return list(drivers.coloured_meshes(G, ws, v, batch=batch, shape_res=shape_res))
    for fn in (drivers.render_sample_sheets, drivers.render_sample_sheets_sharded, meshes):
        G = _StubSheetG()
        with pytest.raises(ValueError, match=match):
            fn(G, args['ws'], args['v'], batch=args['batch'], shapes=True, shape_res=args['shape_res'])
        assert G.calls == []                                            # refused before any call into the generator


# ------------------------------------------------------------------------------------------------ sharded twin (gloo)
def _worker(rank, world, port, S, q):
    from next3d_b200 import distributed as D
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    D.init_from_env('gloo')
    ws, v, noise = _sheet_inputs(S, seed=3)
    sheets, grids = drivers.render_sample_sheets_sharded(_StubSheetG(512), ws, v, batch=6, shapes=True, shape_res=2, sampler_noise=noise,
                                                         device='cpu')
    q.put((rank, None if sheets is None else sheets.numpy(), grids))
    torch.distributed.destroy_process_group()


def test_sharded_sheets_gloo():
    """S = 5 seeds over 2 ranks (3 + 2), 512 x 1536 sheets gathered to rank 0; every rank keeps the grids of its own seeds."""
    S = 5
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, S, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict((r, (sh, gr)) for r, sh, gr in (q.get(timeout=300) for _ in range(2)))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    ws, _, noise = _sheet_inputs(S, seed=3)
    G = _StubSheetG(512)
    sheets = got[0][0]
    assert got[1][0] is None and sheets.shape == (S, 512, 1536, 3)
    assert sorted(got[0][1]) == [0, 1, 2] and sorted(got[1][1]) == [3, 4]
    for i in range(S):
        want_sheet, want_sig = _expected(G, ws, i, noise, 2)
        assert np.array_equal(sheets[i], want_sheet), i
        assert np.array_equal(got[0 if i < 3 else 1][1][i], want_sig), i
