"""CPU: the calls every frame driver makes into the generator, for the six workloads in both variants (single-process generator and
sharded twin): each call's method, batch, backbone-cache flags, sampler seed and rows of injected sampler noise, against the
documented batching and seed rules; and the frames (sheets, density grids) the driver returns, against a per-frame (per-seed) loop
over the same recording stub generator.  The sharded twins run at world size 1 in this process and at world size 2 under gloo.

The rules: a plan splits F frames into steps.  A single-process driver takes exactly `batch` frames per step, ceil(F / batch)
steps; a sharded twin gives rank r the contiguous range shard_range(F, r, world) and the batch in [batch/2, batch] that pads the
largest range least, the same number of steps on every rank.  A short step repeats its last frame; a rank without frames repeats
the previous rank's last.  Step k of rank r has the global step id r * steps + k.  The sampler keywords of a call are the rows of
`sampler_noise` of its global image ids when noise is given, else `seed` + the call's seed id (the step id; 2 step and 2 step + 1 for
the two calls of a sample-sheet step) when a seed is given, else nothing."""
import json
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from next3d_b200 import distributed as D, drivers, inputs

RES = 4                                                                  # stub image resolution (the reenactment grid needs 512)


# ------------------------------------------------------------------------------------------------ the recording stub generator
def _noise(n):
    """Per-image sampler uniforms (u_coarse [n, 3, 2, 1], u_fine [n, 3, 5]) whose row f holds the value f everywhere."""
    u = torch.arange(float(n))
    return u.view(n, 1, 1, 1).expand(n, 3, 2, 1).clone(), u.view(n, 1, 1).expand(n, 3, 5).clone()


def _row_ids(sampler_noise, n):
    """The row ids a call's sampler_noise (u_coarse [n, M, Dc, 1], u_fine [n * M, Df]) carries, None for none."""
    if sampler_noise is None:
        return None
    u_c, u_f = sampler_noise
    rows = u_c.reshape(n, -1)
    fine = u_f.reshape(n, -1)
    assert u_c.shape[0] == n and torch.equal(rows, rows[:, :1].expand_as(rows)) and torch.equal(fine, rows[:, :1].expand_as(fine))
    return [int(r) for r in rows[:, 0]]


def _image(ws, c, v, rows, res):
    """A deterministic image per (ws, camera, mesh, noise row) row, values past [-1, 1] included."""
    s = ws.mean(dim=(1, 2)) * 3 + c.mean(dim=1) + v.mean(dim=(1, 2))
    if rows is not None:
        s = s + 0.01 * torch.tensor(rows, dtype=torch.float32)
    ramp = torch.linspace(-1.5, 1.5, 3 * res * res).reshape(1, 3, res, res)
    return torch.tanh(s)[:, None, None, None] * 2 + ramp


class _StubG(torch.nn.Module):
    """The generator interface of the drivers: synthesis (with the backbone cache), render_views of the cached heads and the
    engine's cached_sigma_grid.  Records every call as (method, batch, cache_backbone, use_cached_backbone, seed, noise rows)."""
    w_dim = 512

    def __init__(self, res=RES):
        super().__init__()
        self.p = torch.nn.Parameter(torch.zeros(1))
        self.img_resolution = self.neural_rendering_resolution = res
        self.rendering_kwargs = dict(avg_camera_pivot=[0, 0, 0.2], avg_camera_radius=2.7)
        self.calls, self.cached = [], None

    def synthesis(self, ws, c, v, noise_mode='random', cache_backbone=False, use_cached_backbone=False, seed=None, sampler_noise=None):
        n = ws.shape[0]
        assert noise_mode == 'const' and c.shape[0] == v.shape[0] == n
        rows = _row_ids(sampler_noise, n)
        self.calls.append(('synthesis', n, cache_backbone, use_cached_backbone, seed, rows))
        if cache_backbone:
            self.cached = ws.clone(), v.clone()
        return {'image': _image(ws, c, v, rows, self.img_resolution)}

    def render_views(self, c, seed=None, sampler_noise=None):
        n = c.shape[0]
        rows = _row_ids(sampler_noise, n)
        self.calls.append(('render_views', n, False, False, seed, rows))
        ws, v = (t.repeat_interleave(n // t.shape[0], 0) for t in self.cached)
        return {'image': _image(ws, c, v, rows, self.img_resolution)}

    def _get_engine(self):
        return self

    def cached_sigma_grid(self, b, shape_res, sigma):
        self.calls.append(('grid', b))
        sigma.copy_(_sigmas(self.cached[0][b], shape_res))


def _sigmas(w, shape_res):
    return w.mean() + torch.arange(float(shape_res ** 3)).reshape((shape_res,) * 3)


def _u8(img):
    return drivers.to_uint8_hwc(img)


def _interp_on_host(ws_keyframes, w_frames):
    """interpolate_ws_device without the device kernel: the same spline evaluated by interpolate_ws, in float32."""
    return drivers.interpolate_ws(ws_keyframes, w_frames).float()


# ------------------------------------------------------------------------------------------------ the documented plan and seed rules
def _plan(F, batch, world, rank):
    """[(global step id, frame ids, valid count)] of every step, and the frame range, of rank `rank` (world None: the single-process
    driver)."""
    if world is None:
        spans, b = [(0, F)], batch
    else:
        spans = [D.shard_range(F, r, world) for r in range(world)]
        nmax = max(e - a for a, e in spans)
        b = min(range(max(1, batch // 2), batch + 1), key=lambda x: (-(-nmax // x) * x, -x))
    steps = -(-max(e - a for a, e in spans) // b)
    a, e = spans[rank]
    return [(rank * steps + k, [min(a + k * b + j, e - 1) for j in range(b)], max(0, min(b, e - a - k * b))) for k in range(steps)], (a, e)


def _sampler(seed, noise, seed_id, rows):
    """(seed, rows) a call receives: the noise rows if noise is given, else seed + seed_id if a seed is given."""
    if noise:
        return None, rows
    return (None if seed is None else seed + seed_id), None


# ------------------------------------------------------------------------------------------------ a driving directory
def _drive_root(path, n=6):
    """dataset.json, NNNN.png (seeded 512 x 512 RGB photos), NNNN.obj and NNNN_kpt2d.txt: frames 1 .. n - 2 are usable."""
    from PIL import Image
    rng = np.random.RandomState(7)
    labels = []
    for k in range(n):
        name = f'{k:04d}'
        Image.fromarray(rng.randint(0, 256, (512, 512, 3), dtype=np.uint8)).save(os.path.join(path, f'{name}.png'))
        with open(os.path.join(path, f'{name}.obj'), 'w') as f:
            f.write(''.join(f'v {a:.6f} {b:.6f} {c:.6f}\n' for a, b, c in rng.randn(11, 3)) + 'f 1 2 3\n')
        with open(os.path.join(path, f'{name}_kpt2d.txt'), 'w') as f:
            f.write('\n'.join(f'{a:.5f} {b:.5f} {c:.5f}' for a, b, c in rng.randn(68, 3)) + '\n')
        labels.append([f'{name}.png', (rng.randn(25) * 0.1).tolist()])
    with open(os.path.join(path, 'dataset.json'), 'w') as f:
        json.dump({'labels': labels}, f)
    return path


@pytest.fixture(scope='module')
def root(tmp_path_factory):
    return _drive_root(str(tmp_path_factory.mktemp('drive')))


def _driving(root, num_frames):
    """(cameras [n, 25], meshes [n][1, V, 3], photos [n][512, 512, 3]) of the schedule's frames."""
    sch = drivers.reenact_schedule(root, num_frames)
    meshes = [inputs.load_frame(o, lm) for o, lm in zip(sch['obj_paths'], sch['lms_paths'])]
    return sch['cams'], meshes, [inputs.load_photo(p) for p in sch['png_paths']]


# ------------------------------------------------------------------------------------------------ the six workloads
def _gen(seed):
    return torch.Generator().manual_seed(seed)


class Frames:
    """render_frames / render_frames_sharded: ws [F, L, D], cams [F, 25], a static, per-frame or iterated mesh."""
    name = 'frames'

    def __init__(self, F, batch, mesh='static'):
        self.F, self.batch, self.mesh = F, batch, mesh
        g = _gen(F * 10 + batch)
        self.ws, self.cams, self.vf = torch.randn(F, 2, 3, generator=g), torch.randn(F, 25, generator=g), torch.randn(max(F, 1), 7, 3, generator=g)

    def verts(self):
        return {'static': self.vf[:1], 'per_frame': self.vf, 'iter': (self.vf[i:i + 1] for i in range(self.F))}[self.mesh]

    def run(self, G, sharded, kw, root):
        if sharded:
            return drivers.render_frames_sharded(G, self.ws, self.cams, self.verts(), batch=self.batch, device='cpu', **kw)
        return list(drivers.render_frames(G, self.ws, self.cams, self.verts(), batch=self.batch, device='cpu', **kw))

    def calls(self, world, rank, seed, noise, root):
        return [('synthesis', len(ids), False, False, *_sampler(seed, noise, sid, ids)) for sid, ids, _ in _plan(self.F, self.batch, world, rank)[0]]

    def frames(self, noise, root):
        v = [self.vf[:1] if self.mesh == 'static' else self.vf[f:f + 1] for f in range(self.F)]
        return [_u8(_image(self.ws[f:f + 1], self.cams[f:f + 1], v[f], [f] if noise else None, RES))[0] for f in range(self.F)]

    def noise(self, root):
        return _noise(self.F)


class Orbit(Frames):
    """render_orbit / render_orbit_sharded: one head ws [1, L, D] and mesh [1, V, 3], cams [F, 25]."""
    name = 'orbit'

    def run(self, G, sharded, kw, root):
        args = (G, self.ws[:1], self.cams, self.vf[:1])
        if sharded:
            return drivers.render_orbit_sharded(*args, batch=self.batch, device='cpu', **kw)
        return list(drivers.render_orbit(*args, batch=self.batch, **kw))

    def calls(self, world, rank, seed, noise, root):
        return [('synthesis', 1, True, False, 0, None)] + [('render_views', len(ids), False, False, *_sampler(seed, noise, sid, ids))
                                                          for sid, ids, _ in _plan(self.F, self.batch, world, rank)[0]]

    def frames(self, noise, root):
        return [_u8(_image(self.ws[:1], self.cams[f:f + 1], self.vf[:1], [f] if noise else None, RES))[0] for f in range(self.F)]


class Reenact:
    """reenact_frames / reenact_frames_sharded: one identity driven by the directory's meshes and cameras (noise_mode 'const':
    the first step caches the backbone, the later ones reuse it)."""
    name = 'reenact'

    def __init__(self, num_frames, batch):
        self.num_frames, self.batch = num_frames, batch
        self.ws = torch.randn(1, 2, 3, generator=_gen(11))

    def n(self, root):
        return len(drivers.reenact_schedule(root, self.num_frames)['ks'])

    def run(self, G, sharded, kw, root):
        if sharded:
            return drivers.reenact_frames_sharded(G, self.ws, root, self.num_frames, batch=self.batch, device='cpu', workers=2, **kw)
        return list(drivers.reenact_frames(G, self.ws, root, self.num_frames, batch=self.batch, workers=2, **kw))

    def calls(self, world, rank, seed, noise, root):
        return [('synthesis', len(ids), k == 0, k > 0, *_sampler(seed, noise, sid, ids))
                for k, (sid, ids, _) in enumerate(_plan(self.n(root), self.batch, world, rank)[0])]

    def frames(self, noise, root):
        cams, meshes, _ = _driving(root, self.num_frames)
        return [_u8(_image(self.ws, cams[f:f + 1], meshes[f], [f] if noise else None, RES))[0] for f in range(len(meshes))]

    def noise(self, root):
        return _noise(self.n(root))


class Grid:
    """render_grid_frames / render_grid_frames_sharded: gh x gw cells, each interpolating its own K keyframes over w_frames; the
    single-process driver batches images (frame-major, cell-minor), the sharded twin whole frames of batch // cells."""
    name = 'grid'

    def __init__(self, grid, K, w_frames, batch):
        self.grid, self.w_frames, self.batch = grid, w_frames, batch
        gw, gh = grid
        g = _gen(K * 100 + batch)
        self.ws_grid, self.verts = torch.randn(gh, gw, K, 2, 3, generator=g), torch.randn(1, 7, 3, generator=g)
        self.cells, self.F = gw * gh, K * w_frames

    def run(self, G, sharded, kw, root):
        args = (G, self.ws_grid, self.verts, self.w_frames)
        if sharded:
            return drivers.render_grid_frames_sharded(*args, batch=self.batch, device='cpu', **kw)
        return list(drivers.render_grid_frames(*args, batch=self.batch, **kw))

    def calls(self, world, rank, seed, noise, root):
        if world is None:                                                # batches of images
            plan = _plan(self.F * self.cells, self.batch, None, 0)[0]
        else:                                                            # batches of frames, every cell of each
            plan = [(sid, [f * self.cells + j for f in ids for j in range(self.cells)], n)
                    for sid, ids, n in _plan(self.F, max(1, self.batch // self.cells), world, rank)[0]]
        return [('synthesis', len(ids), False, False, *_sampler(seed, noise, sid, ids)) for sid, ids, _ in plan]

    def frames(self, noise, root):
        gw, gh = self.grid
        wsf = [_interp_on_host(self.ws_grid[yi, xi], self.w_frames) for yi in range(gh) for xi in range(gw)]
        cams = drivers.orbit_camera_params(self.F, torch.tensor([0, 0, 0.2]), 2.7)
        out = []
        for f in range(self.F):
            cells = torch.cat([_image(wsf[j][f:f + 1], cams[f:f + 1], self.verts, [f * self.cells + j] if noise else None, RES)
                               for j in range(self.cells)])
            out.append(drivers.layout_cells(_u8(cells), gw, gh)[0])
        return out

    def noise(self, root):
        return _noise(self.F * self.cells)


class ReenactGrid:
    """reenact_grid_frames / reenact_grid_frames_sharded: the driving photo next to S identities, S heads x batch // S frames per
    call, head-major; the first step caches the S heads (seed 0), every step reuses them."""
    name = 'reenact_grid'

    def __init__(self, S, grid, num_frames, batch):
        self.S, self.grid, self.num_frames, self.batch = S, grid, num_frames, batch
        self.ws = torch.randn(S, 2, 3, generator=_gen(S))

    def n(self, root):
        return len(drivers.reenact_schedule(root, self.num_frames)['ks'])

    def run(self, G, sharded, kw, root):
        args = (G, self.ws, root, self.num_frames, self.grid)
        if sharded:
            return drivers.reenact_grid_frames_sharded(*args, batch=self.batch, device='cpu', workers=2, **kw)
        return list(drivers.reenact_grid_frames(*args, batch=self.batch, workers=2, **kw))

    def calls(self, world, rank, seed, noise, root):
        S, out = self.S, []
        for k, (sid, ids, _) in enumerate(_plan(self.n(root), max(1, self.batch // S), world, rank)[0]):
            if k == 0:
                out.append(('synthesis', S, True, False, 0, None))
            out.append(('synthesis', S * len(ids), False, True, *_sampler(seed, noise, sid, [f * S + s for s in range(S) for f in ids])))
        return out

    def frames(self, noise, root):
        cams, meshes, photos = _driving(root, self.num_frames)
        out = []
        for f in range(len(meshes)):
            heads = [_u8(_image(self.ws[s:s + 1], cams[f:f + 1], meshes[f], [f * self.S + s] if noise else None, 512))
                     for s in range(self.S)]
            out.append(drivers.layout_cells(torch.cat([drivers.photo_cell(photos[f], 'cpu')[None]] + heads), *self.grid)[0])
        return out

    def noise(self, root):
        return _noise(self.n(root) * self.S)


class Sheets:
    """render_sample_sheets / render_sample_sheets_sharded: batch // 3 heads per step, one caching synthesis call (yaw +0.4, seed id
    2 step) and one render_views call (yaws 0 and -0.4, seed id 2 step + 1); every seed's density grid once."""
    name = 'sheets'

    def __init__(self, S, batch, shapes=True):
        self.S, self.batch, self.shapes = S, batch, shapes
        g = _gen(S * 10 + batch)
        self.ws, self.v = torch.randn(S, 28, 512, generator=g), torch.randn(1, 7, 3, generator=g)

    def run(self, G, sharded, kw, root):
        args = (G, self.ws, self.v)
        if sharded:
            sheets, grids = drivers.render_sample_sheets_sharded(*args, batch=self.batch, shapes=self.shapes, shape_res=2, device='cpu', **kw)
            return sheets, grids
        got = list(drivers.render_sample_sheets(*args, batch=self.batch, shapes=self.shapes, shape_res=2, **kw))
        assert [i for i, _, _ in got] == list(range(self.S))
        return [s for _, s, _ in got], ({i: g for i, _, g in got} if self.shapes else [g for _, _, g in got])

    def calls(self, world, rank, seed, noise, root):
        plan, (a, e) = _plan(self.S, max(1, self.batch // 3), world, rank)
        out, done = [], set()
        for sid, ids, _ in plan:
            out.append(('synthesis', len(ids), True, False, *_sampler(seed, noise, 2 * sid, [3 * i for i in ids])))
            out.append(('render_views', 2 * len(ids), False, False, *_sampler(seed, noise, 2 * sid + 1,
                                                                               [3 * i + 1 + j for i in ids for j in range(2)])))
            new = [i for i in dict.fromkeys(ids) if a <= i < e and i not in done] if self.shapes else []
            done.update(new)
            out += [('grid', b) for b in range(len(new))]
        return out

    def frames(self, noise, root):
        cams, _ = drivers.sample_sheet_cameras(_StubG())
        out = []
        for i in range(self.S):
            imgs = [_image(self.ws[i:i + 1], cams[j:j + 1], self.v, [3 * i + j] if noise else None, RES) for j in range(3)]
            out.append(drivers.sheet_u8(imgs[0], torch.cat(imgs[1:]))[0])
        return out

    def grids(self):
        return {i: _sigmas(self.ws[i], 2).numpy() for i in range(self.S)}

    def noise(self, root):
        return _noise(3 * self.S)


WORKLOADS = {
    'frames_ragged': Frames(5, 2, 'static'),
    'frames_per_frame': Frames(4, 4, 'per_frame'),
    'frames_empty': Frames(0, 3, 'static'),
    'orbit_ragged': Orbit(5, 3),
    'reenact_ragged': Reenact(3, 2),
    'reenact_empty': Reenact(0, 2),
    'grid_split_frames': Grid((2, 1), 2, 3, 3),
    'grid_2x2': Grid((2, 2), 1, 3, 8),
    'reenact_grid_1': ReenactGrid(1, (2, 1), 3, 2),
    'reenact_grid_2': ReenactGrid(2, (3, 1), 3, 4),
    'reenact_grid_empty': ReenactGrid(1, (2, 1), 0, 2),
    'sheets_ragged': Sheets(5, 6),
    'sheets_no_shapes': Sheets(3, 3, shapes=False),
}
SINGLE_ONLY = {'frames_iter': Frames(5, 3, 'iter')}                      # the sharded twins take mesh tensors only


def _kw(seed, noise, w, root):
    """Driver keywords of a (seed, noise) case; the sharded twins' seed defaults to 0."""
    kw = {} if seed is None else {'seed': seed}
    if noise:
        kw['sampler_noise'] = w.noise(root)
    return kw


def _check(w, got, calls, world, rank, seed, noise, root, sharded):
    """The calls of rank `rank` and, unless got is None (a rank other than 0), the frames it returned; the density grids of the
    sample sheets on every rank (a sharded rank holds those of its own seeds)."""
    assert calls == w.calls(world, rank, seed if seed is not None or not sharded else 0, noise, root)
    frames, grids = got if isinstance(w, Sheets) else (got, None)
    if frames is not None:
        want = w.frames(noise, root)
        assert len(frames) == len(want)
        for f, (a, b) in enumerate(zip(frames, want)):
            a = np.asarray(a)
            assert a.dtype == np.uint8 and np.array_equal(a, b.numpy()), f
    if isinstance(w, Sheets) and not w.shapes:
        assert grids == ({} if sharded else [None] * w.S)
    elif isinstance(w, Sheets):
        lo, hi = D.shard_range(w.S, rank, world or 1)
        assert sorted(grids) == list(range(lo, hi))
        for i, g in grids.items():
            assert g.dtype == np.float32 and np.array_equal(g, w.grids()[i]), i


def _res(w):
    return 512 if isinstance(w, ReenactGrid) else RES


SAMPLERS = {'unseeded': (None, False), 'seeded': (5, False), 'noise': (None, True), 'seeded_noise': (5, True)}
VARIANTS = ('single', 'sharded_1', 'sharded_2')                          # the generator; the sharded twin at world size 1, 2


def _noise_replaces_a_seed(name, variant, seed, noise):
    """The calls that once passed a seed next to the noise rows: the single-process drivers given both, and the sharded
    reenactment grid (whose seed defaults to 0).  The renderer draws no random numbers when both uniform arrays are given, so the
    seed never changed a pixel; now noise takes its place."""
    return noise and (isinstance(WORKLOADS[name], ReenactGrid) if variant != 'single' else seed is not None)


def _cases(replaced):
    return [pytest.param(variant, name, seed, noise, id=f'{variant}-{name}-{sampler}')
            for variant in VARIANTS for name in list(WORKLOADS) + (list(SINGLE_ONLY) if variant == 'single' else [])
            for sampler, (seed, noise) in SAMPLERS.items() if _noise_replaces_a_seed(name, variant, seed, noise) == replaced]


def _run_and_check(request, monkeypatch, root, variant, name, seed, noise):
    w = {**WORKLOADS, **SINGLE_ONLY}[name]
    if variant == 'sharded_2':
        for rank, (calls, got) in enumerate(request.getfixturevalue('world_2')[name, seed, noise]):
            assert ((got[0] if isinstance(w, Sheets) else got) is None) == (rank == 1)
            _check(w, got, calls, 2, rank, seed, noise, root, True)
        return
    monkeypatch.setattr(drivers, 'interpolate_ws_device', _interp_on_host)
    G = _StubG(_res(w))
    sharded = variant == 'sharded_1'
    got = w.run(G, sharded, _kw(seed, noise, w, root), root)
    _check(w, got, G.calls, 1 if sharded else None, 0, seed, noise, root, sharded)


@pytest.mark.parametrize('variant,name,seed,noise', _cases(False))
def test_driver_calls(request, monkeypatch, root, variant, name, seed, noise):
    _run_and_check(request, monkeypatch, root, variant, name, seed, noise)


@pytest.mark.parametrize('variant,name,seed,noise', _cases(True))
def test_noise_takes_the_place_of_the_seed(request, monkeypatch, root, variant, name, seed, noise):
    """Given sampler noise, a call gets its noise rows and no seed, whatever `seed` is."""
    _run_and_check(request, monkeypatch, root, variant, name, seed, noise)


# ------------------------------------------------------------------------------------------------ sharded twins, world size 2 (gloo)
def _worker(rank, world, port, root, q):
    """Every sharded case on one rank: [(calls, result)] with the results as numpy arrays."""
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    D.init_from_env('gloo')
    drivers.interpolate_ws_device = _interp_on_host
    out = []
    try:
        for name in WORKLOADS:
            for seed, noise in SAMPLERS.values():
                w = WORKLOADS[name]
                G = _StubG(_res(w))
                got = w.run(G, True, _kw(seed, noise, w, root), root)
                if isinstance(w, Sheets):
                    got = (None if got[0] is None else got[0].numpy(), got[1])
                elif got is not None:
                    got = got.numpy()
                out.append(((name, seed, noise), G.calls, got))
    finally:
        q.put((rank, out))
        torch.distributed.destroy_process_group()


@pytest.fixture(scope='module')
def world_2(root):
    """{(workload, seed, noise): [(calls, result) of rank 0, of rank 1]}: all sharded cases in one gloo world of two processes."""
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, root, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=600) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert len(got[0]) == len(got[1]) == len(WORKLOADS) * len(SAMPLERS)
    return {case: [(calls, res) for r in (0, 1) for c, calls, res in got[r] if c == case] for case, _, _ in got[0]}
