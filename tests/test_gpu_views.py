"""GPU: new camera views without regenerating the head.  The renderer's `views` field (image n reads plane set n // views) against
repeated plane sets; the generator's backbone cache (synthesis with cache_backbone / use_cached_backbone, render_views), eager and
graphed, against plain synthesis; and the drivers built on it (drivers.render_orbit, drivers.reenact_frames)."""
import numpy as np
import pytest
import torch

from tests.helpers import range_rel_err
from tests.test_gpu_normals import _workload
from tests.test_gpu_render_long_rays import _dec

pytestmark = pytest.mark.gpu
DEV = 'cuda'
BATCH_TOL = 1e-5            # test_gpu_generator.py::test_batch_invariance_and_rng_modes: the same image in batches of other sizes
KEYS = ('image', 'image_raw', 'image_depth')


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


# ------------------------------------------------------------------------------------------------ kernel
@pytest.mark.parametrize('D', [48, 96, 144])                 # the 16-, 32- and 64-lane layouts
@pytest.mark.parametrize('B,V', [(1, 5), (2, 3), (3, 1)])
def test_render_rays_views_equal_repeated_planes(K, B, V, D):
    """views = V on B plane sets == views = 1 on the sets repeated V times, bit for bit, with injected and in-kernel uniforms; also
    through render_rays_normals (normals and exported samples).  res 13: ragged pixel blocks in every layout."""
    N, res = B * V, 13
    opts, planes, sd, c, u_c, u_f = _workload(N, res, D, D, 0)
    sets = planes[:B].permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    rep = sets.repeat_interleave(V, 0)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    M = res * res
    dec = _dec(sd)

    def outputs():
        return [torch.full((N, M, 32), float('nan'), device=DEV), torch.full((N, M), float('nan'), device=DEV),
                torch.full((N, M), float('nan'), device=DEV), torch.tensor([float('inf'), 0.0], device=DEV)]

    for noise in (dict(u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV)), dict(seed=77)):
        a, b = outputs(), outputs()
        K.render_rays(rep, cam, intr, res, opts, dec, *a, **noise)
        K.render_rays(sets, cam, intr, res, opts, dec, *b, views=V, **noise)
        for x, y, name in zip(a, b, ('rgb', 'depth', 'wsum', 'depth_minmax')):
            assert torch.equal(x, y), name
        a, b = outputs(), outputs()
        na, nb = (torch.full((N, M, 3), float('nan'), device=DEV) for _ in range(2))
        wa, wb = (torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV) for _ in range(2))
        K.render_rays_normals(rep, cam, intr, res, opts, dec, *a, na, wa, **noise)
        K.render_rays_normals(sets, cam, intr, res, opts, dec, *b, nb, wb, views=V, **noise)
        for x, y, name in zip(a + [na, wa], b + [nb, wb], ('rgb', 'depth', 'wsum', 'depth_minmax', 'normal', 'workspace')):
            assert torch.equal(x.nan_to_num(123.0), y.nan_to_num(123.0)), name


# ------------------------------------------------------------------------------------------------ generator
def _generator(cfg, seed):
    from next3d_b200 import weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    sd = weights.make_state_dict(cfg, seed=seed)
    return sd, TriPlaneGenerator.from_config(cfg, sd, device=DEV)


def _inputs(cfg, G, N, seed):
    """ws, cameras, meshes and per-image sampler uniforms of N images."""
    from next3d_b200 import weights
    z, c_cond, c, v = weights.demo_inputs(cfg, N, seed=seed)
    ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    u_c, u_f = weights.sampler_noise(cfg, N, seed=seed)
    return ws, c.to(DEV), v.to(DEV), (u_c.to(DEV), u_f.to(DEV))


def _clone(out):
    return {k: t.clone() for k, t in out.items()}


def _assert_equal(a, b, keys=None):
    for k in keys or a:
        assert torch.equal(a[k], b[k]), k


def _backbone_launches(G, cfg):
    """Kernel launches of the two ws-only backbones at the engine's current batch (after a synthesis call)."""
    from next3d_b200 import kernels
    eng = G._get_engine()
    n0 = kernels.launches
    eng._backbone('texture_backbone.synthesis', cfg.plane_ch, 'const')
    eng._backbone('backbone.synthesis', cfg.plane_ch * 3, 'const')
    return kernels.launches - n0


@pytest.fixture(scope='module')
def tiny():
    from next3d_b200 import config
    cfg = config.tiny_config(512)
    sd, G = _generator(cfg, 4)
    return cfg, sd, G


def test_cache_fill_returns_plain_synthesis(tiny):
    cfg, _, G = tiny
    ws, c, v, noise = _inputs(cfg, G, 2, 21)
    plain = _clone(G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise))
    cached = G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise, cache_backbone=True)
    _assert_equal(plain, cached, KEYS)
    cache = G._get_engine()._cache
    assert cache['B'] == 2 and cache['noise_mode'] == 'const' and torch.equal(cache['ws'], ws)


def test_use_cached_backbone_equals_plain_synthesis(tiny):
    """The reference's semantics: the ws-only backbones come from the cache, everything that depends on the mesh and the cameras
    is recomputed; the launch count drops by exactly the two backbones'."""
    cfg, _, G = tiny
    ws, c, v, noise = _inputs(cfg, G, 2, 22)
    _, c2, _, noise2 = _inputs(cfg, G, 2, 23)
    v2 = v + torch.randn(v.shape, generator=torch.Generator().manual_seed(1)).to(DEV) * 2e-3          # another expression
    G.synthesis(ws, c, v, noise_mode='const', cache_backbone=True, seed=1)
    plain = _clone(G.synthesis(ws, c2, v2, noise_mode='const', sampler_noise=noise2))
    eng = G._get_engine()
    n_plain = eng.launches
    bb = _backbone_launches(G, cfg)
    reuse = G.synthesis(ws, c2, v2, noise_mode='const', sampler_noise=noise2, use_cached_backbone=True)
    _assert_equal(plain, reuse, KEYS)
    assert bb > 0 and eng.launches == n_plain - bb, (n_plain, eng.launches, bb)
    with pytest.raises(RuntimeError, match='batch 1.*batch 2'):
        G.synthesis(ws[:1], c2[:1], v2[:1], noise_mode='const', use_cached_backbone=True)
    G.repack()                                                         # a rebuilt engine has no cache: computed as usual
    _assert_equal(plain, G.synthesis(ws, c2, v2, noise_mode='const', sampler_noise=noise2, use_cached_backbone=True), KEYS)
    assert G._get_engine().launches == n_plain


def test_render_views_one_view_equals_the_caching_call(tiny):
    cfg, _, G = tiny
    ws, c, v, noise = _inputs(cfg, G, 2, 24)
    out = _clone(G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise, cache_backbone=True))
    _assert_equal(out, G.render_views(c, sampler_noise=noise), KEYS)
    out = _clone(G.synthesis(ws, c, v, noise_mode='const', seed=5, cache_backbone=True))
    _assert_equal(out, G.render_views(c, seed=5), KEYS)


@pytest.mark.parametrize('B,V', [(1, 4), (2, 3)])
def test_render_views_equals_synthesis_of_repeated_heads(tiny, B, V):
    """View n of head n // V == synthesis on the repeated ws and mesh: the planes of a batch of B and of B * V differ only in
    tensor-core tile order (BATCH_TOL on every output, depth included: both renders clamp over the same N views)."""
    cfg, _, G = tiny
    N = B * V
    ws, c, v, noise = _inputs(cfg, G, N, 25)
    heads = torch.arange(B, device=DEV) * V
    G.synthesis(ws[heads], c[heads], v[heads], noise_mode='const', seed=1, cache_backbone=True)
    got = _clone(G.render_views(c, sampler_noise=noise))
    ref = G.synthesis(ws[heads].repeat_interleave(V, 0), c, v[heads].repeat_interleave(V, 0), noise_mode='const', sampler_noise=noise)
    for k in KEYS:
        assert got[k].shape == ref[k].shape and range_rel_err(got[k].cpu(), ref[k].cpu()) < BATCH_TOL, k
    if B > 1:
        with pytest.raises(RuntimeError, match='not a multiple'):
            G.render_views(c[:N - 1])


def test_render_views_normals_graphs_and_cache_lifetime(tiny):
    cfg, sd, G = tiny
    ws, c, v, noise = _inputs(cfg, G, 2, 26)
    _, cams, _, _ = _inputs(cfg, G, 6, 27)
    # return_normal: the caching call's outputs at V = 1, and a normal map per view at V = 3
    G.rendering_kwargs['return_normal'] = True
    try:
        out = _clone(G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise, cache_backbone=True))
        _assert_equal(out, G.render_views(c, sampler_noise=noise))
        n = G.render_views(cams, seed=3)['image_normal']
        R = G.neural_rendering_resolution
        live = torch.isfinite(n).all(1)
        assert n.shape == (6, 3, R, R) and live.float().mean().item() > 0.9
        assert (n.norm(dim=1)[live] - 1).abs().max().item() <= 1e-4
    finally:
        G.rendering_kwargs['return_normal'] = False
    # graph replay == eager for all three forms
    eager_fill = _clone(G.synthesis(ws, c, v, noise_mode='const', seed=3, cache_backbone=True))
    eager_views = _clone(G.render_views(cams, seed=7))
    eager_reuse = _clone(G.synthesis(ws, cams[:2], v.flip(0), noise_mode='const', seed=4, use_cached_backbone=True))
    G.use_cuda_graph = True
    try:
        _assert_equal(eager_fill, G.synthesis(ws, c, v, noise_mode='const', seed=3, cache_backbone=True))
        _assert_equal(eager_views, G.render_views(cams, seed=7))
        _assert_equal(eager_reuse, G.synthesis(ws, cams[:2], v.flip(0), noise_mode='const', seed=4, use_cached_backbone=True))
        assert not torch.equal(G.render_views(cams, seed=8)['image'], eager_views['image'])
        # the cache survives graphed synthesis of other heads, at this batch size and at another one
        ws2, c2, v2, _ = _inputs(cfg, G, 3, 28)
        G.synthesis(ws2[:2], c2[:2], v2[:2], noise_mode='const', seed=1)
        G.synthesis(ws2, c2, v2, noise_mode='const', seed=1)
        _assert_equal(eager_views, G.render_views(cams, seed=7))
    finally:
        G.use_cuda_graph = False
    _assert_equal(eager_views, G.render_views(cams, seed=7))
    # new weights drop the cache
    G.load_state_dict(sd)
    try:
        with pytest.raises(RuntimeError, match='cache_backbone=True'):
            G.render_views(cams, seed=7)
    finally:
        G.repack()


def test_render_views_full_width():
    """The benchmark's widths (C2: full config, 64^2, 48 + 48): B = 1, V = 4."""
    from next3d_b200 import config
    cfg = config.full_config(512)
    _, G = _generator(cfg, 5)
    B, V = 1, 4
    ws, c, v, noise = _inputs(cfg, G, V, 29)
    G.synthesis(ws[:1], c[:1], v[:1], noise_mode='const', seed=1, cache_backbone=True)
    got = _clone(G.render_views(c, sampler_noise=noise))
    ref = G.synthesis(ws[:1].repeat_interleave(V, 0), c, v[:1].repeat_interleave(V, 0), noise_mode='const', sampler_noise=noise)
    for k in KEYS:
        assert range_rel_err(got[k].cpu(), ref[k].cpu()) < BATCH_TOL, k


# ------------------------------------------------------------------------------------------------ drivers
def test_render_orbit_equals_per_frame_loop(tiny):
    """The criterion of test_gpu_drivers.py::test_render_frames_equals_per_frame_loop: batches of 2, a padded last batch,
    per-frame sampler noise; then the graph path."""
    from next3d_b200 import drivers
    cfg, _, G = tiny
    ws, _, v, _ = _inputs(cfg, G, 1, 30)
    F = 5
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    R = G.neural_rendering_resolution
    D, Df = G.rendering_kwargs['depth_resolution'], G.rendering_kwargs['depth_resolution_importance']
    g = torch.Generator().manual_seed(12)
    u_c = torch.rand(F, R * R, D, 1, generator=g).to(DEV)
    u_f = torch.rand(F, R * R, Df, generator=g).to(DEV)
    got = list(drivers.render_orbit(G, ws, cams, v, batch=2, sampler_noise=(u_c, u_f)))
    assert len(got) == F and got[0].shape == (cfg.img_resolution, cfg.img_resolution, 3) and got[0].dtype == np.uint8
    for f in range(F):
        ref = G.synthesis(ws, cams[f:f + 1].to(DEV), v, noise_mode='const', sampler_noise=(u_c[f:f + 1], u_f[f]))['image']
        ref = drivers.to_uint8_hwc(ref)[0].cpu().numpy()
        assert np.array_equal(got[f], ref), f'frame {f}: max |diff| {np.abs(got[f].astype(int) - ref.astype(int)).max()}'
    G.use_cuda_graph = True
    try:
        graphed = list(drivers.render_orbit(G, ws, cams, v, batch=2, seed=7))
    finally:
        G.use_cuda_graph = False
    assert len(graphed) == F and all(f.shape == got[0].shape and f.dtype == np.uint8 for f in graphed)
    assert np.abs(graphed[0].astype(int) - graphed[2].astype(int)).max() > 0


@pytest.mark.parametrize('noise_mode', ['const', 'none', 'random'])
def test_reenact_frames_skips_the_backbones_after_the_first_batch(tiny, tmp_path, noise_mode):
    from next3d_b200 import drivers, inputs
    cfg, _, G = tiny
    ws, c, v, _ = _inputs(cfg, G, 1, 31)
    F, batch = 5, 2
    rng = np.random.RandomState(2)
    verts = np.stack([v[0].cpu().numpy() + rng.randn(*v[0].shape).astype(np.float32) * 1e-4 for _ in range(F)])
    pack = str(tmp_path / 'clip.n3dpack')
    inputs.write_frame_pack(pack, verts, c.cpu().numpy().repeat(F, 0), ids=[f'{k:04d}' for k in range(F)])
    launches, synthesis = [], G.synthesis

    def counting(*a, **kw):
        out = synthesis(*a, **kw)
        launches.append(G._get_engine().launches)
        return out
    G.synthesis = counting
    try:
        frames = list(drivers.reenact_frames(G, ws, pack, 100, batch=batch, noise_mode=noise_mode, seed=3))
    finally:
        del G.synthesis
    assert len(frames) == F and len(launches) == 3
    full = launches[0]
    bb = _backbone_launches(G, cfg)
    want = full if noise_mode == 'random' else full - bb
    assert launches[1:] == [want, want], (launches, bb)
