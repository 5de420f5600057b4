"""GPU: long rays, 97 .. 192 samples per pass (render_fused_kernel<64, *>: one ray across a warp pair), as
gen_videos_next3d.py --sample_mult 2.5 .. 4 asks for.  The renderer against the CPU oracle with injected sampler uniforms, the normal
path at long rays, and the generator / driver entry points with nothing but the sample counts changed."""
import copy
import dataclasses
import math

import numpy as np
import pytest
import torch

from tests.helpers import range_rel_err
from tests.test_gpu_normals import _check_against_oracle, _workload

pytestmark = pytest.mark.gpu
DEV = 'cuda'
TOL = 1e-3                   # generator tolerance of tests/test_gpu_generator.py


@pytest.fixture(scope='module')
def K():
    from next3d_b200 import kernels
    return kernels


def _dec(sd):
    return ((sd['decoder.net.0.weight'] / math.sqrt(32)).to(DEV).contiguous(), sd['decoder.net.0.bias'].to(DEV),
            (sd['decoder.net.2.weight'] / math.sqrt(64)).to(DEV).contiguous(), sd['decoder.net.2.bias'].to(DEV))


# both passes on the new layout, ragged tiles (97, 100, 120, 144), full tiles (192), coarse-only, unequal counts with one pass on
# fewer tiles than the other, odd image sizes (the 1 x 2 pixel block leaves a ragged row), several images with a ragged last group
@pytest.mark.parametrize('N,res,D,Df,ties', [(1, 16, 97, 97, 0), (1, 16, 120, 120, 0), (2, 13, 144, 144, 0), (1, 12, 192, 192, 0),
                                             (1, 16, 192, 0, 0), (1, 16, 48, 192, 0), (1, 16, 192, 48, 0), (1, 12, 100, 37, 0),
                                             (1, 12, 144, 144, 1), (3, 9, 120, 150, 0)])
def test_render_rays_long(K, N, res, D, Df, ties):
    """Same checks and bounds as tests/test_gpu_kernels.py::test_render_rays.  ties: few distinct fine uniforms, so exactly equal fine
    depths (stable order) and crowded rank buckets (the full-count fallback of the merge)."""
    from oracle import renderer as orr
    opts, planes, sd, c, u_c, u_f = _workload(N, res, D, Df, ties)
    o, d = orr.ray_sampler(c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3), res)
    rgb_ref, depth_ref, w_ref = orr.render(sd, planes, o, d, opts, u_c, u_f)
    pl = planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    rgb = torch.full((N, res * res, 32), float('nan'), device=DEV)
    depth = torch.full((N, res * res), float('nan'), device=DEV)
    wsum = torch.full((N, res * res), float('nan'), device=DEV)
    mm = torch.tensor([float('inf'), 0.0], device=DEV)
    K.render_rays(pl, cam, intr, res, opts, _dec(sd), rgb, depth, wsum, mm, u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV))
    K.depth_clamp(depth, mm)
    assert range_rel_err(rgb.cpu(), rgb_ref) < 2e-5
    assert range_rel_err(wsum.cpu(), w_ref[..., 0]) < 2e-5
    assert range_rel_err(depth.cpu(), depth_ref[..., 0]) < 2e-5
    # in-kernel RNG: statistically the same image (different noise), finite
    rgb2 = torch.full_like(rgb, float('nan'))
    mm2 = torch.tensor([float('inf'), 0.0], device=DEV)
    K.render_rays(pl, cam, intr, res, opts, _dec(sd), rgb2, depth, wsum, mm2, seed=123)
    assert torch.isfinite(rgb2).all() and (rgb2.mean() - rgb.mean()).abs().item() < 0.05


@pytest.mark.parametrize('D,Df', [(144, 144), (192, 192)])
def test_render_rays_normals_long(K, D, Df):
    """rgb / depth / wsum bit-identical to render_rays; the exported samples and the normals against the oracle, with the criteria of
    tests/test_gpu_normals.py."""
    from oracle import normals as onr, renderer as orr
    N, res = 1, 12
    opts, planes, sd, c, u_c, u_f = _workload(N, res, D, Df, 0)
    o, d = orr.ray_sampler(c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3), res)
    ref = onr.render_normals(sd, planes, o, d, opts, u_c, u_f, return_samples=True)
    pl = planes.permute(0, 1, 3, 4, 2).contiguous().to(DEV)
    cam, intr = c[:, :16].contiguous().to(DEV), c[:, 16:25].contiguous().to(DEV)
    M = res * res

    def outputs():
        return (torch.zeros(N, M, 32, device=DEV), torch.zeros(N, M, device=DEV), torch.zeros(N, M, device=DEV),
                torch.tensor([float('inf'), 0.0], device=DEV))

    for noise in (dict(u_coarse=u_c.to(DEV), u_fine=u_f.to(DEV)), dict(seed=123)):
        a, b = outputs(), outputs()
        K.render_rays(pl, cam, intr, res, opts, _dec(sd), *a, **noise)
        normal = torch.full((N, M, 3), float('nan'), device=DEV)
        work = torch.full((K.normals_workspace_floats(N, res, opts),), float('nan'), device=DEV)
        assert work.numel() == M * (2 * (D + Df) - 1)
        K.render_rays_normals(pl, cam, intr, res, opts, _dec(sd), *b, normal, work, **noise)
        for x, y, name in zip(a, b, ('rgb', 'depth', 'wsum', 'depth_minmax')):
            assert torch.equal(x, y), name
        assert not torch.isnan(work).any()                     # every ray's D depths and D - 1 weights written
        if 'u_coarse' in noise:
            _check_against_oracle(sd, planes, o, d, opts, work.view(N, M, -1), normal, ref)
        else:
            live = b[2] > 1e-3
            assert torch.isfinite(normal[live]).all()
            assert (normal[live].norm(dim=-1) - 1).abs().max().item() <= 1e-5


def _generator(Dc, Df, seed):
    from next3d_b200 import config, weights
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    base = config.tiny_config(512)
    rk = copy.deepcopy(base.rendering_kwargs)
    rk.update(depth_resolution=Dc, depth_resolution_importance=Df)
    cfg = dataclasses.replace(base, rendering_kwargs=rk)
    sd = weights.make_state_dict(cfg, seed=seed)
    return cfg, sd, TriPlaneGenerator.from_config(cfg, sd, device=DEV)


def test_generator_144_samples_vs_oracle_and_graph():
    """gen_videos_next3d.py --sample_mult 3 (48 * 3 = 144 + 144): synthesis against the oracle generator with injected sampler
    noise (criteria of test_c3_shape_128_render_96_samples), CUDA-graph replay == eager, and return_normal at the same setting."""
    from next3d_b200 import weights
    from oracle import generator as og
    cfg, sd, G = _generator(144, 144, 8)
    N = 2
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, N, seed=8)
    u_c, u_f = weights.sampler_noise(cfg, N, seed=8)
    R = cfg.neural_rendering_resolution
    assert u_c.shape == (N, R * R, 144, 1) and u_f.shape == (N * R * R, 144)
    ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    out = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', sampler_noise=(u_c.to(DEV), u_f.to(DEV)))
    with torch.no_grad():
        ref = og.synthesis(sd, cfg, ws.cpu(), c_cam, v, u_c, u_f)
    for k in ('image', 'image_raw', 'image_depth'):
        assert range_rel_err(out[k].cpu(), ref[k]) < TOL, k
    eager = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7).items()}
    G.use_cuda_graph = True
    try:
        graphed = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7).items()}
    finally:
        G.use_cuda_graph = False
    assert set(graphed) == set(eager)
    for k in eager:
        assert torch.equal(graphed[k], eager[k]), k
    G.rendering_kwargs['return_normal'] = True
    try:
        on = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=7)
    finally:
        G.rendering_kwargs['return_normal'] = False
    for k in ('image', 'image_raw', 'image_depth'):
        assert torch.equal(on[k], eager[k]), k
    n = on['image_normal']
    live = torch.isfinite(n).all(1)
    assert n.shape == (N, 3, R, R) and live.float().mean().item() > 0.9
    assert (n.norm(dim=1)[live] - 1).abs().max().item() <= 1e-4


@pytest.mark.parametrize('mult', [2.5, 4])
def test_generator_sample_mult_returns_images(mult):
    """--sample_mult 2.5 and 4 (gen_videos_next3d.py:290-291: int(48 * mult) coarse and importance samples): synthesis, eager and
    graphed, returns finite images, and drivers.render_frames renders an orbit."""
    from next3d_b200 import drivers, weights
    D = int(48 * mult)
    cfg, sd, G = _generator(D, D, 9)
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, 2, seed=9)
    ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    eager = {k: t.clone() for k, t in G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=3).items()}
    for k in ('image', 'image_raw', 'image_depth'):
        assert torch.isfinite(eager[k]).all(), k
    assert eager['image'].shape == (2, 3, cfg.img_resolution, cfg.img_resolution)
    G.use_cuda_graph = True
    try:
        graphed = G.synthesis(ws, c_cam.to(DEV), v.to(DEV), noise_mode='const', seed=3)
        assert torch.equal(graphed['image'], eager['image'])
    finally:
        G.use_cuda_graph = False
    F = 3
    wsf = drivers.interpolate_ws(ws.cpu(), 3, wraps=1)[:F]
    cams = drivers.orbit_camera_params(F, torch.tensor([0, 0, 0.2]), 2.7)
    frames = list(drivers.render_frames(G, wsf, cams, v[:1], batch=2))
    assert len(frames) == F and frames[0].shape == (cfg.img_resolution, cfg.img_resolution, 3) and frames[0].dtype == np.uint8
    assert not np.array_equal(frames[0], frames[-1])
