"""TriPlaneGenerator.sr_precision = 'fp16': the super-resolution head on fp16 operands, against the fp16 statement of the reference's
CUDA path (oracle/sr_fp16.py), the statement of the engine's own rounding points (sr_fp16.superresolution_engine_order) and the fp32
oracle, on the SR input the generator itself produced (its feature image and ws).

Bounds are range-relative (tests/helpers.range_rel_err) and stated beside the worst case measured on an H100 SXM 80 GB (700 W).
The engine and the statement round at different places (the engine modulates the activations, the reference's fused path the
weights; the engine's epilogue rounds once where the reference rounds after the conv, the noise and bias_act), so the two agree to
a few fp16 ulps of the image range, not bit for bit.
"""
import numpy as np
import pytest
import torch

from next3d_b200 import config, drivers, weights
from next3d_b200.triplane_next3d import TriPlaneGenerator
from oracle import generator as og
from oracle import sr_fp16
from tests.helpers import hot_sr_state_dict, range_rel_err, report_parity

DEV = 'cuda'
pytestmark = pytest.mark.gpu

# image vs the fp16 oracle / vs the fp32 oracle (DESIGN.md section 5).  Worst measured over CONFIGS: 2.29e-3 / 1.15e-3 (full512);
# the fp16 oracle itself is 2.08e-3 from the fp32 oracle there.
BOUND_FP16 = 4e-3
BOUND_FP32 = 3e-3
# The engine against the statement of its own rounding points: mean |d| / range (the max is whole fp16 ulps wherever a rounding
# flips: 3.5e-4 - 5.5e-4).  Measured (tiny512 / full512 / tiny256): fp16 mode 3.7e-5 / 4.7e-5 / 2.9e-5, fp32 mode 2.2e-4 / 2.9e-4 /
# 1.0e-4.  The fp32 mode must be several times further from it than the fp16 mode, so that this check tells the two modes apart.
MEAN_ENGINE_ORDER = 8e-5
MODE_RATIO = 2.5


def _mean_err(a, ref):
    return ((a.double() - ref.double()).abs().mean() / ref.double().abs().max()).item()

CONFIGS = {'tiny512': (config.tiny_config, 512, 2), 'full512': (config.full_config, 512, 1), 'tiny256': (config.tiny_config, 256, 1),
           'tiny512_hot': (config.tiny_config, 512, 2)}
HOT = {'tiny512_hot'}           # the hot SR biases of tests.helpers: every SR layer reaches the +-256 clamp on both sides


def _setup(name, seed=0):
    factory, res, batch = CONFIGS[name]
    cfg = factory(res)
    sd = hot_sr_state_dict(cfg, seed=seed) if name in HOT else weights.make_state_dict(cfg, seed=seed)
    G = TriPlaneGenerator.from_config(cfg, sd, device=DEV)
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, batch, seed=seed)
    u_c, u_f = weights.sampler_noise(cfg, batch, seed=seed)
    with torch.no_grad():
        ws = G.mapping(z.to(DEV), c_cond.to(DEV), truncation_psi=0.7, truncation_cutoff=14)
    return G, cfg, sd, ws, c_cam.to(DEV), v.to(DEV), (u_c.to(DEV), u_f.to(DEV))


def _run(G, ws, c, v, noise, mode, **kw):
    G.sr_precision = mode
    with torch.no_grad():
        out = G.synthesis(ws, c, v, noise_mode='const', sampler_noise=noise, return_intermediates=True, **kw)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize('name', list(CONFIGS))
def test_fp16_image_matches_fp16_oracle(name):
    G, cfg, sd, ws, c, v, noise = _setup(name)
    out = _run(G, ws, c, v, noise, 'fp16')
    feat = out['intermediates']['feature_image'].permute(0, 3, 1, 2).cpu()
    rgb, wsc = feat[:, :3].contiguous(), ws[:, :14].cpu()           # the SR head reads eg3d_ws = ws[:, :14] (triplane_next3d.py:183)
    sd_cpu = {k: t.cpu() if isinstance(t, torch.Tensor) else t for k, t in sd.items()}
    with torch.no_grad():
        ref16 = sr_fp16.superresolution(sd_cpu, cfg, rgb, feat, wsc)
        ref32 = og.superresolution(sd_cpu, cfg, rgb, feat, wsc)
    img = out['image'].cpu()
    img32 = _run(G, ws, c, v, noise, 'fp32')['image'].cpu()
    with torch.no_grad():
        refE = sr_fp16.superresolution_engine_order(sd_cpu, cfg, rgb, feat, wsc)
    m16, m32 = _mean_err(img, refE), _mean_err(img32, refE)
    print(f'{name}: vs the engine-order statement, mean: fp16 mode {m16:.2e}, fp32 mode {m32:.2e}; max fp16 mode '
          f'{range_rel_err(img, refE):.2e}')
    assert m16 < MEAN_ENGINE_ORDER, m16
    assert m16 < m32 / MODE_RATIO, (m16, m32)
    e16, _, _ = report_parity(f'sr_fp16_{name}_vs_fp16_oracle', img, ref16)
    e32, _, _ = report_parity(f'sr_fp16_{name}_vs_fp32_oracle', img, ref32)
    e_oracles = range_rel_err(ref16, ref32)
    report_parity(f'sr_fp16_oracle_{name}_vs_fp32_oracle', ref16, ref32)
    print(f'{name}: engine fp16 vs fp16 oracle {e16:.3e}, vs fp32 oracle {e32:.3e}; fp16 oracle vs fp32 oracle {e_oracles:.3e}')
    assert e16 < BOUND_FP16, e16
    assert e32 < BOUND_FP32, e32


def test_sr_free_outputs_equal_between_modes():
    """image_raw, image_depth and image_normal do not pass through SR: bit-identical in both modes."""
    G, cfg, sd, ws, c, v, noise = _setup('tiny512')
    G.rendering_kwargs['return_normal'] = True
    a = _run(G, ws, c, v, noise, 'fp32')
    b = _run(G, ws, c, v, noise, 'fp16')
    for k in ('image_raw', 'image_depth', 'image_normal'):
        assert torch.equal(a[k], b[k]), k
    assert not torch.equal(a['image'], b['image'])


def test_switching_back_to_fp32_is_bit_identical():
    G, cfg, sd, ws, c, v, noise = _setup('tiny512')
    _run(G, ws, c, v, noise, 'fp16')
    switched = _run(G, ws, c, v, noise, 'fp32')
    F, *_ = _setup('tiny512')
    never = _run(F, ws, c, v, noise, 'fp32')
    for k in ('image', 'image_raw', 'image_depth'):
        assert torch.equal(switched[k], never[k]), k


def test_graph_replay_equals_eager_in_fp16():
    G, cfg, sd, ws, c, v, noise = _setup('tiny512')
    G.sr_precision = 'fp16'
    with torch.no_grad():
        eager = G.synthesis(ws, c, v, noise_mode='const', seed=5)
        G.use_cuda_graph = True
        graphed = {k: t.clone() for k, t in G.synthesis(ws, c, v, noise_mode='const', seed=5).items()}   # replays overwrite
        graphed2 = G.synthesis(ws, c, v, noise_mode='const', seed=5)
        G.sr_precision = 'fp32'                         # another mode: another graph, the fp32 answer
        g32 = {k: t.clone() for k, t in G.synthesis(ws, c, v, noise_mode='const', seed=5).items()}
        G.use_cuda_graph = False
        e32 = G.synthesis(ws, c, v, noise_mode='const', seed=5)
    for k in ('image', 'image_raw', 'image_depth'):
        assert torch.equal(eager[k], graphed[k]), k
        assert torch.equal(graphed[k], graphed2[k]), k
        assert torch.equal(g32[k], e32[k]), k
    assert not torch.equal(graphed['image'], g32['image'])


def test_render_views_and_orbit_run_in_fp16():
    """render_views (eager and graphed) and render_orbit take the mode from G: their image equals synthesis' in fp16 for the same
    camera and sampler noise."""
    G, cfg, sd, ws, c, v, noise = _setup('tiny512')
    ws1, c1, v1 = ws[:1], c[:1], v[:1]
    G.sr_precision = 'fp16'
    R = G.neural_rendering_resolution
    Fn = 3
    cams = drivers.orbit_camera_params(Fn, torch.tensor([0, 0, 0.2]), 2.7).to(DEV)
    D, Df = G.rendering_kwargs['depth_resolution'], G.rendering_kwargs['depth_resolution_importance']
    g = torch.Generator().manual_seed(3)
    u_c = torch.rand(Fn, R * R, D, 1, generator=g).to(DEV)
    u_f = torch.rand(Fn, R * R, Df, generator=g).to(DEV)
    with torch.no_grad():
        want = [G.synthesis(ws1, cams[f:f + 1], v1, noise_mode='const', sampler_noise=(u_c[f:f + 1], u_f[f]))['image'] for f in range(Fn)]
        G.synthesis(ws1, c1, v1, noise_mode='const', cache_backbone=True, seed=0)
        views = G.render_views(cams, sampler_noise=(u_c, u_f.reshape(-1, Df)))['image']
        frames = list(drivers.render_orbit(G, ws1, cams, v1, batch=2, sampler_noise=(u_c, u_f)))
        G.use_cuda_graph = True
        a = G.render_views(cams, seed=9)['image'].clone()
        b = G.render_views(cams, seed=9)['image']
        G.use_cuda_graph = False
        e = G.render_views(cams, seed=9)['image']
    for f in range(Fn):
        ref = drivers.to_uint8_hwc(want[f])[0].cpu().numpy()
        assert np.array_equal(drivers.to_uint8_hwc(views[f:f + 1])[0].cpu().numpy(), ref), f
        assert np.array_equal(frames[f], ref), f
    assert torch.equal(a, b) and torch.equal(a, e)


def test_value_errors():
    G, *_ = _setup('tiny512')
    with pytest.raises(ValueError):
        G.sr_precision = 'bf16'
    G.sr_num_fp16_res = 0
    with pytest.raises(ValueError):
        G.sr_precision = 'fp16'
    assert G.sr_precision == 'fp32'
