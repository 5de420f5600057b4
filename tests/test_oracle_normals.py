"""CPU: the normal-path oracle (oracle.normals.render_normals) against the reference's own ImportanceRenderer.normal_forward +
MipRayMarcher2 (return_normal) on seeded planes, cameras and injected sampler uniforms.  What the reference computed is stored in
tests/golden/reference_normals.npz (tests.helpers.ReferenceVectors; N3D_RECORD_REFERENCE=1 recomputes it where the reference can
be imported)."""
import math

import pytest
import torch

from next3d_b200 import config, weights
from oracle import normals as onr, ref_shim, renderer as orr
from tests.helpers import ReferenceVectors, range_rel_err

REF = ReferenceVectors('reference_normals')

# name: (N, res, Dc, Df, box_warp).  box_warp < 1 puts more samples outside the tri-plane box (zero-padding taps).
CASES = {'fine': (2, 6, 12, 12, 1.0), 'coarse_only': (1, 8, 16, 0, 0.8)}


def _case(name):
    N, res, Dc, Df, box_warp = CASES[name]
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=Dc, depth_resolution_importance=Df, box_warp=box_warp, return_normal=True)
    g = torch.Generator().manual_seed(71 + res)
    planes = torch.randn(N, 3, 32, 16, 16, generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    _, _, c, _ = weights.demo_inputs(cfg, N, seed=5)
    u_c = torch.rand(N, res * res, Dc, 1, generator=g)
    u_f = torch.rand(N * res * res, max(Df, 1), generator=g)
    o, d = orr.ray_sampler(c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3), res)
    return opts, planes, sd, o, d, u_c, u_f


def _reference(name):
    """normal_forward of the reference on the case; the raw composite (before normalising) is taken from the normals and weights
    its ray marcher received and returned."""
    opts, planes, sd, o, d, u_c, u_f = _case(name)
    tp = ref_shim.import_reference()
    import training_avatar_texture.volumetric_rendering.renderer as rr
    dec = tp.OSGDecoder(32, {'decoder_lr_mul': opts['decoder_lr_mul'], 'decoder_output_dim': 32})
    dec.load_state_dict({k[len('decoder.'):]: v for k, v in sd.items()})
    R = rr.ImportanceRenderer()
    run_forward = R.ray_marcher.run_forward
    captured = {}

    def capture(colors, densities, depths, rendering_options, normals=None):
        out = run_forward(colors, densities, depths, rendering_options, normals)
        if normals is not None:
            w = out[-1]
            captured['normal_raw'] = torch.sum(w * (normals[:, :, :-1] + normals[:, :, 1:]) / 2, -2) / w.sum(2)
        return out

    R.ray_marcher.run_forward = capture
    with ref_shim.injected_sampler_noise(u_c, u_f):
        rgb, depth, normal, wsum = R.normal_forward(planes, dec, o, d, opts)
    return dict(rgb=rgb.detach(), normal=normal.detach(), normal_raw=captured['normal_raw'].detach())


_live = {}


def _ref(name, key):
    def compute():
        if name not in _live:
            _live[name] = _reference(name)
        return _live[name][key]
    return REF.get(f'{name}-{key}', compute)


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_normals_match_reference(name):
    opts, planes, sd, o, d, u_c, u_f = _case(name)
    rgb, depth, wsum, normal, normal_raw = onr.render_normals(sd, planes, o, d, opts, u_c, u_f)
    assert range_rel_err(normal_raw, _ref(name, 'normal_raw')) <= 1e-5
    assert (normal - _ref(name, 'normal')).abs().max().item() <= 1e-5
    assert range_rel_err(rgb, _ref(name, 'rgb')) <= 1e-5
    assert torch.allclose(normal.norm(dim=-1), torch.ones(()), atol=1e-5)


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_normals_render_outputs_equal_render(name):
    """Taking the gradient leaves the forward values alone: rgb / depth / wsum are oracle.renderer.render's, bit for bit."""
    opts, planes, sd, o, d, u_c, u_f = _case(name)
    rgb, depth, wsum, _, _ = onr.render_normals(sd, planes, o, d, opts, u_c, u_f)
    rgb_r, depth_r, wsum_r = orr.render(sd, planes, o, d, opts, u_c, u_f)
    assert torch.equal(rgb, rgb_r) and torch.equal(depth, depth_r) and torch.equal(wsum, wsum_r)


def test_cases_cover_zero_padding():
    """Some samples of every case fall outside the tri-plane box, where grid_sample's taps are zeros."""
    for name in CASES:
        opts, planes, sd, o, d, u_c, u_f = _case(name)
        Dc = opts['depth_resolution']
        t = torch.linspace(opts['ray_start'], opts['ray_end'], Dc).reshape(1, 1, Dc, 1) + u_c * ((opts['ray_end'] - opts['ray_start']) / (Dc - 1))
        x = (o[:, :, None] + t * d[:, :, None]) * (2.0 / opts['box_warp'])
        outside = (x.abs() > 1).any(-1)
        assert 0 < outside.float().mean().item() < 0.9, name


def test_normals_point_against_the_density_gradient():
    """Finite-difference check of the oracle's per-sample normals on a single point set (independent of the reference)."""
    opts, planes, sd, *_ = _case('fine')
    g = torch.Generator().manual_seed(3)
    pts = torch.rand(1, 64, 3, generator=g, dtype=torch.float64) * 0.8 - 0.4
    sd64 = {k: v.double() for k, v in sd.items()}
    _, _, n = onr._model_with_normals(sd64, planes[:1].double(), pts, opts)
    eps = 1e-6
    for a in range(3):
        dp = torch.zeros_like(pts)
        dp[..., a] = eps
        _, sp = orr.run_model(sd64, planes[:1].double(), pts + dp, opts)
        _, sm = orr.run_model(sd64, planes[:1].double(), pts - dp, opts)
        fd = -(sp - sm)[..., 0] / (2 * eps)
        assert range_rel_err(n[..., a], fd) < 1e-6
    assert math.isfinite(n.abs().max().item())
