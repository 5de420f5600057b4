"""CPU: long rays (97 .. 192 samples per pass, gen_videos_next3d.py --sample_mult above 2).  The renderer oracle
(oracle.renderer.render) against the reference's own ImportanceRenderer on seeded planes, cameras and injected sampler uniforms;
what the reference computed is stored in tests/golden/reference_long_rays.npz (tests.helpers.ReferenceVectors;
N3D_RECORD_REFERENCE=1 recomputes it where the reference can be imported).  Also the library's sample-count limit, checked before
anything is launched."""
import ctypes as C

import pytest
import torch

from next3d_b200 import config, weights
from oracle import ref_shim, renderer as orr
from tests.helpers import ReferenceVectors, range_rel_err

REF = ReferenceVectors('reference_long_rays')

# name: (N, res, Dc, Df)
CASES = {'144_144': (1, 4, 144, 144), '192_97': (1, 4, 192, 97), '192_0': (1, 4, 192, 0)}


def _case(name):
    N, res, Dc, Df = CASES[name]
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=Dc, depth_resolution_importance=Df)
    g = torch.Generator().manual_seed(7 + Dc + Df)
    planes = torch.randn(N, 3, 32, 16, 16, generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    _, _, c, _ = weights.demo_inputs(cfg, N, seed=5)
    u_c = torch.rand(N, res * res, Dc, 1, generator=g)
    u_f = torch.rand(N * res * res, max(Df, 1), generator=g)
    o, d = orr.ray_sampler(c[:, :16].reshape(-1, 4, 4), c[:, 16:25].reshape(-1, 3, 3), res)
    return opts, planes, sd, o, d, u_c, u_f


def _reference(name):
    opts, planes, sd, o, d, u_c, u_f = _case(name)
    tp = ref_shim.import_reference()
    import training_avatar_texture.volumetric_rendering.renderer as rr
    dec = tp.OSGDecoder(32, {'decoder_lr_mul': opts['decoder_lr_mul'], 'decoder_output_dim': 32})
    dec.load_state_dict({k[len('decoder.'):]: v for k, v in sd.items()})
    with ref_shim.injected_sampler_noise(u_c, u_f):
        rgb, depth, wsum = rr.ImportanceRenderer()(planes, dec, o, d, opts)
    return dict(rgb=rgb.detach(), depth=depth.detach(), wsum=wsum.detach())


_live = {}


def _ref(name, key):
    def compute():
        if name not in _live:
            _live[name] = _reference(name)
        return _live[name][key]
    return REF.get(f'{name}-{key}', compute)


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_render_matches_reference_at_long_rays(name):
    opts, planes, sd, o, d, u_c, u_f = _case(name)
    rgb, depth, wsum = orr.render(sd, planes, o, d, opts, u_c, u_f)
    assert range_rel_err(rgb, _ref(name, 'rgb')) <= 1e-6
    assert range_rel_err(depth, _ref(name, 'depth')) <= 1e-6
    assert range_rel_err(wsum, _ref(name, 'wsum')) <= 1e-6


def _render_call(entry, Dc, Df):
    """rc of n3d_render_rays / n3d_render_rays_normals on CPU tensors with ray_end < ray_start: the sample-count check comes first,
    so a count the renderer lays out gets the ray-setup error and nothing is launched either way."""
    from next3d_b200 import _lib, kernels
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=Dc, depth_resolution_importance=Df, ray_start=2.0, ray_end=1.0)
    planes = torch.zeros(1, 3, 4, 4, 32)
    cam, intr = torch.zeros(1, 16), torch.zeros(1, 9)
    dec = (torch.zeros(64, 32), torch.zeros(64), torch.zeros(33, 64), torch.zeros(33))
    out = torch.zeros(4 * 4 * 32)
    p = kernels._render_full_desc(planes, cam, intr, 4, opts, dec, out, out, out, None, None, None, 0, None)
    if entry == 'n3d_render_rays':
        rc = _lib.lib.n3d_render_rays(C.byref(p), None)
    else:
        rc = _lib.lib.n3d_render_rays_normals(C.byref(p), kernels.ptr(out), kernels.ptr(out), None)
    return rc, _lib.lib.n3d_last_error().decode()


@pytest.mark.parametrize('entry', ['n3d_render_rays', 'n3d_render_rays_normals'])
@pytest.mark.parametrize('Dc,Df', [(193, 48), (48, 193), (193, 0), (193, 193)])
def test_more_than_192_samples_per_pass_are_refused(entry, Dc, Df):
    rc, msg = _render_call(entry, Dc, Df)
    assert rc == -2 and 'above 192 samples per pass' in msg, (rc, msg)


@pytest.mark.parametrize('entry', ['n3d_render_rays', 'n3d_render_rays_normals'])
@pytest.mark.parametrize('Dc,Df', [(192, 192), (97, 0), (144, 144), (48, 192)])
def test_up_to_192_samples_per_pass_pass_the_count_check(entry, Dc, Df):
    rc, msg = _render_call(entry, Dc, Df)
    assert rc == -1 and 'bad ray setup' in msg, (rc, msg)
