"""CPU: the renderer oracle (oracle.renderer.ray_sampler + render) against the reference's own RaySampler + ImportanceRenderer on
the rendering options the fused renderer's conformance suite (tests/test_gpu_render_conformance.py) exercises beyond the demo
workload: white_back with and without fine samples, non-square planes, box_warp 0.5, skewed off-centre intrinsics, transparent and
opaque densities, and the minimum sample counts.  What the reference computed is stored in
tests/golden/reference_render_contract.npz (tests.helpers.ReferenceVectors; N3D_RECORD_REFERENCE=1 recomputes it where the reference
can be imported)."""
import pytest
import torch

from next3d_b200 import config, weights
from oracle import ref_shim, renderer as orr
from tests.helpers import ReferenceVectors, range_rel_err

REF = ReferenceVectors('reference_render_contract')

# name: options that differ from the default (N 2, res 4, 16 x 16 planes, Dc = Df = 12, tiny_config rendering options)
CASES = {
    'white_back_fine': dict(white_back=True),
    'white_back_coarse_only': dict(white_back=True, Df=0),
    'planes_48x80': dict(PH=48, PW=80),
    'box_warp_0.5': dict(box_warp=0.5),
    'skewed_intrinsics': dict(camera='skewed'),
    'transparent': dict(density='transparent'),
    'opaque': dict(density='opaque'),
    'dc4_df1': dict(Dc=4, Df=1),
}


def _case(name):
    c = dict(N=2, res=4, PH=16, PW=16, Dc=12, Df=12, box_warp=1.0, white_back=False, camera='demo', density='mid')
    c.update(CASES[name])
    cfg = config.tiny_config()
    opts = dict(cfg.rendering_kwargs, depth_resolution=c['Dc'], depth_resolution_importance=c['Df'], box_warp=c['box_warp'],
                white_back=c['white_back'])
    g = torch.Generator().manual_seed(11 + sorted(CASES).index(name))
    N, res = c['N'], c['res']
    planes = torch.randn(N, 3, 32, c['PH'], c['PW'], generator=g)
    sd = {'decoder.net.0.weight': torch.randn(64, 32, generator=g), 'decoder.net.0.bias': torch.randn(64, generator=g) * 0.1,
          'decoder.net.2.weight': torch.randn(33, 64, generator=g), 'decoder.net.2.bias': torch.randn(33, generator=g) * 0.1}
    if c['density'] == 'transparent':           # sigma = -200 everywhere: softplus(-201) is 0 in fp32, every weight is 0
        sd['decoder.net.2.weight'][0] = 0
        sd['decoder.net.2.bias'][0] = -200.0
    elif c['density'] == 'opaque':              # alpha = 1 on the first interval
        sd['decoder.net.2.bias'][0] = 1e4
    _, _, cams, _ = weights.demo_inputs(cfg, N, seed=5)
    cam2world, intr = cams[:, :16].reshape(-1, 4, 4).clone(), cams[:, 16:25].reshape(-1, 3, 3).clone()
    if c['camera'] == 'skewed':                 # skew, fx != fy, cx != cy != 0.5
        intr[:, 0, 0], intr[:, 0, 1], intr[:, 0, 2], intr[:, 1, 1], intr[:, 1, 2] = 4.0, 0.35, 0.46, 4.5, 0.57
    u_c = torch.rand(N, res * res, c['Dc'], 1, generator=g)
    u_f = torch.rand(N * res * res, max(c['Df'], 1), generator=g)
    return opts, planes, sd, cam2world, intr, res, u_c, u_f


def _reference(name):
    opts, planes, sd, cam2world, intr, res, u_c, u_f = _case(name)
    tp = ref_shim.import_reference()
    import training_avatar_texture.volumetric_rendering.ray_sampler as rs
    import training_avatar_texture.volumetric_rendering.renderer as rr
    o, d = rs.RaySampler()(cam2world, intr, res)
    dec = tp.OSGDecoder(32, {'decoder_lr_mul': opts['decoder_lr_mul'], 'decoder_output_dim': 32})
    dec.load_state_dict({k[len('decoder.'):]: v for k, v in sd.items()})
    with ref_shim.injected_sampler_noise(u_c, u_f):
        rgb, depth, wsum = rr.ImportanceRenderer()(planes, dec, o, d, opts)
    return dict(origins=o, dirs=d, rgb=rgb.detach(), depth=depth.detach(), wsum=wsum.detach())


_live = {}


def _ref(name, key):
    def compute():
        if name not in _live:
            _live[name] = _reference(name)
        return _live[name][key]
    return REF.get(f'{name}-{key}', compute)


@pytest.mark.parametrize('name', sorted(CASES))
def test_oracle_render_matches_reference_on_contract_options(name):
    opts, planes, sd, cam2world, intr, res, u_c, u_f = _case(name)
    o, d = orr.ray_sampler(cam2world, intr, res)
    assert range_rel_err(o, _ref(name, 'origins')) <= 1e-6
    assert range_rel_err(d, _ref(name, 'dirs')) <= 1e-6
    rgb, depth, wsum = orr.render(sd, planes, o, d, opts, u_c, u_f)
    assert range_rel_err(rgb, _ref(name, 'rgb')) <= 1e-6
    assert range_rel_err(depth, _ref(name, 'depth')) <= 1e-6
    if name == 'transparent':                   # every weight underflows to 0 in both
        assert torch.equal(wsum, _ref(name, 'wsum')) and not wsum.any()
    else:
        assert range_rel_err(wsum, _ref(name, 'wsum')) <= 1e-6
