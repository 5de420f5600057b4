"""CPU: pin the oracle restatement against the reference's OWN code.  What the reference computed on these seeded inputs is
stored in tests/golden/reference_ops.npz and reference_synthesis.npz (tests.helpers.ReferenceVectors; N3D_RECORD_REFERENCE=1
recomputes it where the reference can be imported)."""
import numpy as np
import pytest
import torch

from next3d_b200 import config, weights
from oracle import ops as oo, generator as og, rasterize as orast, ref_shim
from tests.helpers import ReferenceVectors

REF = ReferenceVectors('reference_ops')


def ref():
    """The reference's modules (only called while recording)."""
    ref_shim.import_reference()
    from torch_utils.ops import bias_act, upfirdn2d, conv2d_resample, filtered_lrelu
    import training_avatar_texture.networks_stylegan2 as sg2
    import training_avatar_texture.volumetric_rendering.renderer as rr
    return dict(bias_act=bias_act, upfirdn2d=upfirdn2d, conv2d_resample=conv2d_resample, filtered_lrelu=filtered_lrelu,
                sg2=sg2, rr=rr)


def test_bias_act_all_activations():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(3, 7, 5, 6, generator=g) * 3
    b = torch.randn(7, generator=g)
    for act in oo.ACTIVATIONS:
        for gain, clamp in [(None, None), (0.7, 0.5)]:
            a = REF.get(f'bias_act-{act}-{gain}-{clamp}', lambda: ref()['bias_act'].bias_act(x, b, act=act, gain=gain, clamp=clamp, impl='ref'))
            o = oo.bias_act(x, b, act=act, gain=gain, clamp=clamp)
            assert torch.equal(a, o), act


@pytest.mark.parametrize('up,down,pad', [(1, 1, [1, 1, 1, 1]), (2, 1, [2, 1, 2, 1]), (1, 2, [1, 1, 1, 1]),
                                        (1, 1, [2, 2, 2, 2]), (2, 2, [3, 0, 1, 2]), (1, 1, [-1, 0, 0, -1])])
def test_upfirdn2d(up, down, pad):
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 5, 9, 12, generator=g)
    f = REF.get('setup_filter', lambda: ref()['upfirdn2d'].setup_filter([1, 3, 3, 1]))
    assert torch.equal(f, oo.setup_filter())
    key = f'upfirdn2d-{up}-{down}-' + '_'.join(str(p) for p in pad)
    a = REF.get(key, lambda: ref()['upfirdn2d'].upfirdn2d(x, f, up=up, down=down, padding=pad, gain=up * up, impl='ref'))
    o = oo.upfirdn2d(x, oo.setup_filter(), up=up, down=down, padding=pad, gain=up * up)
    assert torch.equal(a, o)
    assert torch.equal(REF.get(key + '-up2', lambda: ref()['upfirdn2d'].upsample2d(x, f, impl='ref')), oo.upsample2d(x, f))
    assert torch.equal(REF.get(key + '-down2', lambda: ref()['upfirdn2d'].downsample2d(x[..., :8, :], f, impl='ref')),
                       oo.downsample2d(x[..., :8, :], f))


@pytest.mark.parametrize('k,up,down,flip', [(3, 2, 1, False), (3, 1, 2, True), (3, 1, 1, True), (1, 1, 1, True)])
def test_conv2d_resample(k, up, down, flip):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 6, 8, 8, generator=g)
    w = torch.randn(4, 6, k, k, generator=g)
    f = oo.setup_filter()
    a = REF.get(f'conv2d_resample-{k}-{up}-{down}-{flip}',
                lambda: ref()['conv2d_resample'].conv2d_resample(x, w, f=f, up=up, down=down, padding=k // 2, flip_weight=flip))
    o = oo.conv2d_resample(x, w, f=f, up=up, down=down, padding=k // 2, flip_weight=flip)
    assert torch.equal(a, o)


def test_modulated_conv2d():
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 6, 8, 8, generator=g)
    w = torch.randn(4, 6, 3, 3, generator=g)
    s = torch.randn(2, 6, generator=g)
    noise = torch.randn(16, 16, generator=g)
    f = oo.setup_filter()
    a = REF.get('modulated_conv2d', lambda: ref()['sg2'].modulated_conv2d(x, w, s, noise=noise, up=2, padding=1, resample_filter=f,
                                                                        flip_weight=False))
    o = oo.modulated_conv2d(x, w, s, noise=noise, up=2, padding=1, resample_filter=f, flip_weight=False)
    assert torch.equal(a, o)


def test_filtered_lrelu():
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, 10, 10, generator=g)
    b = torch.randn(3, generator=g)
    fu = REF.get('setup_filter', lambda: ref()['upfirdn2d'].setup_filter([1, 3, 3, 1]))
    a = REF.get('filtered_lrelu', lambda: ref()['filtered_lrelu'].filtered_lrelu(x, fu=fu, fd=fu, b=b, up=2, down=2, padding=3, impl='ref'))
    o = oo.filtered_lrelu(x, fu=fu, fd=fu, b=b, up=2, down=2, padding=3)
    assert torch.equal(a, o)


def _edge_filters():
    """Filters of the edge cases: the 4-tap filter, a non-square 3x5 one with unequal taps, 1-D taps of length 4 (raw) and 8 (the
    reference's separable setup_filter)."""
    g = torch.Generator().manual_seed(6)
    f35 = torch.rand(3, 5, generator=g) + 0.1
    return {'f4': oo.setup_filter(), 'f35': f35 / f35.sum(), 'f1d4': torch.tensor([1.0, 2.0, 5.0, 3.0]) / 11,
            'f1d8': REF.get('setup_filter8', lambda: ref()['upfirdn2d'].setup_filter([1, 2, 3, 4, 4, 3, 2, 1]))}


@pytest.mark.parametrize('name,f,up,down,pad,flip,gain', [
    ('up3x2', 'f4', [3, 2], 1, [2, 1, 1, 2], False, 6.0),
    ('down3x2_nonsquare', 'f35', 1, [3, 2], [1, 1, 2, 0], False, 1.0),
    ('updown_1d8', 'f1d8', [2, 3], [2, 1], [3, 4, 4, 3], False, 2.0),
    ('flip_negpad_nonsquare', 'f35', 1, 1, [-1, 2, 0, -2], True, 1.0),
    ('flip_1d4_up2', 'f1d4', 2, 1, [-2, 3, 1, -1], True, 4.0),
    ('negpad_up2_down2', 'f4', 2, 2, [0, -3, -2, 1], False, 4.0),
])
def test_upfirdn2d_edges(name, f, up, down, pad, flip, gain):
    """Asymmetric [x, y] factors, non-square and 1-D filters, flip_filter and negative padding, against the reference's _upfirdn2d_ref."""
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 3, 9, 11, generator=g)
    fv = _edge_filters()[f]
    a = REF.get(f'upfirdn2d_edge-{name}', lambda: ref()['upfirdn2d']._upfirdn2d_ref(x, fv, up=up, down=down, padding=pad, flip_filter=flip, gain=gain))
    assert torch.equal(a, oo.upfirdn2d(x, fv, up=up, down=down, padding=pad, flip_filter=flip, gain=gain))


@pytest.mark.parametrize('name,fu,fd,up,down,pad,flip,clamp', [
    ('fu_none_up2', None, 'f4', 2, 1, [1, 2, 1, 2], False, None),
    ('fd_none_up2_down2', 'f4', None, 2, 2, [2, 1, 2, 1], False, None),
    ('both_none_up2', None, None, 2, 1, 0, False, 0.6),
    ('fu_none_up2_flip', None, 'f35', 2, 2, [1, 0, 2, 1], True, None),
    ('1d_up2_down2_flip', 'f1d8', 'f1d8', 2, 2, [6, 5, 6, 5], True, 0.5),
    ('1d4_up2', 'f1d4', 'f1d4', 2, 1, [3, 2, 3, 2], False, None),
])
def test_filtered_lrelu_edges(name, fu, fd, up, down, pad, flip, clamp):
    """The identity filters (fu / fd = None) at up 2, 1-D filters and flip_filter, against the reference's _filtered_lrelu_ref."""
    g = torch.Generator().manual_seed(8)
    x = torch.randn(2, 3, 10, 9, generator=g)
    b = torch.randn(3, generator=g)
    fs = _edge_filters()
    fu, fd = (fs[k] if k else None for k in (fu, fd))
    kw = dict(fu=fu, fd=fd, b=b, up=up, down=down, padding=pad, flip_filter=flip, clamp=clamp)
    a = REF.get(f'filtered_lrelu_edge-{name}', lambda: ref()['filtered_lrelu']._filtered_lrelu_ref(x, **kw))
    assert torch.equal(a, oo.filtered_lrelu(x, **kw))


def test_fill_mouth_vs_cv2():
    """Our BFS restatement == the reference's cv2.floodFill-based fill_mouth, including fractional alphas."""
    g = torch.Generator().manual_seed(5)
    a = torch.zeros(3, 1, 64, 64)
    a[:, :, 10:50, 12:52] = 1.0
    a[0, :, 25:30, 20:40] = 0.0                      # hole
    a[1, :, 20:24, 20:24] = 0.5                      # interior fractional patch
    a[1, :, 40:44, 30:34] = 0.0
    a[2, :, :5, :5] = 1.0                            # corner covered
    a[2, :, 30:33, 30:36] = 0.0
    a = (a + torch.nn.functional.avg_pool2d(a, 3, 1, 1)) / 2   # fractional edges
    assert torch.equal(REF.get('fill_mouth', lambda: ref()['rr'].fill_mouth(a)), og.fill_mouth(a))


def test_full_synthesis_bit_exact():
    """Whole synthesis, oracle vs reference.  Stored: ws, image_raw, image_depth in full; image every 4th pixel (the stored file stays
    under 1 MB) and the full image's max |value|, so the tolerance is the same as against the live reference."""
    store = ReferenceVectors('reference_synthesis')
    cfg = config.tiny_config(512)
    sd = weights.make_state_dict(cfg, seed=3)
    z, c_cond, c_cam, v = weights.demo_inputs(cfg, 2, seed=3, jitter=1e-4)
    u_c, u_f = weights.sampler_noise(cfg, 2, seed=3)
    live = {}

    def reference_run():
        G = ref_shim.build_reference_generator(cfg)
        G.load_state_dict(sd)
        with torch.no_grad():
            ws_r = G.mapping(z, c_cond, truncation_psi=0.7, truncation_cutoff=14)
            with ref_shim.injected_sampler_noise(u_c, u_f):
                live.update(G.synthesis(ws_r, c_cam, v, noise_mode='const'), ws=ws_r)
        return live

    ws_r = store.get('ws', lambda: reference_run()['ws'])
    r = {k: store.get(k, lambda k=k: live[k]) for k in ('image_raw', 'image_depth')}
    r['image'] = store.get('image_s4', lambda: live['image'][..., ::4, ::4])
    absmax = {k: float(store.get(f'{k}_absmax', lambda k=k: live[k].abs().max())) for k in ('image', 'image_raw', 'image_depth')}
    with torch.no_grad():
        ws = og.mapping(sd, cfg, z, c_cond, 0.7, 14)
        assert torch.equal(ws, ws_r)
        o = og.synthesis(sd, cfg, ws, c_cam, v, u_c, u_f)
    o['image'] = o['image'][..., ::4, ::4]
    for k in ('image', 'image_raw', 'image_depth'):
        assert (o[k] - r[k]).abs().max().item() <= 1e-6 * absmax[k], k


def test_view_transform_is_the_blas_fma_chain():
    """oracle.generator._bmm3_fma (explicit k = 0,1,2 fused chain, float64-emulated) == torch.bmm bit for bit: pins the summation
    order the reference's bmm (renderer.py:505-514) takes on this machine, which the CUDA transform kernel reproduces."""
    g = torch.Generator().manual_seed(0)
    p = torch.randn(3, 5023, 3, generator=g)
    R = torch.randn(3, 3, 3, generator=g)
    assert torch.equal(og._bmm3_fma(p, R), torch.bmm(p, R))
    for view in ((0, 0, 0), (0, 90, 0), (0, -90, 0), (90, 0, 0)):
        Rv = og.angle2matrix(torch.tensor(view, dtype=torch.float32))[None].expand(3, -1, -1)
        assert torch.equal(og._bmm3_fma(p, Rv), torch.bmm(p, Rv))
