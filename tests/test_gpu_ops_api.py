"""GPU: the torch_utils.ops mirror (public op API of the reference) against the CPU oracle, same call signatures."""
import math

import pytest
import torch

from tests.helpers import range_rel_err

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ops():
    import next3d_b200.torch_utils.ops as o
    return o


def _g(s):
    return torch.Generator().manual_seed(s)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('fmt', [torch.contiguous_format, torch.channels_last])
def test_bias_act(ops, dtype, fmt):
    from oracle import ops as oo
    x = (torch.randn(3, 20, 9, 7, generator=_g(1)) * 2)
    b = torch.randn(20, generator=_g(2))
    for act in oo.ACTIVATIONS:
        for gain, clamp in [(None, None), (0.5, 0.7)]:
            ref = oo.bias_act(x.to(dtype).float(), b.to(dtype).float(), act=act, gain=gain, clamp=clamp)
            xd = x.to(dtype).cuda().contiguous(memory_format=fmt)
            y = ops.bias_act.bias_act(xd, b.to(dtype).cuda(), act=act, gain=gain, clamp=clamp)
            assert y.dtype == dtype and y.shape == x.shape and y.is_contiguous(memory_format=fmt)
            assert range_rel_err(y.float().cpu(), ref) < (2e-3 if dtype == torch.float16 else 2e-6), act
    # bias along another dim, no bias, 2-D input (FullyConnectedLayer path)
    x2 = torch.randn(5, 33, generator=_g(3))
    b2 = torch.randn(33, generator=_g(4))
    assert range_rel_err(ops.bias_act.bias_act(x2.cuda(), b2.cuda(), act='lrelu').cpu(), oo.bias_act(x2, b2, act='lrelu')) < 2e-6
    assert range_rel_err(ops.bias_act.bias_act(x2.cuda(), act='sigmoid').cpu(), oo.bias_act(x2, act='sigmoid')) < 2e-6
    with pytest.raises(RuntimeError):
        ops.bias_act.bias_act(x2, b2)                                   # CPU tensor with impl='cuda': loud failure, no fallback
    assert torch.equal(ops.bias_act.bias_act(x2, b2, act='lrelu', impl='ref'), oo.bias_act(x2, b2, act='lrelu'))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('fmt', [torch.contiguous_format, torch.channels_last])
@pytest.mark.parametrize('offset', [1, 2, 3])
def test_bias_act_on_views_at_any_storage_offset(ops, dtype, fmt, offset):
    """Dense views that start 1-3 elements into their storage (not aligned for 4-element vector accesses), numel % 4 in {0..3}."""
    from oracle import ops as oo
    b = torch.randn(5, generator=_g(15)).to(dtype)
    for shape in [(2, 5, 2, 7), (1, 5, 3, 7), (2, 5, 3, 7), (1, 5, 1, 7)]:          # numel % 4 = 0, 1, 2, 3
        N, Cc, H, W = shape
        strides = (Cc * H * W, H * W, W, 1) if fmt == torch.contiguous_format else (H * W * Cc, 1, W * Cc, Cc)
        buf = (torch.randn(N * Cc * H * W + 8, generator=_g(16)) * 2).to(dtype).cuda()
        x = buf.as_strided(shape, strides, offset)
        assert x.is_contiguous(memory_format=fmt) and x.data_ptr() % (4 * x.element_size()) != 0
        y = ops.bias_act.bias_act(x, b.cuda(), act='lrelu', clamp=1.5)
        ref = oo.bias_act(x.cpu().float(), b.float(), act='lrelu', clamp=1.5)
        assert y.is_contiguous(memory_format=fmt)
        assert range_rel_err(y.float().cpu(), ref) < (2e-3 if dtype == torch.float16 else 2e-6), (shape, offset)


@pytest.mark.parametrize('up,down,pad', [(1, 1, [1, 1, 1, 1]), (2, 1, [2, 1, 2, 1]), (1, 2, [1, 1, 1, 1]), (1, 1, [2, 2, 2, 2]), (2, 2, [3, 0, 1, 2]),
                                        (1, 1, [-1, 0, 0, -1]), (4, 1, [3, 2, 3, 2])])
def test_upfirdn2d(ops, up, down, pad):
    from oracle import ops as oo
    x = torch.randn(2, 6, 13, 10, generator=_g(5))
    f = oo.setup_filter()
    assert torch.equal(ops.upfirdn2d.setup_filter([1, 3, 3, 1]), f)
    ref = oo.upfirdn2d(x, f, up=up, down=down, padding=pad, gain=up * up)
    for fmt in (torch.contiguous_format, torch.channels_last):
        y = ops.upfirdn2d.upfirdn2d(x.cuda().contiguous(memory_format=fmt), f.cuda(), up=up, down=down, padding=pad, gain=up * up)
        assert range_rel_err(y.cpu(), ref) < 2e-6
    assert range_rel_err(ops.upfirdn2d.upsample2d(x.cuda(), f.cuda()).cpu(), oo.upsample2d(x, f)) < 2e-6
    assert range_rel_err(ops.upfirdn2d.downsample2d(x[..., :12, :].cuda(), f.cuda()).cpu(), oo.downsample2d(x[..., :12, :], f)) < 2e-6
    # separable 8-tap filter takes the two-pass route
    f8 = ops.upfirdn2d.setup_filter([1, 2, 3, 4, 4, 3, 2, 1])
    assert f8.ndim == 1
    r8 = ops.upfirdn2d.upfirdn2d(x, f8, padding=4, gain=2.0, impl='ref')
    assert range_rel_err(ops.upfirdn2d.upfirdn2d(x.cuda(), f8.cuda(), padding=4, gain=2.0).cpu(), r8) < 2e-6


@pytest.mark.parametrize('k,up,down,flip,groups', [(3, 1, 1, True, 1), (3, 2, 1, False, 1), (3, 1, 2, True, 1), (1, 1, 1, True, 1), (1, 2, 1, True, 1),
                                                  (3, 2, 1, False, 2), (3, 1, 1, True, 3)])
def test_conv2d_resample(ops, k, up, down, flip, groups):
    from oracle import ops as oo
    cin_g, cout_g = 16, 24
    x = torch.randn(2, cin_g * groups, 12, 12, generator=_g(6))
    w = torch.randn(cout_g * groups, cin_g, k, k, generator=_g(7)) / math.sqrt(cin_g * k * k)
    f = oo.setup_filter()
    ref = oo.conv2d_resample(x, w, f=f, up=up, down=down, padding=k // 2, groups=groups, flip_weight=flip)
    y = ops.conv2d_resample.conv2d_resample(x.cuda(), w.cuda(), f=f.cuda(), up=up, down=down, padding=k // 2, groups=groups, flip_weight=flip)
    assert y.shape == ref.shape and y.is_contiguous()
    assert range_rel_err(y.cpu(), ref) < 5e-5
    with pytest.raises(RuntimeError):
        ops.conv2d_resample.conv2d_resample(x.cuda(), torch.randn(8, cin_g * groups, 5, 5).cuda(), padding=2)


@pytest.mark.parametrize('N,cin,cout,H,W,up,down,flip', [(3, 8, 8, 7, 13, 2, 1, False), (1, 512, 512, 10, 18, 1, 1, True),
                                                       (3, 512, 8, 10, 18, 1, 2, True), (1, 8, 512, 7, 13, 2, 1, True)])
def test_conv2d_resample_odd_sizes(ops, N, cin, cout, H, W, up, down, flip):
    """Non-square and odd sizes, batch 1 and 3, 8 and 512 channels, against oracle.ops in fp64 on the device."""
    from oracle import ops as oo
    x = torch.randn(N, cin, H, W, generator=_g(17)).cuda()
    w = (torch.randn(cout, cin, 3, 3, generator=_g(18)) / math.sqrt(cin * 9)).cuda()
    f = oo.setup_filter().cuda()
    kw = dict(up=up, down=down, padding=1, flip_weight=flip)
    ref = oo.conv2d_resample(x.double(), w.double(), f=f.double(), **kw)
    y = ops.conv2d_resample.conv2d_resample(x, w, f=f, **kw)
    assert y.shape == ref.shape
    assert range_rel_err(y, ref) < 5e-5


def test_filtered_lrelu(ops):
    from oracle import ops as oo
    x = torch.randn(2, 5, 11, 9, generator=_g(8))
    b = torch.randn(5, generator=_g(9))
    f = oo.setup_filter()
    for up, down, pad, clamp in [(2, 2, 3, None), (1, 1, [1, 2, 1, 2], 0.8), (2, 1, [2, 1, 2, 1], None)]:
        ref = oo.filtered_lrelu(x, fu=f, fd=f, b=b, up=up, down=down, padding=pad, clamp=clamp)
        y = ops.filtered_lrelu.filtered_lrelu(x.cuda(), fu=f.cuda(), fd=f.cuda(), b=b.cuda(), up=up, down=down, padding=pad, clamp=clamp)
        assert range_rel_err(y.cpu(), ref) < 3e-6
    assert torch.equal(ops.filtered_lrelu.filtered_lrelu(x, fu=f, fd=f, b=b, up=2, down=2, padding=3, impl='ref'),
                       oo.filtered_lrelu(x, fu=f, fd=f, b=b, up=2, down=2, padding=3))


def test_small_shims(ops):
    a, b, c = (torch.randn(4, 5, generator=_g(i)).cuda() for i in (10, 11, 12))
    assert torch.allclose(ops.fma.fma(a, b, c), a * b + c)
    inp = torch.randn(1, 3, 8, 8, generator=_g(13)).cuda()
    grid = (torch.rand(1, 4, 4, 2, generator=_g(14)) * 2 - 1).cuda()
    assert torch.equal(ops.grid_sample_gradfix.grid_sample(inp, grid),
                       torch.nn.functional.grid_sample(inp, grid, mode='bilinear', padding_mode='zeros', align_corners=False))
    assert hasattr(ops.conv2d_gradfix, 'no_weight_gradients') and ops.bias_act.activation_funcs['lrelu'].def_gain == math.sqrt(2)
