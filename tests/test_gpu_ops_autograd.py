"""GPU: gradients of the torch_utils.ops mirror (bias_act, upfirdn2d, conv2d_resample) end to end.  The gradient kernels at their
ABI are tested over every launch configuration by tests/test_gpu_grad_conformance.py.

Truth is oracle.ops under torch.autograd in fp64, on the same inputs rounded as the kernels see them.  Bounds are range-relative
(tests.helpers.range_rel_err) and at most 4x the worst error measured on an H100 80GB HBM3 at a 400 W power limit.  Set
N3D_GRAD_ERRORS=<file> to append every measured error to that file as JSON lines.
"""
import math

import pytest
import torch

from tests.helpers import range_rel_err, record_errors

pytestmark = pytest.mark.gpu

F64 = torch.float64


@pytest.fixture(scope='module')
def ops():
    import next3d_b200.torch_utils.ops as o
    return o


def _g(s):
    return torch.Generator().manual_seed(s)


def _check(case, what, a, ref, bound):
    err = range_rel_err(a.detach().cpu(), ref.detach().cpu())
    record_errors('N3D_GRAD_ERRORS', [{'case': case, 'what': what, 'err': err, 'bound': bound}])
    assert err < bound, (case, what, err, bound)


# ------------------------------------------------------------------------------------------------ bias_act
# fp32: the kernel's derivative formulas in fp32 from the fp32-rounded saved output.  fp16 (looser): dy, the saved y and dx are
# stored in fp16, 2^-11 relative each.
_BA_BOUND = {torch.float32: {'dx': 9e-7, 'db': 9e-7}, torch.float16: {'dx': 2.8e-3, 'db': 2.4e-3}}
_BA_BOUND2 = {torch.float32: {'dx': 6e-7, 'd2x': 1e-6, 'd2b': 1.6e-6, 'd2dy': 9e-7},
              torch.float16: {'dx': 2e-3, 'd2x': 5.9e-3, 'd2b': 5.8e-3, 'd2dy': 3.1e-3}}


def _oracle_grads(x, b, dy, act, gain, clamp, mask):
    """fp64 oracle: dx, db of sum(y * dy) with y = oracle bias_act without the clamp, times the clamp mask."""
    from oracle import ops as oo
    x64 = x.double().requires_grad_()
    b64 = b.double().requires_grad_() if b is not None else None
    y = oo.bias_act(x64, b64, act=act, gain=gain)
    gs = torch.autograd.grad(y, [x64] + ([b64] if b is not None else []), dy.double() * mask)
    return gs[0], (gs[1] if b is not None else None), y.detach()


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('fmt', [torch.contiguous_format, torch.channels_last])
def test_bias_act_first_order(ops, dtype, fmt):
    from oracle import ops as oo
    x = (torch.randn(3, 20, 9, 7, generator=_g(1)) * 2).to(dtype)
    b = torch.randn(20, generator=_g(2)).to(dtype)
    dy = torch.randn(3, 20, 9, 7, generator=_g(3)).to(dtype)
    for act in oo.ACTIVATIONS:
        for with_b in (True, False):
            for gain, clamp in [(None, None), (2.0, 0.75)]:
                case = f'bias_act/{act}/{dtype}/{fmt}/b{int(with_b)}/g{gain}/c{clamp}'
                xg = x.cuda().contiguous(memory_format=fmt).requires_grad_()
                bg = b.cuda().requires_grad_() if with_b else None
                y = ops.bias_act.bias_act(xg, bg, act=act, gain=gain, clamp=clamp)
                assert y.requires_grad and y.is_contiguous(memory_format=fmt)
                grads = torch.autograd.grad(y, [xg] + ([bg] if with_b else []), dy.cuda().contiguous(memory_format=fmt))
                mask = torch.ones(x.shape, dtype=F64)
                if clamp is not None and act != 'linear':
                    # the clamp mask comes from the saved output, compared in fp32 (swish: recomputed in fp32 from x + b, as fp64 here);
                    # 'linear' saves no output, so its gradient is not masked (the reference plugin's behaviour)
                    yk = oo.bias_act(x.double(), b.double() if with_b else None, act=act, gain=gain) if act == 'swish' else y.detach().cpu()
                    yk, c32 = yk.float(), torch.tensor(clamp, dtype=torch.float32)
                    mask = ((yk > -c32) & (yk < c32)).double()
                    assert (mask == 0).any(), case                             # clamped elements are present
                dx64, db64, _ = _oracle_grads(x, b if with_b else None, dy, act, gain, None, mask)
                _check(case, 'dx', grads[0], dx64, _BA_BOUND[dtype]['dx'])
                if with_b:
                    _check(case, 'db', grads[1], db64, _BA_BOUND[dtype]['db'])
    # bias along dim 0 of a 2-D input (FullyConnectedLayer) and along dim 2
    for shape, dim in [((33, 5), 0), ((2, 3, 16, 4), 2)]:
        x2 = torch.randn(*shape, generator=_g(4)).to(dtype)
        b2 = torch.randn(shape[dim], generator=_g(5)).to(dtype)
        dy2 = torch.randn(*shape, generator=_g(6)).to(dtype)
        xg, bg = x2.cuda().requires_grad_(), b2.cuda().requires_grad_()
        dx, db = torch.autograd.grad(ops.bias_act.bias_act(xg, bg, dim=dim, act='lrelu'), [xg, bg], dy2.cuda())
        x64, b64 = x2.double().requires_grad_(), b2.double().requires_grad_()
        dx64, db64 = torch.autograd.grad(oo.bias_act(x64, b64, dim=dim, act='lrelu'), [x64, b64], dy2.double())
        _check(f'bias_act/dim{dim}/{dtype}', 'dx', dx, dx64, _BA_BOUND[dtype]['dx'])
        _check(f'bias_act/dim{dim}/{dtype}', 'db', db, db64, _BA_BOUND[dtype]['db'])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('act', ['tanh', 'sigmoid', 'elu', 'selu', 'softplus', 'swish'])
def test_bias_act_second_order(ops, dtype, act):
    from oracle import ops as oo
    x = (torch.randn(2, 12, 5, 6, generator=_g(7)) * 2).to(dtype)
    b = torch.randn(12, generator=_g(8)).to(dtype)
    dy = torch.randn(2, 12, 5, 6, generator=_g(9)).to(dtype)
    v = torch.randn(2, 12, 5, 6, generator=_g(10)).to(dtype)
    for gain in (None, 0.5):
        case = f'bias_act2/{act}/{dtype}/g{gain}'
        xg, bg, dyg = x.cuda().requires_grad_(), b.cuda().requires_grad_(), dy.cuda().requires_grad_()
        dx, = torch.autograd.grad(ops.bias_act.bias_act(xg, bg, act=act, gain=gain), xg, dyg, create_graph=True)
        d_x, d_b, d_dy = torch.autograd.grad(dx, [xg, bg, dyg], v.cuda())
        x64, b64, dy64 = x.double().requires_grad_(), b.double().requires_grad_(), dy.double().requires_grad_()
        dx64, = torch.autograd.grad(oo.bias_act(x64, b64, act=act, gain=gain), x64, dy64, create_graph=True)
        r_x, r_b, r_dy = torch.autograd.grad(dx64, [x64, b64, dy64], v.double())
        for what, a, r in [('dx', dx, dx64), ('d2x', d_x, r_x), ('d2b', d_b, r_b), ('d2dy', d_dy, r_dy)]:
            _check(case, what, a, r, _BA_BOUND2[dtype][what])


# ------------------------------------------------------------------------------------------------ upfirdn2d
_UFD_BOUND = 5.9e-7


@pytest.mark.parametrize('up,down,pad', [(1, 1, [1, 1, 1, 1]), (2, 1, [2, 1, 2, 1]), (1, 2, [1, 1, 1, 1]), (1, 1, [2, 2, 2, 2]), (2, 2, [3, 0, 1, 2]),
                                        (1, 1, [-1, 0, 0, -1]), (4, 1, [3, 2, 3, 2])])
def test_upfirdn2d_grad(ops, up, down, pad):
    from oracle import ops as oo
    x = torch.randn(2, 6, 13, 10, generator=_g(11))
    f = oo.setup_filter()
    f8 = ops.upfirdn2d.setup_filter([1, 2, 3, 4, 4, 3, 2, 1])
    for ff, flip, gain in [(f, False, up * up), (f8, False, 2.0), (f8, True, 1.0), (oo.setup_filter([1, 2, 7, 1]), True, 3.0)]:
        case = f'upfirdn2d/{up}/{down}/{pad}/{tuple(ff.shape)}/{flip}/{gain}'
        y_ref = oo.upfirdn2d(x.double(), ff.double(), up=up, down=down, padding=pad, flip_filter=flip, gain=gain)
        dy = torch.randn(y_ref.shape, generator=_g(12))
        v = torch.randn(x.shape, generator=_g(13))
        xg, dyg = x.cuda().requires_grad_(), dy.cuda().requires_grad_()
        y = ops.upfirdn2d.upfirdn2d(xg, ff.cuda(), up=up, down=down, padding=pad, flip_filter=flip, gain=gain)
        dx, = torch.autograd.grad(y, xg, dyg, create_graph=True)
        d_dy, = torch.autograd.grad(dx, dyg, v.cuda())                 # second order: the backward of the backward
        x64, dy64 = x.double().requires_grad_(), dy.double().requires_grad_()
        dx64, = torch.autograd.grad(oo.upfirdn2d(x64, ff.double(), up=up, down=down, padding=pad, flip_filter=flip, gain=gain), x64, dy64,
                                    create_graph=True)
        r_dy, = torch.autograd.grad(dx64, dy64, v.double())
        _check(case, 'dx', dx, dx64, _UFD_BOUND)
        _check(case, 'd2', d_dy, r_dy, _UFD_BOUND)
    # filter2d / upsample2d / downsample2d inherit the gradient; a filter gradient is refused
    xg = x[..., :12, :].cuda().requires_grad_()
    for fn, rfn in [(ops.upfirdn2d.upsample2d, oo.upsample2d), (ops.upfirdn2d.downsample2d, oo.downsample2d)]:
        y = fn(xg, f.cuda())
        dy = torch.randn(y.shape, generator=_g(14))
        dx, = torch.autograd.grad(y, xg, dy.cuda())
        x64 = x[..., :12, :].double().requires_grad_()
        dx64, = torch.autograd.grad(rfn(x64, f.double()), x64, dy.double())
        _check(f'{fn.__name__}/{up}/{down}', 'dx', dx, dx64, _UFD_BOUND)
    with pytest.raises(RuntimeError, match='upfirdn2d'):
        ops.upfirdn2d.upfirdn2d(xg, f.cuda().requires_grad_(), up=up, down=down, padding=pad)


# ------------------------------------------------------------------------------------------------ conv2d_resample
# bf16x3 products (2^-16 relative per operand split) summed in fp32 over K = 9 * Cin (dx) or the positions (dw).
_CONV_BOUND = {'dx': 3.8e-5, 'dw': 2.7e-5}


def _conv_case(k, up, down, groups):
    cin_g = 16
    cout_g = 3 if (k == 1 and groups == 1) else 20          # ToRGB's Cout = 3; 20 = a channel tail of the adjoint's Cin
    x = torch.randn(2, cin_g * groups, 12, 12, generator=_g(15))
    w = torch.randn(cout_g * groups, cin_g, k, k, generator=_g(16)) / math.sqrt(cin_g * k * k)
    return x, w


@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('up,down', [(1, 1), (2, 1), (1, 2)])
@pytest.mark.parametrize('groups', [1, 3])
@pytest.mark.parametrize('flip', [True, False])
def test_conv2d_resample_grad(ops, k, up, down, groups, flip):
    from oracle import ops as oo
    case = f'conv/k{k}/up{up}/down{down}/g{groups}/flip{flip}'
    x, w = _conv_case(k, up, down, groups)
    f = oo.setup_filter()
    kw = dict(up=up, down=down, padding=k // 2, groups=groups, flip_weight=flip)
    x64, w64 = x.double().requires_grad_(), w.double().requires_grad_()
    y64 = oo.conv2d_resample(x64, w64, f=f.double(), **kw)
    dy = torch.randn(y64.shape, generator=_g(17))
    dx64, dw64 = torch.autograd.grad(y64, [x64, w64], dy.double())
    conv = ops.conv2d_resample.conv2d_resample

    def run():
        xg, wg = x.cuda().requires_grad_(), w.cuda().requires_grad_()
        y = conv(xg, wg, f=f.cuda(), **kw)
        return torch.autograd.grad(y, [xg, wg], dy.cuda())

    dx, dw = run()
    _check(case, 'dx', dx, dx64, _CONV_BOUND['dx'])
    _check(case, 'dw', dw, dw64, _CONV_BOUND['dw'])
    dx2, dw2 = run()
    assert torch.equal(dx, dx2) and torch.equal(dw, dw2), case        # bit-identical from run to run
    # no_weight_gradients(): w.grad stays None, x.grad is unchanged
    xg, wg = x.cuda().requires_grad_(), w.cuda().requires_grad_()
    with ops.conv2d_gradfix.no_weight_gradients():
        conv(xg, wg, f=f.cuda(), **kw).backward(dy.cuda())
    assert wg.grad is None and torch.equal(xg.grad, dx)
    # second order is refused, naming the op
    y = conv(x.cuda().requires_grad_(), w.cuda().requires_grad_(), f=f.cuda(), **kw)
    with pytest.raises(RuntimeError, match='conv2d_resample'):
        y.backward(dy.cuda(), create_graph=True)
    # without grad the forward is the plain path, bit for bit
    with torch.no_grad():
        y0 = conv(x.cuda(), w.cuda(), f=f.cuda(), **kw)
    assert torch.equal(y0, conv(x.cuda().requires_grad_(), w.cuda(), f=f.cuda(), **kw).detach())


def _fir_plans(N, cin, cout, H, W, up, down, sms):
    """FIR launches of a 3x3 conv2d_resample call (forward, backward) -> {direction: plan} (tests/test_gpu_fir_conformance.py)."""
    from tests.test_gpu_fir_conformance import fir_down_plan, fir_up_plan
    cpad = -(-cout // 8) * 8                                    # the input gradient's channels, zero-padded to a multiple of 8
    if up == 2:
        return {'forward fir-up': fir_up_plan(N, 2 * H, 2 * W, cout, sms), 'backward fir-down': fir_down_plan(N, 2 * H, 2 * W, cpad, sms)}
    if down == 2:
        return {'forward fir-down': fir_down_plan(N, H, W, cin, sms), 'backward fir-up': fir_up_plan(N, H, W, cin, sms)}
    return {}


# Beyond 12 x 12: odd and non-square sizes, batch 1 and 3, 8 and 512 channels, and layers whose FIR passes take the streamed kernels
# (`streamed`: the directions that must, according to the launch rules).
_CONV_LARGE = [
    dict(name='up_7x13_n3_c8', N=3, cin=8, cout=8, H=7, W=13, up=2, down=1, flip=False, streamed=()),
    dict(name='same_10x18_n1_c512', N=1, cin=512, cout=512, H=10, W=18, up=1, down=1, flip=True, streamed=()),
    dict(name='down_10x18_n3_c512', N=3, cin=512, cout=8, H=10, W=18, up=1, down=2, flip=True, streamed=()),
    dict(name='up_192x176_streamed', N=1, cin=8, cout=64, H=192, W=176, up=2, down=1, flip=True,
         streamed=('forward fir-up', 'backward fir-down')),
    dict(name='down_384x352_streamed', N=1, cin=64, cout=16, H=384, W=352, up=1, down=2, flip=False,
         streamed=('forward fir-down', 'backward fir-up')),
]


@pytest.mark.parametrize('c', _CONV_LARGE, ids=[c['name'] for c in _CONV_LARGE])
def test_conv2d_resample_grad_large(ops, c, monkeypatch):
    """Forward, dx and dw against oracle.ops under fp64 autograd on the device; where a FIR pass streams, everything is bit-identical
    under N3D_FIR_STREAM=0 (the register-tiled FIR kernels)."""
    from oracle import ops as oo
    monkeypatch.delenv('N3D_FIR_STREAM', raising=False)
    case = f'conv_large/{c["name"]}'
    plans = _fir_plans(c['N'], c['cin'], c['cout'], c['H'], c['W'], c['up'], c['down'], torch.cuda.get_device_properties(0).multi_processor_count)
    assert {d for d, p in plans.items() if p['streamed']} == set(c['streamed']), (case, plans)
    x = torch.randn(c['N'], c['cin'], c['H'], c['W'], generator=_g(18)).cuda()
    w = (torch.randn(c['cout'], c['cin'], 3, 3, generator=_g(19)) / math.sqrt(c['cin'] * 9)).cuda()
    f = oo.setup_filter().cuda()
    kw = dict(up=c['up'], down=c['down'], padding=1, flip_weight=c['flip'])
    x64, w64 = x.double().requires_grad_(), w.double().requires_grad_()
    y64 = oo.conv2d_resample(x64, w64, f=f.double(), **kw)
    dy = torch.randn(y64.shape, generator=_g(20)).cuda()
    dx64, dw64 = torch.autograd.grad(y64, [x64, w64], dy.double())
    y64 = y64.detach()

    def run():
        xg, wg = x.clone().requires_grad_(), w.clone().requires_grad_()
        y = ops.conv2d_resample.conv2d_resample(xg, wg, f=f, **kw)
        return (y.detach(),) + torch.autograd.grad(y, [xg, wg], dy)

    y, dx, dw = run()
    _check(case, 'y', y, y64, 5e-5)
    _check(case, 'dx', dx, dx64, _CONV_BOUND['dx'])
    _check(case, 'dw', dw, dw64, _CONV_BOUND['dw'])
    if c['streamed']:
        monkeypatch.setenv('N3D_FIR_STREAM', '0')
        for a, b in zip((y, dx, dw), run()):
            assert torch.equal(a, b), case


# ------------------------------------------------------------------------------------------------ end to end
def _synthesis_block(bias_act, conv2d_resample, upsample2d, fma, ws, P, x, img, f, noise):
    """A StyleGAN2 synthesis block restated (networks_stylegan2.py:280-380, fused modconv): up-sampling conv0, conv1, ToRGB and the
    FIR-upsampled skip image, with styles from ws, demodulation, noise via fma and bias_act."""
    N = ws.shape[0]

    def affine(w_i, A, b):
        return bias_act(w_i @ (A / math.sqrt(A.shape[1])).t(), b)

    def modconv(x, weight, styles, up, demod, act_b, noise_map, act, gain=None):
        cout, cin, kh, kw = weight.shape
        wgt = weight[None] * styles.reshape(N, 1, cin, 1, 1)
        if demod:
            d = (wgt.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()
            wgt = wgt * d.reshape(N, cout, 1, 1, 1)
        y = conv2d_resample(x.reshape(1, N * cin, *x.shape[2:]), wgt.reshape(N * cout, cin, kh, kw), f=f, up=up, padding=kh // 2, groups=N,
                            flip_weight=(up == 1))
        y = y.reshape(N, cout, *y.shape[2:])
        if noise_map is not None:
            y = fma(y, torch.ones_like(y[:1, :1]), noise_map * P['noise_strength'])
        return bias_act(y, act_b, act=act, gain=gain)

    s0 = affine(ws[:, 0], P['A0'], P['Ab0'])
    x = modconv(x, P['W0'], s0, 2, True, P['b0'], noise, 'lrelu')
    s1 = affine(ws[:, 1], P['A1'], P['Ab1'])
    x = modconv(x, P['W1'], s1, 1, True, P['b1'], None, 'lrelu')
    s2 = affine(ws[:, 2], P['A2'], P['Ab2']) / math.sqrt(P['W2'].shape[1])
    rgb = modconv(x, P['W2'], s2, 1, False, P['b2'], None, 'linear')
    return upsample2d(img, f) + rgb


def test_synthesis_block_gradients(ops):
    from oracle import ops as oo
    gen = _g(20)
    N, C0, C1, R = 2, 32, 24, 8
    P = {'A0': torch.randn(C0, 64, generator=gen), 'Ab0': torch.ones(C0), 'W0': torch.randn(C1, C0, 3, 3, generator=gen) * 0.2,
         'b0': torch.randn(C1, generator=gen) * 0.1, 'A1': torch.randn(C1, 64, generator=gen), 'Ab1': torch.ones(C1),
         'W1': torch.randn(C1, C1, 3, 3, generator=gen) * 0.2, 'b1': torch.randn(C1, generator=gen) * 0.1,
         'A2': torch.randn(C1, 64, generator=gen), 'Ab2': torch.ones(C1), 'W2': torch.randn(3, C1, 1, 1, generator=gen) * 0.2,
         'b2': torch.randn(3, generator=gen) * 0.1, 'noise_strength': torch.tensor(0.3)}
    ws = torch.randn(N, 3, 64, generator=gen)
    x = torch.randn(N, C0, R, R, generator=gen)
    img = torch.randn(N, 3, R, R, generator=gen)
    noise = torch.randn(N, 1, 2 * R, 2 * R, generator=gen)
    dout = torch.randn(N, 3, 2 * R, 2 * R, generator=gen)
    f = oo.setup_filter()
    names = ['W0', 'b0', 'W1', 'b1', 'W2', 'b2', 'A0', 'A1', 'A2', 'Ab0', 'Ab1', 'Ab2']

    def grads(dev, dtype, bias_act, conv, up2d, fma):
        Pd = {k: v.to(dev, dtype).requires_grad_(k in names) for k, v in P.items()}
        wsd = ws.to(dev, dtype).requires_grad_()
        out = _synthesis_block(bias_act, conv, up2d, fma, wsd, Pd, x.to(dev, dtype), img.to(dev, dtype), f.to(dev, dtype), noise.to(dev, dtype))
        return torch.autograd.grad(out, [wsd] + [Pd[k] for k in names], dout.to(dev, dtype))

    ours = grads('cuda', torch.float32, ops.bias_act.bias_act, ops.conv2d_resample.conv2d_resample, ops.upfirdn2d.upsample2d, ops.fma.fma)
    ref = grads('cpu', F64, lambda x, b=None, act='linear', gain=None: oo.bias_act(x, b, act=act, gain=gain),
                lambda x, w, f, up, padding, groups, flip_weight: oo.conv2d_resample(x, w, f=f, up=up, padding=padding, groups=groups,
                                                                                        flip_weight=flip_weight),
                oo.upsample2d, lambda a, b, c: a * b + c)
    for name, a, r in zip(['ws'] + names, ours, ref):
        _check('synthesis_block', name, a, r, 7e-5)


# ------------------------------------------------------------------------------------------------ filtered_lrelu
def test_filtered_lrelu_refuses_grad(ops):
    from oracle import ops as oo
    x = torch.randn(2, 5, 11, 9, generator=_g(21)).cuda()
    b = torch.randn(5, generator=_g(22)).cuda()
    f = oo.setup_filter().cuda()
    kw = dict(fu=f, fd=f, up=2, down=2, padding=3)
    y0 = ops.filtered_lrelu.filtered_lrelu(x, b=b, **kw)
    for xr, br in [(True, False), (False, True)]:
        with pytest.raises(RuntimeError, match='filtered_lrelu.*not implemented'):
            ops.filtered_lrelu.filtered_lrelu(x.clone().requires_grad_(xr), b=b.clone().requires_grad_(br), **kw)
    with torch.no_grad():
        assert torch.equal(ops.filtered_lrelu.filtered_lrelu(x.clone().requires_grad_(), b=b, **kw), y0)
