"""CPU oracle: the op layer (fp32 torch restatements).  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Restates, in plain fp32 torch ops on CPU tensors:
  bias_act          torch_utils/ops/bias_act.py:93-122 (_bias_act_ref) + activation table :23-33
  upfirdn2d         torch_utils/ops/upfirdn2d.py:169-213 (_upfirdn2d_ref), setup_filter :72-116,
                    upsample2d :315-350, downsample2d :354-389
  conv2d_resample   torch_utils/ops/conv2d_resample.py:48-143
  modulated_conv2d  training_avatar_texture/networks_stylegan2.py:34-91 (fused, inference path)
  filtered_lrelu    torch_utils/ops/filtered_lrelu.py:123-155 (_filtered_lrelu_ref)
Pinned against the reference's own functions by tests/test_oracle_vs_reference.py.
"""
import math

import torch
import torch.nn.functional as F

SQRT2 = math.sqrt(2.0)

# name -> (function, default alpha, default gain)            bias_act.py:23-33
ACTIVATIONS = {
    'linear': (lambda x, a: x, 0.0, 1.0),
    'relu': (lambda x, a: F.relu(x), 0.0, SQRT2),
    'lrelu': (lambda x, a: F.leaky_relu(x, a), 0.2, SQRT2),
    'tanh': (lambda x, a: torch.tanh(x), 0.0, 1.0),
    'sigmoid': (lambda x, a: torch.sigmoid(x), 0.0, 1.0),
    'elu': (lambda x, a: F.elu(x), 0.0, 1.0),
    'selu': (lambda x, a: F.selu(x), 0.0, 1.0),
    'softplus': (lambda x, a: F.softplus(x), 0.0, 1.0),
    'swish': (lambda x, a: torch.sigmoid(x) * x, 0.0, SQRT2),
}


def bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None):
    fn, def_alpha, def_gain = ACTIVATIONS[act]
    alpha = def_alpha if alpha is None else float(alpha)
    gain = def_gain if gain is None else float(gain)
    if b is not None:
        shape = [1] * x.ndim
        shape[dim] = -1
        x = x + b.reshape(shape)
    x = fn(x, alpha)
    if gain != 1:
        x = x * gain
    if clamp is not None and clamp >= 0:
        x = x.clamp(-clamp, clamp)
    return x


def setup_filter(taps=(1, 3, 3, 1), gain=1.0):
    """Normalised non-separable FIR (outer product for < 8 taps), upfirdn2d.py:101-111."""
    f = torch.as_tensor(taps, dtype=torch.float32)
    if f.ndim == 1:
        f = torch.outer(f, f)
    f = f / f.sum()
    return f * gain


def _pad4(padding):
    if isinstance(padding, int):
        return padding, padding, padding, padding
    if len(padding) == 2:
        return padding[0], padding[0], padding[1], padding[1]
    return tuple(padding)


def _scaling2(s):
    """An up / down factor as (x, y): an int or an [x, y] pair, upfirdn2d.py:37-44."""
    return (s, s) if isinstance(s, int) else tuple(s)


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1.0):
    """zero-insert upsample -> pad/crop -> correlate with the flipped filter -> decimate.  up / down: an int or an [x, y] pair."""
    N, C, H, W = x.shape
    upx, upy = _scaling2(up)
    downx, downy = _scaling2(down)
    px0, px1, py0, py1 = _pad4(padding)
    if f is None:
        f = torch.ones(1, 1, dtype=torch.float32, device=x.device)
    if upx > 1 or upy > 1:
        z = x.new_zeros(N, C, H, upy, W, upx)
        z[:, :, :, 0, :, 0] = x
        x = z.reshape(N, C, H * upy, W * upx)
    x = F.pad(x, [max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)])
    x = x[:, :, max(-py0, 0): x.shape[2] - max(-py1, 0), max(-px0, 0): x.shape[3] - max(-px1, 0)]
    f = f.to(x.dtype) * (gain ** (f.ndim / 2))
    if not flip_filter:
        f = f.flip(list(range(f.ndim)))
    if f.ndim == 2:
        x = F.conv2d(x, f[None, None].repeat(C, 1, 1, 1), groups=C)
    else:
        x = F.conv2d(x, f[None, None, None, :].repeat(C, 1, 1, 1), groups=C)
        x = F.conv2d(x, f[None, None, :, None].repeat(C, 1, 1, 1), groups=C)
    return x[:, :, ::downy, ::downx]


def upsample2d(x, f, up=2):
    fw = f.shape[-1]
    p = ((fw + up - 1) // 2, (fw - up) // 2)
    return upfirdn2d(x, f, up=up, padding=[p[0], p[1], p[0], p[1]], gain=up * up)


def downsample2d(x, f, down=2):
    fw = f.shape[-1]
    p = ((fw - down + 1) // 2, (fw - down) // 2)
    return upfirdn2d(x, f, down=down, padding=[p[0], p[1], p[0], p[1]])


def conv2d_resample(x, w, f=None, up=1, down=1, padding=0, groups=1, flip_weight=True):
    """Only the branches the hot path reaches: up=2 (transposed conv + FIR), down=2 (FIR + strided conv),
    plain conv, and the generic fallback for other combinations."""
    cout, cin_g, kh, kw = w.shape
    fw = f.shape[-1] if f is not None else 1
    px0, px1, py0, py1 = _pad4(padding)
    if up > 1:
        px0 += (fw + up - 1) // 2; px1 += (fw - up) // 2; py0 += (fw + up - 1) // 2; py1 += (fw - up) // 2
    if down > 1:
        px0 += (fw - down + 1) // 2; px1 += (fw - down) // 2; py0 += (fw - down + 1) // 2; py1 += (fw - down) // 2

    def conv(x, w, stride=1, pad=(0, 0), transpose=False, flip=True):
        if not flip and (kw > 1 or kh > 1):
            w = w.flip([2, 3])
        if transpose:
            return F.conv_transpose2d(x, w, stride=stride, padding=pad, groups=groups)
        return F.conv2d(x, w, stride=stride, padding=pad, groups=groups)

    if kw == 1 and kh == 1 and down > 1 and up == 1:
        x = upfirdn2d(x, f, down=down, padding=[px0, px1, py0, py1])
        return conv(x, w, flip=flip_weight)
    if kw == 1 and kh == 1 and up > 1 and down == 1:
        x = conv(x, w, flip=flip_weight)
        return upfirdn2d(x, f, up=up, padding=[px0, px1, py0, py1], gain=up ** 2)
    if down > 1 and up == 1:
        x = upfirdn2d(x, f, padding=[px0, px1, py0, py1])
        return conv(x, w, stride=down, flip=flip_weight)
    if up > 1:
        if groups == 1:
            wt = w.transpose(0, 1)
        else:
            wt = w.reshape(groups, cout // groups, cin_g, kh, kw).transpose(1, 2)
            wt = wt.reshape(groups * cin_g, cout // groups, kh, kw)
        px0 -= kw - 1; px1 -= kw - up; py0 -= kh - 1; py1 -= kh - up
        pxt = max(min(-px0, -px1), 0)
        pyt = max(min(-py0, -py1), 0)
        x = conv(x, wt, stride=up, pad=(pyt, pxt), transpose=True, flip=not flip_weight)
        x = upfirdn2d(x, f, padding=[px0 + pxt, px1 + pxt, py0 + pyt, py1 + pyt], gain=up ** 2)
        if down > 1:
            x = upfirdn2d(x, f, down=down)
        return x
    if px0 == px1 and py0 == py1 and px0 >= 0 and py0 >= 0:
        return conv(x, w, pad=(py0, px0), flip=flip_weight)
    x = upfirdn2d(x, None, padding=[px0, px1, py0, py1])
    return conv(x, w, flip=flip_weight)


def modulated_conv2d(x, weight, styles, noise=None, up=1, padding=0, resample_filter=None, demodulate=True,
                     flip_weight=True):
    """Per-sample modulated weights, grouped conv with groups = batch (the reference's fused inference path)."""
    N = x.shape[0]
    cout, cin, kh, kw = weight.shape
    w = weight[None] * styles.reshape(N, 1, cin, 1, 1)
    if demodulate:
        d = (w.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt()
        w = w * d.reshape(N, cout, 1, 1, 1)
    y = conv2d_resample(x.reshape(1, N * cin, *x.shape[2:]), w.reshape(N * cout, cin, kh, kw),
                        f=resample_filter, up=up, padding=padding, groups=N, flip_weight=flip_weight)
    y = y.reshape(N, cout, *y.shape[2:])
    if noise is not None:
        y = y + noise
    return y


def fully_connected(x, weight, bias=None, activation='linear', lr_multiplier=1.0):
    """FullyConnectedLayer.forward, networks_stylegan2.py:114-127."""
    w = weight * (lr_multiplier / math.sqrt(weight.shape[1]))
    b = bias * lr_multiplier if (bias is not None and lr_multiplier != 1) else bias
    if activation == 'linear' and b is not None:
        return torch.addmm(b[None], x, w.t())
    return bias_act(x.matmul(w.t()), b, act=activation)


def filtered_lrelu(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=SQRT2, slope=0.2, clamp=None,
                   flip_filter=False):
    """bias -> FIR upsample -> lrelu*gain (+clamp) -> FIR downsample, filtered_lrelu.py:123-155."""
    px0, px1, py0, py1 = _pad4(padding)
    x = bias_act(x, b)
    x = upfirdn2d(x, fu, up=up, padding=[px0, px1, py0, py1], gain=up ** 2, flip_filter=flip_filter)
    x = bias_act(x, act='lrelu', alpha=slope, gain=gain, clamp=clamp)
    return upfirdn2d(x, fd, down=down, flip_filter=flip_filter)
