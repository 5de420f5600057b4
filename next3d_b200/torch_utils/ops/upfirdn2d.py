"""`torch_utils.ops.upfirdn2d` on libnext3d_b200 (reference: torch_utils/ops/upfirdn2d.py, plugin upfirdn2d.cpp:20-102).

Same functions, signatures and defaults: setup_filter :72, upfirdn2d :120, filter2d :279, upsample2d :315,
downsample2d :354 and the private helpers conv2d_resample imports (:36-66).  impl='cuda' requires CUDA tensors (no silent
fallback); impl='ref' is the torch-op reference implementation (:169-213).

Differentiable with respect to x to any order, as the reference's `Upfirdn2dCuda` (:233-270): the gradient is upfirdn2d itself with
up and down swapped, the filter flipped and the padding of :258-263, called through this same function.  A gradient with respect to
the filter is refused.
"""
import numpy as np
import torch

from ... import _lib
from ._layout import suggest_memory_format

_DTYPES = {torch.float32: 0, torch.float16: 1}


def _parse_scaling(scaling):
    if isinstance(scaling, int):
        scaling = [scaling, scaling]
    assert isinstance(scaling, (list, tuple)) and all(isinstance(x, int) for x in scaling)
    sx, sy = scaling
    assert sx >= 1 and sy >= 1
    return sx, sy


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(x, int) for x in padding)
    if len(padding) == 2:
        padx, pady = padding
        padding = [padx, padx, pady, pady]
    padx0, padx1, pady0, pady1 = padding
    return padx0, padx1, pady0, pady1


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and f.ndim in [1, 2]
    return int(f.shape[-1]), int(f.shape[0])


def setup_filter(f, device=torch.device('cpu'), normalize=True, flip_filter=False, gain=1, separable=None):
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in [0, 1, 2] and f.numel() > 0
    if f.ndim == 0:
        f = f[np.newaxis]
    if separable is None:
        separable = (f.ndim == 1 and f.numel() >= 8)
    if f.ndim == 1 and not separable:
        f = f.ger(f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def _upfirdn2d_ref(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1):
    assert isinstance(x, torch.Tensor) and x.ndim == 4
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
    batch_size, num_channels, in_height, in_width = x.shape
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    x = x.reshape([batch_size, num_channels, in_height, 1, in_width, 1])
    x = torch.nn.functional.pad(x, [0, upx - 1, 0, 0, 0, upy - 1])
    x = x.reshape([batch_size, num_channels, in_height * upy, in_width * upx])
    x = torch.nn.functional.pad(x, [max(padx0, 0), max(padx1, 0), max(pady0, 0), max(pady1, 0)])
    x = x[:, :, max(-pady0, 0): x.shape[2] - max(-pady1, 0), max(-padx0, 0): x.shape[3] - max(-padx1, 0)]
    f = f * (gain ** (f.ndim / 2))
    f = f.to(x.dtype)
    if not flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f[np.newaxis, np.newaxis].repeat([num_channels, 1] + [1] * f.ndim)
    if f.ndim == 4:
        x = torch.nn.functional.conv2d(input=x, weight=f, groups=num_channels)
    else:
        x = torch.nn.functional.conv2d(input=x, weight=f.unsqueeze(2), groups=num_channels)
        x = torch.nn.functional.conv2d(input=x, weight=f.unsqueeze(3), groups=num_channels)
    return x[:, :, ::downy, ::downx]


def _launch(x, f2d, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain):
    N, C, H, W = x.shape
    fh, fw = f2d.shape
    outH = (H * upy + pady0 + pady1 - fh + downy) // downy
    outW = (W * upx + padx0 + padx1 - fw + downx) // downx
    assert outH >= 1 and outW >= 1
    # y in x's suggested layout, as the reference's plugin allocates it (upfirdn2d.cpp:42); the kernel takes any y strides
    y = torch.empty([N, C, outH, outW], dtype=x.dtype, device=x.device, memory_format=suggest_memory_format(x))
    xs = (_lib.I64 * 4)(*x.stride())
    ys = (_lib.I64 * 4)(*y.stride())
    _lib.check(_lib.lib.n3d_upfirdn2d(x.data_ptr(), f2d.data_ptr(), y.data_ptr(), _DTYPES[x.dtype], N, C, H, W, xs, ys, fh, fw, upx, upy, downx, downy,
                                      padx0, padx1, pady0, pady1, int(bool(flip_filter)), float(gain), outH, outW, _lib.stream_ptr(x.device)),
               'n3d_upfirdn2d')
    return y


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl='cuda'):
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        return _upfirdn2d_ref(x, f, up=up, down=down, padding=padding, flip_filter=flip_filter, gain=gain)
    _lib.require_cuda(x, 'upfirdn2d(x)')
    if x.dtype not in _DTYPES:
        raise RuntimeError(f'upfirdn2d: dtype {x.dtype} is only available with impl="ref"')
    assert x.ndim == 4
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    if f is None:
        f = torch.ones([1, 1], dtype=torch.float32, device=x.device)
    assert f.dtype == torch.float32 and f.ndim in [1, 2]
    f = f.to(x.device)
    if torch.is_grad_enabled() and (x.requires_grad or f.requires_grad):
        if f.requires_grad:
            raise RuntimeError('upfirdn2d: gradients with respect to the filter f are not implemented (as in the reference)')
        return _Upfirdn2dCuda.apply(x, f, (upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain))
    return _forward(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain)


def _forward(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain):
    if f.ndim == 2:
        return _launch(x, f.contiguous(), upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain)
    # separable: horizontal pass then vertical pass, gain split evenly (upfirdn2d.py:262-264)
    g = float(np.sqrt(gain))
    y = _launch(x, f[np.newaxis, :].contiguous(), upx, 1, downx, 1, padx0, padx1, 0, 0, flip_filter, g)
    return _launch(y, f[:, np.newaxis].contiguous(), 1, upy, 1, downy, 0, 0, pady0, pady1, flip_filter, g)


def _adjoint_padding(x_shape, dy_shape, f, upx, upy, downx, downy, padx0, pady0):
    """Padding of the upfirdn2d that maps dy back onto x (upfirdn2d.py:257-263)."""
    _, _, ih, iw = x_shape
    _, _, oh, ow = dy_shape
    fw, fh = _get_filter_size(f)
    return [fw - padx0 - 1, iw * upx - ow * downx + padx0 - upx + 1, fh - pady0 - 1, ih * upy - oh * downy + pady0 - upy + 1]


def adjoint(dy, f, x_shape, up=1, down=1, padding=0, flip_filter=False, gain=1):
    """The gradient of upfirdn2d(x, f, up, down, padding, flip_filter, gain) with respect to x (x of shape x_shape), given the output
    gradient dy: upfirdn2d with up and down swapped and the filter flipped."""
    upx, upy = _parse_scaling(up)
    downx, downy = _parse_scaling(down)
    padx0, _, pady0, _ = _parse_padding(padding)
    p = _adjoint_padding(x_shape, dy.shape, f, upx, upy, downx, downy, padx0, pady0)
    return upfirdn2d(dy, f, up=[downx, downy], down=[upx, upy], padding=p, flip_filter=not flip_filter, gain=gain)


class _Upfirdn2dCuda(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, f, cfg):
        ctx.save_for_backward(f)
        ctx.cfg, ctx.x_shape = cfg, x.shape
        return _forward(x, f, *cfg)

    @staticmethod
    def backward(ctx, dy):
        f, = ctx.saved_tensors
        upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip_filter, gain = ctx.cfg
        dx = None
        if ctx.needs_input_grad[0]:
            dx = adjoint(dy, f, ctx.x_shape, [upx, upy], [downx, downy], [padx0, padx1, pady0, pady1], flip_filter, gain)
        return dx, None, None


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl='cuda'):
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + fw // 2, padx1 + (fw - 1) // 2, pady0 + fh // 2, pady1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    upx, upy = _parse_scaling(up)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw + upx - 1) // 2, padx1 + (fw - upx) // 2, pady0 + (fh + upy - 1) // 2, pady1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy, impl=impl)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl='cuda'):
    downx, downy = _parse_scaling(down)
    padx0, padx1, pady0, pady1 = _parse_padding(padding)
    fw, fh = _get_filter_size(f)
    p = [padx0 + (fw - downx + 1) // 2, padx1 + (fw - downx) // 2, pady0 + (fh - downy + 1) // 2, pady1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain, impl=impl)
