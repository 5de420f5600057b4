"""`torch_utils.ops.filtered_lrelu` on libnext3d_b200 (reference: torch_utils/ops/filtered_lrelu.py:58-118, plugin
filtered_lrelu.cpp:20-213).  Never executed by TriPlaneGenerator.synthesis (only reachable through networks_stylegan3,
SURVEY.md N3); kept for API completeness: same signature, forward only, impl='ref' = torch-op reference (:123-155).  Under grad mode
with x or b requiring grad the CUDA path raises instead of returning a result cut from the graph: the reference's backward
(filtered_lrelu.py:161-270, which replays the forward's sign tensor) is not implemented."""
import numpy as np
import torch

from ... import _lib
from . import bias_act, upfirdn2d
from ._layout import suggest_memory_format

_DTYPES = {torch.float32: 0, torch.float16: 1}


def _get_filter_size(f):
    if f is None:
        return 1, 1
    assert isinstance(f, torch.Tensor) and 1 <= f.ndim <= 2
    return f.shape[-1], f.shape[0]


def _parse_padding(padding):
    if isinstance(padding, int):
        padding = [padding, padding]
    assert isinstance(padding, (list, tuple)) and all(isinstance(x, (int, np.integer)) for x in padding)
    padding = [int(x) for x in padding]
    if len(padding) == 2:
        px, py = padding
        padding = [px, px, py, py]
    return tuple(padding)


def _filtered_lrelu_ref(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=np.sqrt(2), slope=0.2, clamp=None, flip_filter=False):
    px0, px1, py0, py1 = _parse_padding(padding)
    x = bias_act.bias_act(x=x, b=b, impl='ref')
    x = upfirdn2d.upfirdn2d(x=x, f=fu, up=up, padding=[px0, px1, py0, py1], gain=up ** 2, flip_filter=flip_filter, impl='ref')
    x = bias_act.bias_act(x=x, act='lrelu', alpha=slope, gain=gain, clamp=clamp, impl='ref')
    return upfirdn2d.upfirdn2d(x=x, f=fd, down=down, flip_filter=flip_filter, impl='ref')


def _as_2d(f, device):
    if f is None:
        return torch.ones(1, 1, dtype=torch.float32, device=device)
    f = f.to(device=device, dtype=torch.float32)
    return (f.ger(f) if f.ndim == 1 else f).contiguous()


def filtered_lrelu(x, fu=None, fd=None, b=None, up=1, down=1, padding=0, gain=np.sqrt(2), slope=0.2, clamp=None, flip_filter=False, impl='cuda'):
    assert isinstance(x, torch.Tensor) and x.ndim == 4
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        return _filtered_lrelu_ref(x, fu=fu, fd=fd, b=b, up=up, down=down, padding=padding, gain=gain, slope=slope, clamp=clamp, flip_filter=flip_filter)
    _lib.require_cuda(x, 'filtered_lrelu(x)')
    if x.dtype not in _DTYPES:
        raise RuntimeError(f'filtered_lrelu: dtype {x.dtype} is only available with impl="ref"')
    if torch.is_grad_enabled() and (x.requires_grad or (b is not None and b.requires_grad)):
        raise RuntimeError('filtered_lrelu: the backward pass (the reference\'s sign-tensor gradient, filtered_lrelu.py:161-270) is not implemented; '
                           'call it under torch.no_grad() or with impl="ref"')
    px0, px1, py0, py1 = _parse_padding(padding)
    fmt = suggest_memory_format(x)              # the layout the reference's plugin returns (filtered_lrelu.cpp:84)
    x = x.contiguous()
    N, C, H, W = x.shape
    fu2, fd2 = _as_2d(fu, x.device), _as_2d(fd, x.device)
    fuh, fuw = fu2.shape
    fdh, fdw = fd2.shape
    upH, upW = H * up + py0 + py1 - fuh + 1, W * up + px0 + px1 - fuw + 1
    outH, outW = (upH - fdh + down) // down, (upW - fdw + down) // down
    assert upH >= fdh and upW >= fdw and outH >= 1 and outW >= 1
    tmp = torch.empty(N * C * upH * upW, dtype=torch.float32, device=x.device)
    y = torch.empty(N, C, outH, outW, dtype=x.dtype, device=x.device)
    bb = b.to(x.dtype).contiguous() if b is not None else None
    _lib.check(_lib.lib.n3d_filtered_lrelu(x.data_ptr(), fu2.data_ptr() if fu is not None else None, fd2.data_ptr() if fd is not None else None,
                                           _lib.ptr(bb), y.data_ptr(), tmp.data_ptr(), _DTYPES[x.dtype], N, C, H, W, fuh, fuw, fdh, fdw, up, down,
                                           px0, px1, py0, py1, float(gain), float(slope), float(clamp if clamp is not None else -1),
                                           int(bool(flip_filter)), outH, outW, _lib.stream_ptr(x.device)), 'n3d_filtered_lrelu')
    return y.contiguous(memory_format=fmt)
