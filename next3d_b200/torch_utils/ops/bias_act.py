"""`torch_utils.ops.bias_act` on libnext3d_b200 (reference: torch_utils/ops/bias_act.py:54-88, plugin bias_act.cpp:36-94).

Same signature and defaults.  impl='cuda' (default) launches n3d_bias_act and REQUIRES a CUDA tensor (no silent CPU
fallback, unlike bias_act.py:86-88); impl='ref' evaluates the same formula with plain torch ops on any device -- it is
the per-op reference implementation the upstream file ships as `_bias_act_ref` (:93-122).

Differentiable to second order like the reference's `BiasActCuda` / `BiasActCudaGrad` (:143-205): the same tensors are saved, the
first-order gradient is n3d_bias_act_grad mode 1, the second-order one mode 2 for the activations with `has_2nd_grad`, and
db = dx summed over every dim except `dim`.  Without grad mode, or when neither x nor b requires grad, the forward is the plain
n3d_bias_act launch.
"""
import numpy as np
import torch

from ... import _lib
from ._layout import suggest_memory_format


class _Spec(dict):
    __getattr__ = dict.__getitem__


activation_funcs = {                                                        # bias_act.py:23-33
    'linear': _Spec(func=lambda x, **_: x, def_alpha=0, def_gain=1, cuda_idx=1, ref='', has_2nd_grad=False),
    'relu': _Spec(func=lambda x, **_: torch.nn.functional.relu(x), def_alpha=0, def_gain=np.sqrt(2), cuda_idx=2, ref='y', has_2nd_grad=False),
    'lrelu': _Spec(func=lambda x, alpha, **_: torch.nn.functional.leaky_relu(x, alpha), def_alpha=0.2, def_gain=np.sqrt(2), cuda_idx=3, ref='y', has_2nd_grad=False),
    'tanh': _Spec(func=lambda x, **_: torch.tanh(x), def_alpha=0, def_gain=1, cuda_idx=4, ref='y', has_2nd_grad=True),
    'sigmoid': _Spec(func=lambda x, **_: torch.sigmoid(x), def_alpha=0, def_gain=1, cuda_idx=5, ref='y', has_2nd_grad=True),
    'elu': _Spec(func=lambda x, **_: torch.nn.functional.elu(x), def_alpha=0, def_gain=1, cuda_idx=6, ref='y', has_2nd_grad=True),
    'selu': _Spec(func=lambda x, **_: torch.nn.functional.selu(x), def_alpha=0, def_gain=1, cuda_idx=7, ref='y', has_2nd_grad=True),
    'softplus': _Spec(func=lambda x, **_: torch.nn.functional.softplus(x), def_alpha=0, def_gain=1, cuda_idx=8, ref='y', has_2nd_grad=True),
    'swish': _Spec(func=lambda x, **_: torch.sigmoid(x) * x, def_alpha=0, def_gain=np.sqrt(2), cuda_idx=9, ref='x', has_2nd_grad=True),
}

_DTYPES = {torch.float32: 0, torch.float16: 1}


def _bias_act_ref(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None):
    spec = activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    clamp = float(clamp if clamp is not None else -1)
    if b is not None:
        assert b.ndim == 1 and 0 <= dim < x.ndim and b.shape[0] == x.shape[dim]
        x = x + b.reshape([-1 if i == dim else 1 for i in range(x.ndim)])
    x = spec.func(x, alpha=alpha)
    if gain != 1:
        x = x * gain
    if clamp >= 0:
        x = x.clamp(-clamp, clamp)
    return x


def bias_act(x, b=None, dim=1, act='linear', alpha=None, gain=None, clamp=None, impl='cuda'):
    assert isinstance(x, torch.Tensor)
    assert impl in ['ref', 'cuda']
    if impl == 'ref':
        return _bias_act_ref(x=x, b=b, dim=dim, act=act, alpha=alpha, gain=gain, clamp=clamp)
    _lib.require_cuda(x, 'bias_act(x)')
    if x.dtype not in _DTYPES:
        raise RuntimeError(f'bias_act: dtype {x.dtype} is only available with impl="ref"')
    spec = activation_funcs[act]
    alpha = float(alpha if alpha is not None else spec.def_alpha)
    gain = float(gain if gain is not None else spec.def_gain)
    clamp = float(clamp if clamp is not None else -1)
    assert clamp is None or clamp >= 0 or clamp == -1
    if b is not None:
        assert b.ndim == 1 and 0 <= dim < x.ndim and b.shape[0] == x.shape[dim]
    if torch.is_grad_enabled() and (x.requires_grad or (b is not None and b.requires_grad)):
        return _BiasActCuda.apply(x, b, (dim, act, spec, alpha, gain, clamp))
    return _forward(x, b, dim, spec, alpha, gain, clamp)


def _forward(x, b, dim, spec, alpha, gain, clamp):
    if not (x.is_contiguous() or x.is_contiguous(memory_format=torch.channels_last)):
        x = x.contiguous(memory_format=suggest_memory_format(x))               # plugin requires dense x (bias_act.cpp:51)
    y = torch.empty_like(x)
    size_b = step_b = 0
    if b is not None:
        b = b.to(x.dtype).contiguous()
        size_b, step_b = b.shape[0], max(int(x.stride(dim)), 1)
    if x.numel() > 0:
        _lib.check(_lib.lib.n3d_bias_act(x.data_ptr(), _lib.ptr(b), y.data_ptr(), _DTYPES[x.dtype], x.numel(), size_b, step_b, spec.cuda_idx,
                                         alpha, gain, clamp, _lib.stream_ptr(x.device)), 'n3d_bias_act')
    return y


def _memory_format(t):
    return torch.channels_last if t.ndim == 4 and t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous() \
        else torch.contiguous_format


def _grad(mode, dy, b, x, y, dyref, cfg):
    """n3d_bias_act_grad: dy / x / y / dyref in one dense layout (dy's); x and y may be None where the activation does not read them."""
    dim, act, spec, alpha, gain, clamp = cfg
    fmt = _memory_format(dy)
    dy = dy.contiguous(memory_format=fmt)
    x, y, dyref = (None if t is None else t.contiguous(memory_format=fmt) for t in (x, y, dyref))
    dx = torch.empty_like(dy)
    size_b = step_b = 0
    if b is not None:
        b = b.to(dy.dtype).contiguous()
        size_b, step_b = b.shape[0], max(int(dy.stride(dim)), 1)
    if dy.numel() > 0:
        _lib.check(_lib.lib.n3d_bias_act_grad(dy.data_ptr(), _lib.ptr(b), _lib.ptr(x), _lib.ptr(y), _lib.ptr(dyref), dx.data_ptr(), _DTYPES[dy.dtype],
                                              dy.numel(), size_b, step_b, mode, spec.cuda_idx, alpha, gain, clamp, _lib.stream_ptr(dy.device)),
                   'n3d_bias_act_grad')
    return dx


def _sum_but(t, dim):
    return t.sum([i for i in range(t.ndim) if i != dim])


class _BiasActCuda(torch.autograd.Function):
    """bias_act.py:144-174: saves x and b where the activation reads x or has a second derivative, y where it reads y."""

    @staticmethod
    def forward(ctx, x, b, cfg):
        dim, act, spec, alpha, gain, clamp = cfg
        y = _forward(x, b, dim, spec, alpha, gain, clamp)
        keep_x = 'x' in spec.ref or spec.has_2nd_grad
        ctx.cfg = cfg
        ctx.save_for_backward(x if keep_x else None, b if keep_x else None, y if 'y' in spec.ref else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        dim, act, spec, alpha, gain, clamp = ctx.cfg
        x, b, y = ctx.saved_tensors
        dx = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dx = dy
            if act != 'linear' or gain != 1 or clamp >= 0:
                dx = _BiasActCudaGrad.apply(dy, x, b, y, ctx.cfg)
        if ctx.needs_input_grad[1]:
            db = _sum_but(dx, dim)
        return dx, db, None


class _BiasActCudaGrad(torch.autograd.Function):
    """bias_act.py:177-205: dx = grad mode 1; its gradient with respect to dy is itself, and with respect to x (and b) grad mode 2."""

    @staticmethod
    def forward(ctx, dy, x, b, y, cfg):
        spec = cfg[2]
        dx = _grad(1, dy, b, x, y, None, cfg)
        ctx.cfg = cfg
        ctx.save_for_backward(dy if spec.has_2nd_grad else None, x, b, y)
        return dx

    @staticmethod
    def backward(ctx, d_dx):
        dim, spec = ctx.cfg[0], ctx.cfg[2]
        dy, x, b, y = ctx.saved_tensors
        d_dy = d_x = d_b = None
        if ctx.needs_input_grad[0]:
            d_dy = _BiasActCudaGrad.apply(d_dx, x, b, y, ctx.cfg)
        if spec.has_2nd_grad and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            d_x = _grad(2, d_dx, b, x, y, dy, ctx.cfg)
        if spec.has_2nd_grad and ctx.needs_input_grad[2]:
            d_b = _sum_but(d_x, dim)
        return d_dy, d_x, d_b, None, None
