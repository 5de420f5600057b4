"""`torch_utils.ops.conv2d_resample` on the wgmma implicit-GEMM kernel (reference: torch_utils/ops/conv2d_resample.py:48-143).

Same signature.  NCHW in / NCHW out like the reference; internally the input is converted to the engine's NHWC split-bf16
layout and the convolution runs as n3d_conv_gemm launches:
    up == 2 : 4 transposed-conv parity classes + n3d_fir_up_epilogue   (reference path :114-131)
    down == 2: n3d_fir_down_split + one stride-2 GEMM                  (:108-111)
    otherwise: one GEMM                                                (:134-136)
`groups > 1` (the reference's fused modulated conv uses groups = batch) is executed group by group.
Supported configurations = what the generator uses: 1x1 / 3x3 kernels, padding = k // 2, up/down in {1, 2}, the
[1,3,3,1] x [1,3,3,1] / 64 FIR; anything else raises (no silent fallback).  The fused engine (next3d_b200.engine) does not go
through this wrapper -- it keeps activations in NHWC split form between layers.

Backward (first order, one autograd Function around the whole call): the input gradient of each forward path is another path of
the same kernels -- stride-1 k x k: the k x k GEMM with Cin and Cout swapped and the taps mirrored; up 2: the FIR adjoint onto the
stride-2 lattice (n3d_fir_down_split, gain 4 folded into the weights) and the stride-2 GEMM; down 2: the transposed GEMM and the
FIR-up adjoint (n3d_fir_up_epilogue, gain 1/4 folded into the weights).  The adjoint's input channels (the forward's Cout) are
zero-padded to a multiple of 8.  The weight gradient of all groups and taps is one n3d_conv_wgrad launch (split K, fixed-order
reduction: bit-identical from run to run), skipped under conv2d_gradfix.no_weight_gradients().  Second order is refused.
"""
import torch
import torch.nn.functional as F

from ... import _lib
from ... import kernels as K
from . import conv2d_gradfix, upfirdn2d
from .upfirdn2d import _parse_padding, _get_filter_size  # noqa: F401  (imported by reference code)


def _get_weight_shape(w):
    return [int(sz) for sz in w.shape]


def _check_fir(f):
    ref = upfirdn2d.setup_filter([1, 3, 3, 1], device=f.device)
    if tuple(f.shape) != (4, 4) or not torch.allclose(f, ref, atol=1e-7):
        raise RuntimeError('conv2d_resample: only the [1,3,3,1] (x) [1,3,3,1] / 64 resampling filter is supported by the sm_90a kernels')


def _one_group(x, w, f, up, down, flip_weight):
    """x [N,Cin,H,W] fp32, w [Cout,Cin,k,k] fp32 -> [N,Cout,H',W'] fp32."""
    N, Cin, H, W = x.shape
    Cout, _, k, _ = w.shape
    dev = x.device
    if up > 1:
        flip_weight = not flip_weight                                   # conv2d_resample.py:127 (transposed conv with flip = not flip_weight)
    if not flip_weight and k > 1:
        w = w.flip([2, 3])
    w_hi, w_lo = K.pack_conv_weight(w)
    xn = x.permute(0, 2, 3, 1).contiguous()
    if down == 2 and k == 3:
        if H % 2 or W % 2:
            raise RuntimeError(f'conv2d_resample: down=2 with a 3x3 kernel needs an even input size, got {H}x{W}')
        sh, sw = (H + 2) // 2, (W + 2) // 2
        a_hi = torch.empty(4 * N, sh, sw, Cin, dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        K.fir_down_split(xn, a_hi, a_lo)
        out = torch.empty(N, H // 2, W // 2, Cout, device=dev)
        K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_stride2(), N, H // 2, W // 2, a_img_mul=N, out_f32=out, f32_cstride=Cout)
        return out.permute(0, 3, 1, 2)
    a_hi = torch.empty(N, H, W, Cin, dtype=torch.bfloat16, device=dev)
    a_lo = torch.empty_like(a_hi)
    K.modulate_split(xn, None, a_hi, a_lo)
    if up == 2 and k == 3:
        raw = torch.empty(N, 2 * H + 1, 2 * W + 1, Cout, device=dev)
        K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, H, W, raw)
        out = torch.empty(N, 2 * H, 2 * W, Cout, device=dev)
        K.fir_up_epilogue(raw, Cout, None, None, None, 1.0, 1.0, -1.0, out_f32=out, f32_cstride=Cout)
        return out.permute(0, 3, 1, 2)
    out = torch.empty(N, H, W, Cout, device=dev)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_conv3x3() if k == 3 else K.taps_conv1x1(), N, H, W, out_f32=out, f32_cstride=Cout)
    return out.permute(0, 3, 1, 2)


def conv2d_resample(x, w, f=None, up=1, down=1, padding=0, groups=1, flip_weight=True, flip_filter=False):
    assert isinstance(x, torch.Tensor) and x.ndim == 4
    assert isinstance(w, torch.Tensor) and w.ndim == 4 and w.dtype == x.dtype
    _lib.require_cuda(x, 'conv2d_resample(x)')
    out_channels, in_channels_per_group, kh, kw = _get_weight_shape(w)
    px0, px1, py0, py1 = _parse_padding(padding)
    if kh != kw or kh not in (1, 3) or up not in (1, 2) or down not in (1, 2) or (up == 2 and down == 2):
        raise RuntimeError(f'conv2d_resample: kernel {kh}x{kw}, up={up}, down={down} is not supported by the sm_90a kernels')
    if not (px0 == px1 == py0 == py1 == kh // 2):
        raise RuntimeError('conv2d_resample: only padding == kernel_size // 2 is supported by the sm_90a kernels')
    if in_channels_per_group % 8 != 0:
        raise RuntimeError('conv2d_resample: input channels per group must be a multiple of 8 (TMA stride alignment)')
    if up > 1 or down > 1:
        assert f is not None, 'resampling needs the FIR filter'
        f = f.to(x.device)
        _check_fir(f)
    cfg = (f, up, down, groups, flip_weight, kh)
    if torch.is_grad_enabled() and (x.requires_grad or w.requires_grad):
        return _Conv2dResample.apply(x, w, cfg)
    return _forward(x, w, *cfg)


def _forward(x, w, f, up, down, groups, flip_weight, kh):
    in_channels_per_group, out_channels = w.shape[1], w.shape[0]
    dtype = x.dtype
    xf, wf = x.float(), w.float()
    if kh == 1 and down == 2:                                            # fast path :96-99: downsample first, then 1x1 conv
        xf = upfirdn2d.downsample2d(xf, f)
        up = down = 1
    post_up = kh == 1 and up == 2                                        # fast path :102-105: 1x1 conv first, then upsample
    outs = []
    cin_g, cout_g = in_channels_per_group, out_channels // groups
    for g in range(groups):
        xg = xf[:, g * cin_g:(g + 1) * cin_g]
        wg = wf[g * cout_g:(g + 1) * cout_g]
        outs.append(_one_group(xg, wg, f, 1 if post_up else up, down, flip_weight))
    y = outs[0] if groups == 1 else torch.cat(outs, 1)
    if post_up:
        y = upfirdn2d.upsample2d(y.contiguous(), f)
    return y.contiguous().to(dtype)


# ------------------------------------------------------------------------------------------------ backward
def _round_up(v, m):
    return -(-v // m) * m


def _used_weight_flipped(kind, flip_weight):
    """Whether the weight the GEMMs run (W_used) is w mirrored in both spatial dims (see _one_group)."""
    return (flip_weight if kind == 'up' else not flip_weight)


def _input_grad_group(dy, w_used, kind):
    """dy fp32 NCHW [N, Cout_g, H', W'] of one group, w_used [Cout_g, Cin_g, k, k] -> dx fp32 NCHW [N, Cin_g, H, W]."""
    N, cout, OH, OW = dy.shape
    cin, k = w_used.shape[1], w_used.shape[2]
    cpad = _round_up(cout, 8)
    gain = 4.0 if kind == 'up' else 0.25 if kind == 'down' else 1.0
    w_adj = F.pad(w_used.transpose(0, 1), (0, 0, 0, 0, 0, cpad - cout))            # [Cin, Cout_pad, k, k]
    w_hi, w_lo = K.pack_conv_weight(w_adj, gain)                                        # [T, Cin, Cout_pad], tap = ky * k + kx
    dyn = F.pad(dy.permute(0, 2, 3, 1), (0, cpad - cout)).contiguous()                  # NHWC, zero channels up to Cout_pad
    dev = dy.device
    if kind == 'up':                  # FIR adjoint (pad 2) onto the parity sub-images of the (2H+1)^2 lattice, then the stride-2 GEMM
        H, W = OH // 2, OW // 2
        a_hi = torch.empty(4 * N, H + 1, W + 1, cpad, dtype=torch.bfloat16, device=dev)
        a_lo = torch.empty_like(a_hi)
        K.fir_down_split(dyn, a_hi, a_lo)
        out = torch.empty(N, H, W, cin, device=dev)
        K.conv_gemm(a_hi, a_lo, w_hi, w_lo, K.taps_stride2(), N, H, W, a_img_mul=N, out_f32=out, f32_cstride=cin)
        return out.permute(0, 3, 1, 2)
    a_hi = torch.empty(N, OH, OW, cpad, dtype=torch.bfloat16, device=dev)
    a_lo = torch.empty_like(a_hi)
    K.modulate_split(dyn, None, a_hi, a_lo)
    if kind == 'down':                # transposed stride-2 GEMM onto the (H+1)^2 FIR output, then the FIR adjoint (pad 1)
        H, W = 2 * OH, 2 * OW
        raw = torch.empty(N, H + 1, W + 1, cin, device=dev)
        K.conv_transposed_gemm(a_hi, a_lo, w_hi, w_lo, N, OH, OW, raw)
        out = torch.empty(N, H, W, cin, device=dev)
        K.fir_up_epilogue(raw, cin, None, None, None, 1.0, 1.0, -1.0, out_f32=out, f32_cstride=cin)
        return out.permute(0, 3, 1, 2)
    taps = [(1 - ky, 1 - kx, 0, ky * 3 + kx) for ky in range(3) for kx in range(3)] if k == 3 else K.taps_conv1x1()
    out = torch.empty(N, OH, OW, cin, device=dev)
    K.conv_gemm(a_hi, a_lo, w_hi, w_lo, taps, N, OH, OW, out_f32=out, f32_cstride=cin)
    return out.permute(0, 3, 1, 2)


def _operand(t, s, pad, PH, PW, ld, shifts=(0,)):
    """n3d_wgrad_operand of t once per horizontal shift, stacked along the rows: [len(shifts) * C, ld] (hi, lo)."""
    C = t.shape[1]
    hi = torch.empty(len(shifts) * C, ld, dtype=torch.bfloat16, device=t.device)
    lo = torch.empty_like(hi)
    for i, sh in enumerate(shifts):
        K.wgrad_operand(t, s, pad, pad, PH, PW, ld, hi[i * C:(i + 1) * C], lo[i * C:(i + 1) * C], shift=sh)
    return hi, lo


def _weight_grad(a, dy, f, kind, k, groups):
    """dW_used [G, k*k, Cout_g, Cin_g] of the whole grouped convolution in one n3d_conv_wgrad launch.  a: the GEMMs' input
    fp32 NCHW [N, Cin, H, W]; dy fp32 NCHW [N, Cout, H', W'].  Grid rows are padded to a multiple of 8 positions, so a tap's
    vertical shift (and parity sub-image) is a column offset that is a multiple of 8; its horizontal shift selects a copy of the
    shifted operand by a row offset."""
    N, cin, H, W = a.shape
    cout = dy.shape[1]
    taps = [(ky, kx) for ky in range(k) for kx in range(k)]
    none = [0] * len(taps)
    if kind == 'same':                # positions on the (H + 2p) x (W + 2p) grid, p = k // 2; tap (ky, kx) reads the input at (ky - p, kx - p)
        p = k // 2
        PH, PW = H + 2 * p, _round_up(W + 2 * p, 8)
        Kp = _round_up(N * PH * PW, 64)
        A, B = _operand(dy, 1, p, PH, PW, Kp), _operand(a, 1, p, PH, PW, Kp, shifts=[kx - p for kx in range(k)])
        a_off, a_row = none, none
        b_off, b_row = [(ky - p) * PW for ky, kx in taps], [kx * cin for ky, kx in taps]
    elif kind == 'down':              # dW[ky,kx] = sum dy[o] * F[2o + (ky, kx)], F = the FIR output (H+1)^2, split by parity
        PH, PW = H // 2 + 1, _round_up(W // 2 + 1, 8)
        fa = upfirdn2d.upfirdn2d(a, f, padding=2)
        Kp = _round_up(N * PH * PW, 64)
        A, B = _operand(dy, 1, 0, PH, PW, Kp), _operand(fa, 2, 0, PH, PW, 4 * N * PH * PW, shifts=[0, 1])
        a_off, a_row = none, none
        b_off = [((ky & 1) * 2 + (kx & 1)) * N * PH * PW + (ky >> 1) * PW for ky, kx in taps]
        b_row = [(kx >> 1) * cin for ky, kx in taps]
    else:                             # 'up': dW[ky,kx] = sum x[i] * R[2i + (ky, kx)], R = the raw (2H+1)^2 gradient, split by parity
        PH, PW = H + 1, _round_up(W + 1, 8)
        draw = upfirdn2d.upfirdn2d(dy, f, padding=2, flip_filter=True, gain=4)
        Kp = _round_up(N * PH * PW, 64)
        A, B = _operand(draw, 2, 0, PH, PW, 4 * N * PH * PW, shifts=[0, 1]), _operand(a, 1, 0, PH, PW, Kp)
        a_off = [((ky & 1) * 2 + (kx & 1)) * N * PH * PW + (ky >> 1) * PW for ky, kx in taps]
        a_row = [(kx >> 1) * cout for ky, kx in taps]
        b_off, b_row = none, none
    cout_g, cin_g = cout // groups, cin // groups
    T = len(taps)
    dw = torch.empty(groups, T, cout_g, cin_g, device=a.device)
    splits = K.wgrad_splits(groups, T, cout_g, cin_g, Kp)
    partial = torch.empty(splits, groups, T, cout_g, cin_g, device=a.device) if splits > 1 else None
    K.conv_wgrad(A[0], A[1], B[0], B[1], groups, cout_g, cin_g, Kp, a_off, b_off, dw, splits=splits, partial=partial, a_row=a_row, b_row=b_row)
    return dw


class _Conv2dResample(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, cfg):
        ctx.save_for_backward(x, w)
        ctx.cfg = cfg
        return _forward(x, w, *cfg)

    @staticmethod
    def backward(ctx, dy):
        if torch.is_grad_enabled():
            raise RuntimeError('conv2d_resample: second-order gradients (backward with create_graph=True) are not implemented by the '
                               'sm_90a kernels')
        x, w = ctx.saved_tensors
        f, up, down, groups, flip_weight, k = ctx.cfg
        need_dx = ctx.needs_input_grad[0]
        need_dw = ctx.needs_input_grad[1] and not conv2d_gradfix.weight_gradients_disabled
        xf, wf, dy = x.float(), w.float(), dy.float()
        kind = 'up' if (up == 2 and k == 3) else 'down' if (down == 2 and k == 3) else 'same'
        if k == 1 and up == 2:                                          # forward: 1x1 conv, then upsample2d
            dy = upfirdn2d.adjoint(dy, f, (dy.shape[0], dy.shape[1], dy.shape[2] // 2, dy.shape[3] // 2), up=2, padding=[2, 1, 2, 1], gain=4)
        a = upfirdn2d.downsample2d(xf, f) if (k == 1 and down == 2) else xf    # forward: downsample2d, then 1x1 conv
        w_used = wf.flip([2, 3]) if (k > 1 and _used_weight_flipped(kind, flip_weight)) else wf
        dx = dw = None
        if need_dx:
            cin_g, cout_g = w.shape[1], w.shape[0] // groups
            parts = [_input_grad_group(dy[:, g * cout_g:(g + 1) * cout_g], w_used[g * cout_g:(g + 1) * cout_g], kind) for g in range(groups)]
            dx = parts[0] if groups == 1 else torch.cat(parts, 1)
            if k == 1 and down == 2:
                dx = upfirdn2d.adjoint(dx, f, xf.shape, down=2, padding=1)
            dx = dx.contiguous().to(x.dtype)
        if need_dw:
            g4 = _weight_grad(a.contiguous(), dy.contiguous(), f, kind, k, groups)     # [G, T, Cout_g, Cin_g]
            dw = g4.reshape(groups, k, k, g4.shape[2], g4.shape[3]).permute(0, 3, 4, 1, 2).reshape(w.shape)
            if k > 1 and _used_weight_flipped(kind, flip_weight):
                dw = dw.flip([2, 3])
            dw = dw.contiguous().to(w.dtype)
        return dx, dw, None
