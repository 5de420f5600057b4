"""CPU oracle: the super-resolution head in fp16, as the reference runs it on CUDA with sr_num_fp16_res > 0.
TEST INFRASTRUCTURE, NOT PRODUCT CODE (see oracle/__init__.py).

SuperresolutionHybrid8XDC / 4X build both SR blocks with use_fp16 (superresolution.py:268-277, :66-74); on a CUDA device a block
then runs in fp16 (networks_stylegan2.py:547-549; only the CPU path forces fp32), and at inference every modulated conv takes the
fused path (fused_modconv_default='inference_only', train_next3d.py:382).  This restates that forward cast by cast:
  block entry            x.to(float16)                                            networks_stylegan2.py:557
  pre-normalisation      weight * (1/sqrt(Cin k^2) / max|W[o]|), styles / max|s|   :54-56
  modulate + demodulate  in fp32, then w.to(float16)                              :61-67, :77
  convolution            fp16 operands, fp32 accumulate, output rounded to fp16   :77 (conv2d_resample; up=2: the transposed
                         conv's output and the FIR's output are each rounded)      conv2d_resample.py:114-131
  noise                  x.add_(noise) on the fp16 tensor                         :80
  bias_act               fp16 in / out, fp32 inside (the CUDA plugin), bias.to(float16), clamp 256     :330
  ToRGB                  fp16 modulated 1x1 conv (no demodulation), bias_act with the clamp, then .to(float32)   :353-357, :576
  img                    upsampled and accumulated in fp32                        :573-577
An fp16 tensor is held here as the fp32 tensor of its values (_h rounds to fp16); every op computes in fp32 on those values and
rounds its result, as the CUDA kernels do for fp16 inputs and outputs.

plugins=False rounds instead where the reference's CPU fallbacks round, the one difference between the reference's fp16 forward on
CPU and on CUDA: _bias_act_ref (bias_act.py:93-122) is a chain of fp16 tensor ops, so x + b, leaky_relu, * gain and the clamp each
round to fp16, where the CUDA plugin (bias_act.cu) computes the chain in fp32 and rounds once.  The other ops round at the same
points on both devices: the convolutions (fp16 output), _upfirdn2d_ref (f.to(float16), whose taps k/64 * 4 are exact, then one
fp16 convolution, upfirdn2d.py:197-209) and the fp32 ToRGB accumulation.  tests/test_oracle_sr_fp16.py pins plugins=False to the
reference's own SR blocks run in fp16 on CPU.
"""
import math

import torch
import torch.nn.functional as F

from . import ops


def _h(t):
    """Round to fp16 (round to nearest even), keep fp32 storage."""
    return t.to(torch.float16).to(torch.float32)


def _grouped_conv(x, w, up):
    """conv2d_resample(x, w, f, up, padding=1, groups=N) of modulated weights w [N, Cout, Cin, k, k], x [N, Cin, H, W], with the
    fp16 roundings of the CUDA path.  up=2: transposed conv (flip_weight=False, conv2d_resample.py:114-127) then the 4x4 FIR with
    gain 4 and padding 1 (:129-131)."""
    N, cout, cin, kh, kw = w.shape
    xg = x.reshape(1, N * cin, *x.shape[2:])
    if up == 1:
        y = F.conv2d(xg, w.reshape(N * cout, cin, kh, kw), padding=kh // 2, groups=N)
        return _h(y.reshape(N, cout, *y.shape[2:]))
    wt = w.transpose(1, 2).reshape(N * cin, cout, kh, kw)
    y = _h(F.conv_transpose2d(xg, wt, stride=2, groups=N))
    y = y.reshape(N, cout, *y.shape[2:])
    return _h(ops.upfirdn2d(y, ops.setup_filter(), padding=[1, 1, 1, 1], gain=4))


def _bias_act(y, b, act, clamp, plugins):
    """bias_act(y, b.to(float16), act, clamp) on fp16 values: one rounding (the CUDA plugin) or one per op (_bias_act_ref)."""
    b = _h(b)
    if plugins:
        return _h(ops.bias_act(y, b, act=act, clamp=clamp))
    y = _h(y + b.reshape(1, -1, 1, 1))
    if act == 'lrelu':
        y = _h(_h(F.leaky_relu(y, 0.2)) * math.sqrt(2))
    return y.clamp(-clamp, clamp) if clamp is not None else y


def synthesis_layer(sd, p, x, w, up=1, noise_mode='none', clamp=None, plugins=True):
    """SynthesisLayer.forward (networks_stylegan2.py:311-330) on the fp16 values x."""
    styles = ops.fully_connected(w, sd[f'{p}.affine.weight'], sd[f'{p}.affine.bias'])
    weight = sd[f'{p}.weight']
    N = x.shape[0]
    cout, cin, kh, kw = weight.shape
    weight = weight * (1 / math.sqrt(cin * kh * kw) / weight.abs().amax(dim=[1, 2, 3], keepdim=True))
    styles = styles / styles.abs().amax(dim=1, keepdim=True)
    wm = weight[None] * styles.reshape(N, 1, cin, 1, 1)
    wm = wm * (wm.square().sum(dim=[2, 3, 4]) + 1e-8).rsqrt().reshape(N, cout, 1, 1, 1)
    y = _grouped_conv(x, _h(wm), up)
    if noise_mode == 'const':
        y = _h(y + sd[f'{p}.noise_const'] * sd[f'{p}.noise_strength'])
    elif noise_mode != 'none':
        raise ValueError('the fp16 SR oracle supports superresolution_noise_mode const / none')
    return _bias_act(y, sd[f'{p}.bias'], 'lrelu', clamp, plugins)


def torgb(sd, p, x, w, clamp=None, plugins=True):
    """ToRGBLayer.forward (networks_stylegan2.py:353-357) on the fp16 values x -> fp32 values of the fp16 result."""
    weight = sd[f'{p}.weight']
    N = x.shape[0]
    cout, cin, kh, kw = weight.shape
    styles = ops.fully_connected(w, sd[f'{p}.affine.weight'], sd[f'{p}.affine.bias']) * (1 / math.sqrt(cin * kh * kw))
    wm = _h(weight[None] * styles.reshape(N, 1, cin, 1, 1))
    y = _grouped_conv(x, wm, 1)
    return _bias_act(y, sd[f'{p}.bias'], 'linear', clamp, plugins)


def synthesis_block(sd, p, x, img, ws, noise_mode='none', clamp=None, up=True, plugins=True):
    """SynthesisBlock.forward (networks_stylegan2.py:544-588; SynthesisBlockNoUp superresolution.py:209-254 with up=False), fp16."""
    it = iter(ws.unbind(1))
    x = _h(x)
    x = synthesis_layer(sd, f'{p}.conv0', x, next(it), up=2 if up else 1, noise_mode=noise_mode, clamp=clamp, plugins=plugins)
    x = synthesis_layer(sd, f'{p}.conv1', x, next(it), noise_mode=noise_mode, clamp=clamp, plugins=plugins)
    if up:
        img = ops.upsample2d(img, sd[f'{p}.resample_filter'])
    return x, img + torgb(sd, f'{p}.torgb', x, next(it), clamp=clamp, plugins=plugins)


def superresolution(sd, cfg, rgb, x, ws, plugins=True):
    """SuperresolutionHybrid8XDC.forward (superresolution.py:279-290) / 4X (:77-88) with both blocks in fp16.  rgb [N,3,R,R] and
    x [N,32,R,R] fp32, ws [N, >= 1, 512] (the last row is used) -> the fp32 image.  plugins: the CUDA plugins' rounding (True, the
    reference on a GPU) or its CPU fallbacks' (False), see the module docstring."""
    if not cfg.sr_num_fp16_res > 0:
        raise ValueError('with sr_num_fp16_res == 0 the reference runs the SR head in fp32 (oracle.generator.superresolution)')
    ws = ws[:, -1:, :].repeat(1, 3, 1)
    aa = cfg.rendering_kwargs['sr_antialias']
    need = x.shape[-1] != 128 if cfg.sr_module == '8XDC' else x.shape[-1] < 128
    if need:
        x = F.interpolate(x, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
        rgb = F.interpolate(rgb, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
    nm = cfg.rendering_kwargs['superresolution_noise_mode']
    x, rgb = synthesis_block(sd, 'superresolution.block0', x, rgb, ws, noise_mode=nm, clamp=cfg.sr_clamp, up=(cfg.sr_module == '8XDC'),
                             plugins=plugins)
    x, rgb = synthesis_block(sd, 'superresolution.block1', x, rgb, ws, noise_mode=nm, clamp=cfg.sr_clamp, plugins=plugins)
    return rgb


# ------------------------------------------------------------------------------------------ where the engine rounds
def superresolution_engine_order(sd, cfg, rgb, x, ws):
    """The fp16 SR head with the roundings of next3d_b200's sr_precision='fp16' path instead of the reference's: the activation is
    pre-multiplied by its consumer's style and rounded to fp16 once (after the whole epilogue of the producing layer); the weights
    carry the reference's pre-normalisation (networks_stylegan2.py:54) and are rounded to fp16 unmodulated, shared by the batch;
    demodulation (with the raw styles, which it cancels), noise, bias, lrelu * sqrt(2), the clamp and the ToRGB sums are fp32.  The
    GPU tests hold the engine to this statement tightly, and to `superresolution` (the reference's order) at fp16 accuracy."""
    if not cfg.sr_num_fp16_res > 0:
        raise ValueError('with sr_num_fp16_res == 0 the reference runs the SR head in fp32 (oracle.generator.superresolution)')
    w = ws[:, -1]
    aa = cfg.rendering_kwargs['sr_antialias']
    need = x.shape[-1] != 128 if cfg.sr_module == '8XDC' else x.shape[-1] < 128
    if need:
        x = F.interpolate(x, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
        rgb = F.interpolate(rgb, size=(128, 128), mode='bilinear', align_corners=False, antialias=aa)
    nm = cfg.rendering_kwargs['superresolution_noise_mode']
    clamp = cfg.sr_clamp

    def style(p):
        return ops.fully_connected(w, sd[f'{p}.affine.weight'], sd[f'{p}.affine.bias'])

    def layer(p, x16, up, nxt):
        W = sd[f'{p}.weight']
        cout, cin, kh, kw = W.shape
        Wn = W * (1 / math.sqrt(cin * kh * kw) / W.abs().amax(dim=[1, 2, 3], keepdim=True))
        d = ((style(p).square()[:, None, :] * Wn.square().sum(dim=[2, 3])[None]).sum(-1) + 1e-8).rsqrt()
        W16 = _h(Wn)
        if up == 1:
            acc = F.conv2d(x16, W16, padding=kh // 2)
        else:
            acc = ops.upfirdn2d(F.conv_transpose2d(x16, W16.transpose(0, 1), stride=2), ops.setup_filter(), padding=[1, 1, 1, 1], gain=4)
        v = acc * d[:, :, None, None]
        if nm == 'const':
            v = v + sd[f'{p}.noise_const'] * sd[f'{p}.noise_strength']
        elif nm != 'none':
            raise ValueError('the fp16 SR oracle supports superresolution_noise_mode const / none')
        v = ops.bias_act(v, sd[f'{p}.bias'], act='lrelu', clamp=clamp)
        return v, (_h(v * style(nxt)[:, :, None, None]) if nxt else None)

    def torgb(p, v):
        s = style(p) * (1 / math.sqrt(v.shape[1]))
        y = torch.einsum('nchw,oc,nc->nohw', v, sd[f'{p}.weight'][:, :, 0, 0], s)
        return ops.bias_act(y, sd[f'{p}.bias'], clamp=clamp)

    b0, b1 = 'superresolution.block0', 'superresolution.block1'
    x16 = _h(x * style(f'{b0}.conv0')[:, :, None, None])
    v, x16 = layer(f'{b0}.conv0', x16, 2 if cfg.sr_module == '8XDC' else 1, f'{b0}.conv1')
    v, x16 = layer(f'{b0}.conv1', x16, 1, f'{b1}.conv0')
    if cfg.sr_module == '8XDC':
        rgb = ops.upsample2d(rgb, sd[f'{b0}.resample_filter'])
    img = rgb + torgb(f'{b0}.torgb', v)
    v, x16 = layer(f'{b1}.conv0', x16, 2, f'{b1}.conv1')
    v, _ = layer(f'{b1}.conv1', x16, 1, None)
    return ops.upsample2d(img, sd[f'{b1}.resample_filter']) + torgb(f'{b1}.torgb', v)
