"""The gradient kernels against an fp64 reference, over a table of launches that reaches every kernel and configuration their entry
points can select:

    n3d_conv_wgrad      conv_wgrad_kernel<32 | 64 | 128> (split K) and, for more than one K slice, wgrad_reduce_kernel
    n3d_wgrad_operand   wgrad_operand_kernel
    n3d_bias_act_grad   bias_act_grad_kernel<float | __half>
    conv2d_resample     the backward of torch_utils.ops.conv2d_resample: the operand copies and the one n3d_conv_wgrad launch its
                        weight gradient makes, for every kind of layer

References:
- n3d_conv_wgrad: the exact fp64 products of the bf16 operands, hi*hi + hi*lo + lo*hi, so only the fp32 summation order is left.
- n3d_wgrad_operand: bit for bit, kernels.split_bf16 of the gathered fp32 operand (the same round-to-nearest split).
- n3d_bias_act_grad: the fp64 derivative of oracle.ops.bias_act at the saved input, times the plugin's strict clamp mask taken from the
  saved output.  At a kink (elu / selu at exactly 0) the plugin takes the derivative of the right-hand branch, and so does the reference.
- conv2d_resample: y, dx and dw against oracle.ops.conv2d_resample under fp64 autograd on the device.

Every output is a view into a larger allocation filled with a NaN sentinel: the elements a launch owns must be written (and match), the
guard bands must keep the sentinel's bits.  Each case is rerun and must be bit-identical.

`wgrad_plan`, `wgrad_splits_mirror`, `operand_plan`, `bias_act_grad_plan` and `resample_plan` mirror the launch rules in plain Python.
The CPU test checks that the table covers everything in COVERAGE; the profiler test checks on the GPU that each case launched the
kernel instance and grid the mirror predicts.
"""
import math
import re

import numpy as np
import pytest
import torch

from tests.helpers import Guarded, RangeErr, cdiv, grid_stride, launched_kernels, range_rel_err, record_errors, rerun_identical

DEV = 'cuda'
SMS = 132                   # SM count the table is planned at (H100 SXM)
F64 = torch.float64

# Range-relative error bounds, max |got - ref| / max |ref| over an output, each at most 4x the worst case measured over the table on
# an H100 80GB HBM3 (700 W power limit), which is given beside it.  The weight-gradient kinds are scaled by wgrad_scale, the length
# of the longest K slice in units of 512 positions (at least 1); the worst case beside them is the worst err / scale.
# N3D_GRAD_ERRORS=<file> appends every measured error to that file as JSON lines.
BOUNDS = {
    'wgrad': 8e-6,          # n3d_conv_wgrad against the exact bf16 products: fp32 summation only.  Worst: 2.0e-6 (wgrad_bn64_wrap)
    'conv.y': 6.9e-5,       # conv2d_resample fp32, forward.  Worst: 1.74e-5 (conv_prod_same3_c512_64)
    'conv.dx': 6.9e-5,      # input gradient.  Worst: 1.74e-5 (conv_prod_same3_c512_64)
    'conv.dw': 2.5e-5,      # weight gradient (scaled).  Worst: 8.4e-6 (conv_up3_w15_g3_cl)
    'conv16.y': 1.6e-3,     # conv2d_resample fp16: x, w, dy and the results in fp16 (2^-11 relative each).  Worst: 4.2e-4 (conv_same1_w8_g3_k64)
    'conv16.dx': 1.4e-3,    # Worst: 3.7e-4 (conv_down3_w30_g3_f16_cl_k64)
    'conv16.dw': 1.3e-3,    # (scaled).  Worst: 3.4e-4 (conv_same3_odd_f16_cl)
    'ba1.f32': 6.5e-7,      # bias_act grad mode 1, fp32: fp32 formulas from the fp32-rounded saved output.  Worst: 1.6e-7 (ba_softplus_g1_f32_nchw)
    'ba2.f32': 7.9e-7,      # grad mode 2, fp32.  Worst: 2.0e-7 (ba_sigmoid_g2_f32_cl)
    'ba1.f16': 1.9e-3,      # fp16: dy, the saved output and dx in fp16.  Worst: 4.8e-4 (ba_sigmoid_g1_f16_cl)
    'ba2.f16': 5.2e-3,      # Worst: 1.3e-3 (ba_sigmoid_g2_f16_nchw)
}


def wgrad_scale(longest_ksteps):
    """The factor a weight-gradient bound is scaled by: the longest K slice over 512 positions, at least 1.  The error of the tensor
    cores' fp32 accumulation grows about linearly with the length of the sum: measured over the table, about 2e-6 per 512 positions,
    from 256 to 8192 positions in one slice."""
    return max(longest_ksteps * KBK, 512) / 512


# ------------------------------------------------------------------------------------------------ the launch rules, mirrored
KBM, KBK = 128, 64              # conv_wgrad tile: 128 output channels, 64 positions per stage
RING_BYTES, MAX_STAGES = 200 * 1024, 6


def block_n(N):
    return 32 if N <= 32 else 64 if N <= 64 else 128


def wgrad_plan(G, T, M, N, K, splits, sms=SMS):
    """n3d_conv_wgrad: the conv_wgrad_kernel<block_n> instance, its stage ring (as many 2 x (A + B) split-bf16 stages as fit in 200 KB,
    at most 6), the tiles, each K slice's [kb, ke) K steps (per = ceil(ksteps / splits) steps each, the last ones possibly empty), the
    main grid and, for splits > 1, the reduction's grid-stride grid over G*T*M*N / 4 float4."""
    bn = block_n(N)
    stages = min(MAX_STAGES, RING_BYTES // (2 * KBM * KBK * 2 + 2 * bn * KBK * 2))
    m_tiles, n_tiles, ksteps = cdiv(M, KBM), cdiv(N, bn), K // KBK
    per = cdiv(ksteps, splits)
    slices = []
    for s in range(splits):
        kb = min(ksteps, s * per)
        slices.append((kb, min(ksteps, kb + per)))
    lengths = [ke - kb for kb, ke in slices]
    n4 = G * T * M * N // 4
    p = dict(kernel=f'conv_wgrad_kernel<{bn}>', block_n=bn, stages=stages, m_tiles=m_tiles, n_tiles=n_tiles, ksteps=ksteps, splits=splits,
             slices=slices, empty=[n == 0 for n in lengths], longest=max(lengths), last=lengths[-1],
             grid=(m_tiles * n_tiles * splits, T, G), reduce_grid=None, reduce_passes=0)
    if splits > 1:
        p['reduce_grid'] = grid_stride(n4, sms, 8)
        p['reduce_passes'] = cdiv(n4, p['reduce_grid'] * 256)
    return p


def wgrad_splits_mirror(G, T, M, N, K, sms=SMS):
    """kernels.wgrad_splits restated: the slices that bring the CTAs (tiles x taps x groups x slices) to two waves over the SMs, but no
    more slices than leave 8 K steps in each, and at least one."""
    tiles = cdiv(M, KBM) * cdiv(N, block_n(N)) * T * G
    want = cdiv(2 * sms, tiles)
    cap = max(1, (K // KBK) // 8)
    return max(1, min(want, cap))


def operand_plan(C, ld, sms=SMS):
    """n3d_wgrad_operand: one thread per element of [C, ld], grid-stride at 16 blocks per SM."""
    return dict(kernel='wgrad_operand_kernel', grid=grid_stride(C * ld, sms, 16), passes=cdiv(C * ld, grid_stride(C * ld, sms, 16) * 256))


def bias_act_grad_plan(numel, dtype, sms=SMS):
    """n3d_bias_act_grad: nothing for numel 0, else one thread per element, grid-stride at 8 blocks per SM."""
    if numel == 0:
        return None
    grid = grid_stride(numel, sms, 8)
    return dict(kernel=f'bias_act_grad_kernel<{"float" if dtype == torch.float32 else "__half"}>', grid=grid,
                passes=cdiv(numel, grid * 256))


def _r8(v):
    return cdiv(v, 8) * 8


def resample_kind(k, up, down):
    """The forward path of conv2d_resample: 'same' (stride 1, also the 1x1 fast paths), 'up' (up-2 3x3), 'down' (down-2 3x3), with
    'up1' / 'down1' naming the 1x1 post-upsample and pre-downsample fast paths."""
    if k == 3:
        return 'up' if up == 2 else 'down' if down == 2 else 'same3'
    return 'up1' if up == 2 else 'down1' if down == 2 else 'same1'


def resample_plan(N, cin, cout, H, W, k, up, down, groups, sms=SMS):
    """The weight gradient of one conv2d_resample backward, restated from its geometry: the position grid (PH x PW, PW the padded width
    rounded up to 8), K = N*PH*PW rounded up to 64, the wgrad_operand copies in launch order (source, channels, s, pad, ld, shift), the
    taps' (a_off, b_off, a_row, b_row) and the conv_wgrad plan.

    same (k x k, p = k // 2):  dy and the input on the (H + 2p) x (W + 2p) grid; tap (ky, kx) is the input copy shifted by kx - p
                               columns (row offset kx * Cin) at column offset (ky - p) * PW.
    down (3x3): dy on the (H/2 + 1)-row grid; the FIR output (H + 1)^2 split into 4 parity images at stride 2, copies shifted by 0 and
                1; tap (ky, kx) reads parity ((ky & 1), (kx & 1)) at row ky >> 1 of it, from copy kx >> 1.
    up (3x3): the input on the (H + 1)-row grid; the raw (2H + 1)^2 gradient split into parity images likewise.
    The 1x1 fast paths are 'same' 1x1 at the input size (post-upsample) or at the downsampled size (pre-downsample)."""
    kind = resample_kind(k, up, down)
    if kind == 'down1':
        H, W = (H - 2) // 2 + 1, (W - 2) // 2 + 1                    # downsample2d's output
    cout_g, cin_g = cout // groups, cin // groups
    taps = [(ky, kx) for ky in range(k) for kx in range(k)]
    zero = [0] * len(taps)
    if kind in ('same3', 'same1', 'up1', 'down1'):
        p = k // 2
        PH, PW, width = H + 2 * p, _r8(W + 2 * p), W + 2 * p
        Kp = cdiv(N * PH * PW, 64) * 64
        ops = [('dy', cout, 1, p, Kp, 0)] + [('x', cin, 1, p, Kp, kx - p) for kx in range(k)]
        a_off, a_row = zero, zero
        b_off, b_row = [(ky - p) * PW for ky, kx in taps], [kx * cin for ky, kx in taps]
    elif kind == 'down':
        PH, PW, width = H // 2 + 1, _r8(W // 2 + 1), W // 2 + 1
        Kp, block = cdiv(N * PH * PW, 64) * 64, N * PH * PW
        ops = [('dy', cout, 1, 0, Kp, 0), ('fir(x)', cin, 2, 0, 4 * block, 0), ('fir(x)', cin, 2, 0, 4 * block, 1)]
        a_off, a_row = zero, zero
        b_off = [((ky & 1) * 2 + (kx & 1)) * block + (ky >> 1) * PW for ky, kx in taps]
        b_row = [(kx >> 1) * cin for ky, kx in taps]
    else:
        PH, PW, width = H + 1, _r8(W + 1), W + 1
        Kp, block = cdiv(N * PH * PW, 64) * 64, N * PH * PW
        ops = [('fir(dy)', cout, 2, 0, 4 * block, 0), ('fir(dy)', cout, 2, 0, 4 * block, 1), ('x', cin, 1, 0, Kp, 0)]
        a_off = [((ky & 1) * 2 + (kx & 1)) * block + (ky >> 1) * PW for ky, kx in taps]
        a_row = [(kx >> 1) * cout for ky, kx in taps]
        b_off, b_row = zero, zero
    splits = wgrad_splits_mirror(groups, len(taps), cout_g, cin_g, Kp, sms)
    return dict(kind=kind, PH=PH, PW=PW, pw_exact=PW == width, positions=N * PH * PW, Kp=Kp, operands=ops, a_off=a_off, b_off=b_off,
                a_row=a_row, b_row=b_row, wgrad=wgrad_plan(groups, len(taps), cout_g, cin_g, Kp, splits, sms))


def launches(c, sms=SMS):
    """(kernel, grid) of every launch of a case that the profiler test matches, in launch order."""
    if c['op'] == 'wgrad':
        w = case_plan(c, sms)
        return [(w['kernel'], w['grid'])] + ([('wgrad_reduce_kernel', (w['reduce_grid'], 1, 1))] if w['splits'] > 1 else [])
    if c['op'] == 'operand':
        p = case_plan(c, sms)
        return [(p['kernel'], (p['grid'], 1, 1))]
    if c['op'] == 'bias_act':
        p = case_plan(c, sms)
        return [] if p is None else [(p['kernel'], (p['grid'], 1, 1))]
    p = case_plan(c, sms)
    w = p['wgrad']
    out = [('wgrad_operand_kernel', (operand_plan(C, ld, sms)['grid'], 1, 1)) for _, C, _, _, ld, _ in p['operands']]
    out.append((w['kernel'], w['grid']))
    if w['splits'] > 1:
        out.append(('wgrad_reduce_kernel', (w['reduce_grid'], 1, 1)))
    return out


# ------------------------------------------------------------------------------------------------ the case table
# n3d_conv_wgrad at the ABI.  offs: per tap (a_off, b_off, a_row, b_row); splits 'auto' = what kernels.wgrad_splits picks.
OFFS = [(-8, 24, 0, 8), (40, -64, 5, 0), (0, 96, 2, 16), (8, 16, 0, 24), (-128, 0, 1, 0), (64, 8, 3, 8), (16, -8, 0, 0), (-16, -16, 4, 16),
        (72, 8, 1, 24)]
A_EXTRA_ROWS, B_EXTRA_ROWS = 5, 24          # the largest a_row / b_row above


def _wg(name, G, M, N, T, K, a_cols, b_cols, splits):
    return dict(op='wgrad', name=name, G=G, M=M, N=N, T=T, K=K, a_cols=a_cols, b_cols=b_cols, splits=splits, offs=OFFS[:T])


WGRAD = [
    _wg('wgrad_tails_m130_n136', 1, 130, 136, 3, 640, 700, 640, 1),           # M and N tile tails, offsets past both ends
    _wg('wgrad_tails_s10', 1, 130, 136, 3, 640, 700, 640, 10),                 # every slice one K step
    _wg('wgrad_cout3_taps9', 5, 3, 8, 9, 1024, 1100, 1024, 4),                 # Cout = 3, narrow N, 9 taps
    _wg('wgrad_groups40', 40, 24, 32, 2, 128, 128, 200, 2),                    # many groups
    _wg('wgrad_1x1', 3, 64, 64, 1, 256, 256, 256, 1),                          # 1x1
    _wg('wgrad_k512sq', 1, 16, 16, 1, 512 * 512, 512 * 512, 512 * 512, 32),    # K = 512^2 positions
    _wg('wgrad_bn32_ring_full', 2, 40, 24, 2, 320, 320, 320, 1),               # ksteps == stages (5)
    _wg('wgrad_bn64_short', 1, 256, 40, 1, 192, 192, 256, 1),                  # ksteps < stages (4), M = 2 x 128
    _wg('wgrad_bn64_wrap', 1, 300, 64, 2, 1280, 1300, 1280, 1),                # 3 m-tiles, the ring wraps 4 times
    _wg('wgrad_bn128_ring_full', 2, 128, 72, 1, 192, 192, 192, 1),             # ksteps == stages (3)
    _wg('wgrad_bn128_uneven', 1, 128, 256, 1, 640, 640, 648, 3),               # slices of 4, 4, 2 steps
    _wg('wgrad_empty_slices', 1, 64, 64, 9, 5184, 5184, 5184, 'auto'),         # 81 steps, 10 slices of 9: the last one is empty
    _wg('wgrad_reduce_passes', 1, 512, 512, 9, 1408, 1408, 1408, 'auto'),      # 2 slices, 590k float4 to reduce
    _wg('wgrad_groups64', 64, 8, 16, 1, 128, 128, 128, 'auto'),                # G >= 64
    _wg('wgrad_group_straddle', 3, 100, 48, 2, 384, 400, 384, 'auto'),         # group 1's rows 100..199 straddle a 128-row tile
]

# n3d_wgrad_operand.  layout: nchw, cl (channels_last), cslice (a channel slice of a wider tensor), nslice (every other image).
# LAYOUT: the three layouts of one small tensor that the weight gradient was first written with, from an NCHW and a channels_last
# x (test_wgrad_operand_layout); OPERAND: the rest of the table.
LAYOUT = [dict(op='operand', name=f'operand_{name}_{lay}', N=2, C=5, H=7, W=6, s=s, pad=pad, PH=PH, PW=PW, shift=shift, layout=lay)
          for name, s, pad, PH, PW, shift in [('s1_p1_shm1', 1, 1, 9, 8, -1), ('s2_p0_sh1', 2, 0, 4, 4, 1), ('s1_p0_sh0', 1, 0, 7, 6, 0)]
          for lay in ('nchw', 'cl')]
OPERAND = [
    dict(op='operand', name='operand_s2_p2_cslice', N=2, C=5, H=10, W=12, s=2, pad=2, PH=8, PW=8, shift=0, layout='cslice'),
    dict(op='operand', name='operand_s1_p2_row_shift_nslice', N=3, C=4, H=9, W=11, s=1, pad=2, PH=13, PW=16, shift=19, layout='nslice'),
    dict(op='operand', name='operand_s2_p1_shm1_cl', N=1, C=6, H=9, W=7, s=2, pad=1, PH=6, PW=8, shift=-1, layout='cl'),
    dict(op='operand', name='operand_grid_stride', N=2, C=96, H=64, W=64, s=1, pad=1, PH=66, PW=72, shift=1, layout='nchw'),
]
for c in LAYOUT + OPERAND:
    c['ld'] = _r8(c['s'] ** 2 * c['N'] * c['PH'] * c['PW']) + 8


# conv2d_resample backward.  xcl / dycl: x / dy channels_last.
def _cv(name, N, cin, cout, H, W, k, up=1, down=1, groups=1, flip=True, dtype=torch.float32, xcl=False, dycl=False):
    return dict(op='conv', name=name, N=N, cin=cin, cout=cout, H=H, W=W, k=k, up=up, down=down, groups=groups, flip=flip, dtype=dtype,
                xcl=xcl, dycl=dycl)


F16 = torch.float16
CONV = [
    _cv('conv_same3_w6_k64', 1, 8, 8, 6, 6, 3),
    _cv('conv_same3_w14_g3', 2, 24, 30, 9, 14, 3, groups=3, flip=False),
    _cv('conv_same3_odd_f16_cl', 2, 16, 12, 7, 11, 3, dtype=F16, xcl=True, dycl=True),
    _cv('conv_same1_torgb_odd', 2, 16, 3, 11, 13, 1),
    _cv('conv_same1_w8_g3_k64', 1, 24, 9, 8, 8, 1, groups=3, flip=False, dtype=F16),
    _cv('conv_up3_w7_odd_k64', 1, 8, 16, 7, 7, 3, up=2, flip=False),
    _cv('conv_up3_w15_g3_cl', 1, 24, 12, 6, 15, 3, up=2, groups=3, xcl=True),        # the up-2 forward needs cout_g % 4 == 0
    _cv('conv_up3_w10_f16', 2, 16, 20, 9, 10, 3, up=2, dtype=F16, dycl=True),
    _cv('conv_down3_w14', 2, 16, 12, 10, 14, 3, down=2),
    _cv('conv_down3_w30_g3_f16_cl_k64', 1, 24, 24, 14, 30, 3, down=2, groups=3, flip=False, dtype=F16, xcl=True, dycl=True),
    _cv('conv_down3_w12_torgb', 2, 8, 3, 8, 12, 3, down=2, flip=False),
    _cv('conv_up1_torgb_odd', 2, 16, 3, 7, 9, 1, up=2),
    _cv('conv_up1_w16_g3_f16_cl_k64', 1, 24, 12, 8, 16, 1, up=2, groups=3, flip=False, dtype=F16, xcl=True, dycl=True),
    _cv('conv_down1_torgb', 2, 16, 3, 14, 18, 1, down=2, flip=False),
    _cv('conv_down1_odd_w17_g3_cl', 1, 24, 9, 9, 17, 1, down=2, groups=3, xcl=True),
    # production layers
    _cv('conv_prod_same3_c512_64', 1, 512, 512, 64, 64, 3),
    _cv('conv_prod_up3_c128_128', 1, 128, 128, 128, 128, 3, up=2, flip=False),
    _cv('conv_prod_torgb_c128_256', 1, 128, 3, 256, 256, 1),
]

# n3d_bias_act_grad at the ABI.  act: (cuda index, default alpha, default gain); acts 4-9 have grad mode 2 and save x and b, 2-8
# differentiate from the saved output, 9 (swish) from the saved input.
ACTS = {'linear': (1, 0.0, 1.0), 'relu': (2, 0.0, math.sqrt(2)), 'lrelu': (3, 0.2, math.sqrt(2)), 'tanh': (4, 0.0, 1.0),
        'sigmoid': (5, 0.0, 1.0), 'elu': (6, 0.0, 1.0), 'selu': (7, 0.0, 1.0), 'softplus': (8, 0.0, 1.0), 'swish': (9, 0.0, math.sqrt(2))}
SELU_S, SELU_A = 1.0507009873554805, 1.6732632423543772


def _ba(name, act, grad, dtype, cl, shape=(2, 12, 9, 7), dim=1, gain=None, clamp=None):
    idx, alpha, dgain = ACTS[act]
    smooth = act not in ('linear', 'relu', 'lrelu', 'swish')
    if gain is None:
        gain = (0.5 if cl else 1.0) if smooth else dgain
    if clamp is None:
        clamp = 0.75 * gain if smooth else 0.75 if act != 'swish' else 2.0
    return dict(op='bias_act', name=name, act=act, grad=grad, dtype=dtype, cl=cl, shape=shape, dim=dim, gain=gain, clamp=clamp, alpha=alpha)


BIAS_ACT = [_ba(f'ba_{act}_g{grad}_{"f32" if dt == torch.float32 else "f16"}_{"cl" if cl else "nchw"}', act, grad, dt, cl)
            for act in ACTS for grad in ((1, 2) if ACTS[act][0] >= 4 else (1,)) for dt in (torch.float32, F16) for cl in (False, True)] + [
    _ba('ba_swish_bias_dim0', 'swish', 1, torch.float32, False, dim=0, clamp=-1.0),
    _ba('ba_swish_bias_dim2_cl', 'swish', 1, torch.float32, True, dim=2, clamp=-1.0),
    _ba('ba_swish_bias_dim3_f16', 'swish', 2, F16, False, dim=3),
    _ba('ba_tanh_bias_dim3_cl', 'tanh', 2, torch.float32, True, dim=3),
    _ba('ba_swish_no_bias', 'swish', 1, torch.float32, False, dim=None),
    _ba('ba_selu_no_bias_f16', 'selu', 2, F16, True, dim=None, clamp=-1.0),
    _ba('ba_numel0', 'tanh', 1, torch.float32, False, shape=(0, 12, 9, 7)),
    _ba('ba_grid_swish', 'swish', 1, torch.float32, False, shape=(3, 37, 61, 41)),
    _ba('ba_grid_tanh_f16_cl', 'tanh', 2, F16, True, shape=(3, 37, 61, 41)),
]

CASES = WGRAD + OPERAND + CONV + BIAS_ACT        # test_kernel_matches_fp64_reference, one parameter set each
CASE_IDS = [c['name'] for c in CASES]
TABLE = WGRAD + LAYOUT + OPERAND + CONV + BIAS_ACT  # everything the coverage, memory and profiler tests see; the seed is the index here
TABLE_IDS = [c['name'] for c in TABLE]


def case_plan(c, sms=SMS):
    if c['op'] == 'wgrad':
        splits = wgrad_splits_mirror(c['G'], c['T'], c['M'], c['N'], c['K'], sms) if c['splits'] == 'auto' else c['splits']
        return wgrad_plan(c['G'], c['T'], c['M'], c['N'], c['K'], splits, sms)
    if c['op'] == 'operand':
        return operand_plan(c['C'], c['ld'], sms)
    if c['op'] == 'bias_act':
        return bias_act_grad_plan(math.prod(c['shape']), c['dtype'], sms)
    return resample_plan(c['N'], c['cin'], c['cout'], c['H'], c['W'], c['k'], c['up'], c['down'], c['groups'], sms)


def saves_input(act):
    """The autograd Function saves x and b (and passes them to the gradient) for the activations with a second derivative."""
    return ACTS[act][0] >= 4


def reads_output(act):
    return 2 <= ACTS[act][0] <= 8


def _one_ulp_in(v, dtype):
    """The value of `dtype` one ulp closer to zero than v (v > 0 and exact in dtype)."""
    it = torch.int32 if dtype == torch.float32 else torch.int16
    return (torch.tensor(v, dtype=dtype).view(it) - 1).view(dtype).item()


def _inverse(act, t, alpha):
    """The pre-activation whose activation (without gain) is t, or None when no input reaches t."""
    if act == 'linear':
        return t
    if act == 'relu':
        return t if t > 0 else None
    if act == 'lrelu':
        return t if t > 0 else t / alpha
    if act == 'tanh':
        return math.atanh(t) if abs(t) < 1 else None
    if act == 'sigmoid':
        return math.log(t / (1 - t)) if 0 < t < 1 else None
    if act == 'elu':
        return t if t >= 0 else (math.log1p(t) if t > -1 else None)
    if act == 'selu':
        return t / SELU_S if t >= 0 else (math.log1p(t / (SELU_S * SELU_A)) if t > -SELU_S * SELU_A else None)
    if act == 'softplus':
        return math.log(math.expm1(t)) if t > 0 else None
    return None


def edges(c):
    """The special elements of a bias_act case: [(what, pre-activation target, saved output or None)].  'clamp' / 'ulp': a saved output
    exactly at +-clamp / one ulp inside it; 'zero': x + b exactly 0; 'tail': swish x + b > 40 or < -80, softplus x + b > 20."""
    act, out = c['act'], []
    if math.prod(c['shape']) == 0:
        return out
    if act in ('relu', 'lrelu', 'elu', 'selu'):
        out.append(('zero', 0.0, None))
    if act == 'swish':
        out += [('tail', v, None) for v in (41.0, 60.0, 100.0, -81.0, -90.0, -100.0)]
    if act == 'softplus':
        out += [('tail', v, None) for v in (25.0, 30.0)]
    if reads_output(act) and c['clamp'] >= 0:
        cl = c['clamp']
        for what, y in [('clamp', cl), ('ulp', _one_ulp_in(cl, c['dtype']))]:
            for sgn in (1.0, -1.0):
                pre = _inverse(act, sgn * y / c['gain'], c['alpha'])
                if pre is not None:
                    out.append((what, pre, sgn * y))
    return out


def _any(cs, op, pred):
    return any(pred(c, p) for c, p in cs if c['op'] == op)


def _wgrad_cover():
    items = {}
    for bn, stages in ((32, 5), (64, 4), (128, 3)):
        w = lambda cs, bn=bn: [(c, p) for c, p in cs if c['op'] == 'wgrad' and p['block_n'] == bn]       # noqa: E731
        items[f'conv_wgrad_kernel<{bn}> with {stages} stages'] = lambda cs, w=w, s=stages: bool(w(cs)) and all(p['stages'] == s for c, p in w(cs))
        items[f'conv_wgrad_kernel<{bn}>: a slice shorter than the ring'] = lambda cs, w=w: any(p['longest'] < p['stages'] for c, p in w(cs))
        items[f'conv_wgrad_kernel<{bn}>: a slice exactly the ring'] = lambda cs, w=w: any(p['longest'] == p['stages'] for c, p in w(cs))
        items[f'conv_wgrad_kernel<{bn}>: a ring that wraps 3 times'] = lambda cs, w=w: any((p['longest'] - 1) // p['stages'] >= 3 for c, p in w(cs))
        items[f'conv_wgrad_kernel<{bn}>: a partial last n-tile'] = lambda cs, w=w, bn=bn: any(c['N'] % bn for c, p in w(cs))
    return items


def _wgrad_straddles(c):
    return c['G'] > 1 and any((g * c['M']) // KBM != (g * c['M'] + c['M'] - 1) // KBM for g in range(1, c['G']))


def _conv_kinds(cs):
    return [(c, p) for c, p in cs if c['op'] == 'conv']


KINDS = ('same3', 'same1', 'up', 'down', 'up1', 'down1')

COVERAGE = {
    **_wgrad_cover(),
    'M < 8': lambda cs: _any(cs, 'wgrad', lambda c, p: c['M'] < 8),
    'M % 128 != 0 and M a multiple of 128': lambda cs: _any(cs, 'wgrad', lambda c, p: c['M'] % 128) and _any(cs, 'wgrad', lambda c, p: c['M'] % 128 == 0),
    'more than 2 m-tiles': lambda cs: _any(cs, 'wgrad', lambda c, p: p['m_tiles'] > 2),
    'N an exact multiple of block_n': lambda cs: _any(cs, 'wgrad', lambda c, p: c['N'] % p['block_n'] == 0),
    'splits = 1': lambda cs: _any(cs, 'wgrad', lambda c, p: p['splits'] == 1),
    'split K with every slice full': lambda cs: _any(cs, 'wgrad', lambda c, p: p['splits'] > 1 and p['ksteps'] == p['splits'] * p['longest']),
    'split K with an uneven last slice': lambda cs: _any(cs, 'wgrad', lambda c, p: p['splits'] > 1 and 0 < p['last'] < p['longest']),
    'empty trailing slices at the splits wgrad_splits picks': lambda cs: _any(cs, 'wgrad', lambda c, p: c['splits'] == 'auto' and any(p['empty'])),
    'a reduction of more than one grid-stride pass': lambda cs: _any(cs, 'wgrad', lambda c, p: p['reduce_passes'] > 1),
    'T = 1, 2 and 9': lambda cs: {c['T'] for c, p in cs if c['op'] == 'wgrad'} >= {1, 2, 9},
    'G = 1, G >= 64, G > 1 with group rows straddling a tile': lambda cs: _any(cs, 'wgrad', lambda c, p: c['G'] == 1)
        and _any(cs, 'wgrad', lambda c, p: c['G'] >= 64) and _any(cs, 'wgrad', lambda c, p: _wgrad_straddles(c)),
    'negative column offsets': lambda cs: _any(cs, 'wgrad', lambda c, p: any(o[0] < 0 for o in c['offs']) and any(o[1] < 0 for o in c['offs'])),
    'column offsets past a_cols and b_cols': lambda cs: _any(cs, 'wgrad', lambda c, p: any(o[0] + c['K'] > c['a_cols'] for o in c['offs']))
        and _any(cs, 'wgrad', lambda c, p: any(o[1] + c['K'] > c['b_cols'] for o in c['offs'])),
    'non-zero row offsets': lambda cs: _any(cs, 'wgrad', lambda c, p: any(o[2] for o in c['offs']) and any(o[3] for o in c['offs'])),
    # conv2d_resample backward
    'every conv2d_resample kind with flip_weight both ways': lambda cs: {(p['kind'], c['flip']) for c, p in _conv_kinds(cs)}
        == {(k, f) for k in KINDS for f in (False, True)},
    'groups 1 and 3': lambda cs: {c['groups'] for c, p in _conv_kinds(cs)} >= {1, 3},
    'cout_g = 3 and a cout_g not a multiple of 8': lambda cs: {c['cout'] // c['groups'] == 3 for c, p in _conv_kinds(cs)} == {True, False}
        and any(c['cout'] // c['groups'] % 8 for c, p in _conv_kinds(cs) if c['cout'] // c['groups'] != 3),
    'cin_g = 8': lambda cs: any(c['cin'] // c['groups'] == 8 for c, p in _conv_kinds(cs)),
    'for each kind, PW exactly the padded width and not': lambda cs: {(p['kind'], p['pw_exact']) for c, p in _conv_kinds(cs)}
        == {(k, e) for k in KINDS for e in (False, True)},
    'N*PH*PW a multiple of 64 and not': lambda cs: {p['positions'] % 64 == 0 for c, p in _conv_kinds(cs)} == {True, False},
    'odd H and W on same 3x3, same 1x1, up 3x3 and the 1x1 paths': lambda cs: {p['kind'] for c, p in _conv_kinds(cs) if c['H'] % 2 and c['W'] % 2}
        >= {'same3', 'same1', 'up', 'up1', 'down1'},
    'conv2d_resample fp32 and fp16': lambda cs: {c['dtype'] for c, p in _conv_kinds(cs)} == {torch.float32, F16},
    'x and dy NCHW and channels_last': lambda cs: {c['xcl'] for c, p in _conv_kinds(cs)} == {False, True} and {c['dycl'] for c, p in _conv_kinds(cs)} == {False, True},
    'production layers: 512-channel 3x3 at 64^2, 128-channel up-2 at 128^2, 3-channel 1x1 ToRGB at 256^2': lambda cs: {
        (p['kind'], c['cin'], c['cout'], c['H']) for c, p in _conv_kinds(cs)} >= {('same3', 512, 512, 64), ('up', 128, 128, 128), ('same1', 128, 3, 256)},
    # wgrad_operand (with LAYOUT)
    'operand s 1 and 2': lambda cs: {c['s'] for c, p in cs if c['op'] == 'operand'} == {1, 2},
    'operand pads 0, 1, 2': lambda cs: {c['pad'] for c, p in cs if c['op'] == 'operand'} == {0, 1, 2},
    'operand shifts -1, 0, +1 and past a row': lambda cs: {c['shift'] for c, p in cs if c['op'] == 'operand'} >= {-1, 0, 1}
        and any(c['shift'] > c['PW'] for c, p in cs if c['op'] == 'operand'),
    'operand x NCHW, channels_last, a channel slice, a batch slice': lambda cs: {c['layout'] for c, p in cs if c['op'] == 'operand'}
        == {'nchw', 'cl', 'cslice', 'nslice'},
    'operand grid-stride': lambda cs: _any(cs, 'operand', lambda c, p: p['passes'] > 1),
    # bias_act_grad
    'every act x grad mode x dtype x layout': lambda cs: {(c['act'], c['grad'], c['dtype'], c['cl']) for c, p in cs if c['op'] == 'bias_act'}
        == {(a, g, d, l) for a in ACTS for g in ((1, 2) if ACTS[a][0] >= 4 else (1,)) for d in (torch.float32, F16) for l in (False, True)},
    'a bias along dims 0-3 and no bias': lambda cs: {c['dim'] for c, p in cs if c['op'] == 'bias_act' and saves_input(c['act'])} >= {0, 1, 2, 3, None},
    'outputs exactly at +-clamp and one ulp inside, for every act that reads its output': lambda cs: all(
        any(c['act'] == a and {(w, y > 0) for w, _, y in edges(c) if y is not None} >= {('clamp', True), ('ulp', True)} for c, p in cs
            if c['op'] == 'bias_act') for a in ACTS if reads_output(a)) and any(
        {(w, y > 0) for w, _, y in edges(c) if y is not None} == {(w, s) for w in ('clamp', 'ulp') for s in (False, True)} for c, p in cs
        if c['op'] == 'bias_act'),
    'swish at x > 40 and x < -80, softplus at y > 20': lambda cs: any(c['act'] == 'swish' and {t > 40 for w, t, _ in edges(c) if w == 'tail'}
        == {True, False} for c, p in cs if c['op'] == 'bias_act') and any(c['act'] == 'softplus' and any(w == 'tail' for w, _, _ in edges(c))
                                                                           for c, p in cs if c['op'] == 'bias_act'),
    'elu, selu, relu, lrelu at exactly 0': lambda cs: {c['act'] for c, p in cs if c['op'] == 'bias_act' and any(w == 'zero' for w, _, _ in edges(c))}
        == {'elu', 'selu', 'relu', 'lrelu'},
    'numel 0 launches nothing': lambda cs: any(c['op'] == 'bias_act' and p is None for c, p in cs),
    'bias_act_grad grid-stride with numel % 256 != 0': lambda cs: _any(cs, 'bias_act', lambda c, p: p is not None and p['passes'] > 1
                                                                          and math.prod(c['shape']) % 256),
}


def case_bytes(c):
    """Device memory of a case: inputs, guarded outputs and the fp64 reference's tensors."""
    if c['op'] == 'wgrad':
        splits = case_plan(c)['splits']
        lda, ldb = _r8(c['a_cols']) + 8, _r8(c['b_cols'])
        ops = (c['G'] * c['M'] + A_EXTRA_ROWS) * lda * 4 + (c['G'] * c['N'] + B_EXTRA_ROWS) * ldb * 4          # fp32 source, bf16 hi + lo
        ref = 3 * c['G'] * (c['M'] + c['N']) * c['K'] * 8                    # fp64 shifted hi and lo operands and a transient copy
        return ops + ref + (splits + 2) * c['G'] * c['T'] * c['M'] * c['N'] * 8
    if c['op'] == 'operand':
        return c['N'] * c['C'] * c['H'] * c['W'] * 16 + c['C'] * c['ld'] * 24
    if c['op'] == 'bias_act':
        return math.prod(c['shape']) * 8 * 12
    s = 2 if c['up'] == 2 else 1
    big = c['N'] * max(c['cin'], c['cout']) * (s * c['H'] + 4) * (s * c['W'] + 4)
    return 6 * 8 * big                          # fp64 output, the zero-inserted / raw / FIR intermediates and their gradients


def test_case_table_covers_every_launch_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rules, at <= 512 MB per case."""
    planned = [(c, case_plan(c)) for c in TABLE]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(TABLE_IDS)) == len(TABLE_IDS)
    big = {c['name']: case_bytes(c) / 2 ** 20 for c in TABLE if case_bytes(c) > 512 * 2 ** 20}
    assert not big, big


def test_mirror_examples():
    """CPU: the mirror at the examples the launch rules were written down with."""
    p = resample_plan(1, 64, 64, 70, 70, 3, 1, 1, 1)                      # x [1, 64, 70, 70], 3x3 same
    assert (p['PH'], p['PW'], p['Kp']) == (72, 72, 5184)
    assert p['wgrad']['splits'] == 10 and p['wgrad']['slices'][-1] == (81, 81) and p['wgrad']['empty'] == [False] * 9 + [True]
    p = resample_plan(1, 512, 512, 32, 32, 3, 1, 1, 1)['wgrad']
    assert p['splits'] == 2 and p['reduce_grid'] == SMS * 8 and p['reduce_passes'] == 3
    assert [wgrad_plan(1, 1, 128, n, 64, 1)['stages'] for n in (32, 64, 128)] == [5, 4, 3]


# ------------------------------------------------------------------------------------------------ inputs and launches
def _gen(c):
    return torch.Generator(device=DEV).manual_seed(3000 + TABLE_IDS.index(c['name']))


def _kernels():
    from next3d_b200 import kernels as K
    return K


def setup_wgrad(c):
    K = _kernels()
    g = _gen(c)
    p = case_plan(c, torch.cuda.get_device_properties(0).multi_processor_count)
    G, M, N, T = c['G'], c['M'], c['N'], c['T']
    lda, ldb = _r8(c['a_cols']) + 8, _r8(c['b_cols'])
    a_hi, a_lo = K.split_bf16(torch.randn(G * M + A_EXTRA_ROWS, lda, device=DEV, generator=g))
    b_hi, b_lo = K.split_bf16(torch.randn(G * N + B_EXTRA_ROWS, ldb, device=DEV, generator=g))
    s = dict(c=c, plan=p, a=(a_hi, a_lo), b=(b_hi, b_lo), dw=Guarded((G, T, M, N)),
             partial=Guarded((p['splits'], G, T, M, N)) if p['splits'] > 1 else None)
    return s


def launch_wgrad(s):
    c = s['c']
    o = c['offs']
    _kernels().conv_wgrad(*s['a'], *s['b'], c['G'], c['M'], c['N'], c['K'], [t[0] for t in o], [t[1] for t in o], s['dw'].view,
                          splits=s['plan']['splits'], partial=s['partial'].view if s['partial'] else None, a_cols=c['a_cols'],
                          b_cols=c['b_cols'], a_row=[t[2] for t in o], b_row=[t[3] for t in o])


def _shifted(t, off, cols, K):
    """t [rows, ld] -> [rows, K]: column k holds t[:, k + off] for 0 <= k + off < cols, else 0."""
    out = torch.zeros(t.shape[0], K, dtype=t.dtype, device=t.device)
    lo, hi = max(0, -off), min(K, cols - off)
    if hi > lo:
        out[:, lo:hi] = t[:, lo + off:hi + off]
    return out


def check_wgrad(s):
    c = s['c']
    G, M, N, K = c['G'], c['M'], c['N'], c['K']
    e = RangeErr()
    for t, (ao, bo, ar, br) in enumerate(c['offs']):
        sa = [_shifted(u[ar:ar + G * M].double(), ao, c['a_cols'], K).view(G, M, K) for u in s['a']]
        sb = [_shifted(u[br:br + G * N].double(), bo, c['b_cols'], K).view(G, N, K).transpose(1, 2) for u in s['b']]
        ref = torch.bmm(sa[0], sb[0]) + torch.bmm(sa[0], sb[1]) + torch.bmm(sa[1], sb[0])
        e.add(s['dw'].view[:, t], ref)
        del sa, sb, ref
    return {'wgrad': (e.value(), wgrad_scale(s['plan']['longest']))}


def _operand_source(c, g):
    N, C, H, W, lay = c['N'], c['C'], c['H'], c['W'], c['layout']
    if lay == 'cslice':
        return torch.randn(N, C + 4, H, W, device=DEV, generator=g)[:, 2:2 + C]
    if lay == 'nslice':
        return torch.randn(2 * N, C, H, W, device=DEV, generator=g)[::2]
    x = torch.randn(N, C, H, W, device=DEV, generator=g)
    return x.contiguous(memory_format=torch.channels_last) if lay == 'cl' else x


def setup_operand(c):
    return dict(c=c, x=_operand_source(c, _gen(c)), hi=Guarded((c['C'], c['ld']), torch.bfloat16), lo=Guarded((c['C'], c['ld']), torch.bfloat16))


def launch_operand(s):
    c = s['c']
    _kernels().wgrad_operand(s['x'], c['s'], c['pad'], c['pad'], c['PH'], c['PW'], c['ld'], s['hi'].view, s['lo'].view, shift=c['shift'])


def operand_reference(x, s, pad, PH, PW, shift, ld):
    """fp32 [C, ld]: column j holds x[n, :, s*(py - pad) + par // s, s*(px - pad) + par % s] for the grid position j + shift =
    ((par * N + n) * PH + py) * PW + px, and 0 where that position is outside the grid or its pixel outside x -> (values, valid)."""
    N, C, H, W = x.shape
    used = s * s * N * PH * PW
    j = torch.arange(ld, device=x.device) + shift
    valid = (j >= 0) & (j < used)
    jj = j.clamp(0, used - 1)
    px, r = jj % PW, jj // PW
    py, r = r % PH, r // PH
    n, par = r % N, r // N
    iy, ix = s * (py - pad) + par // s, s * (px - pad) + par % s
    valid &= (iy >= 0) & (iy < H) & (ix >= 0) & (ix < W)
    v = x[n, :, iy.clamp(0, H - 1), ix.clamp(0, W - 1)]            # [ld, C]
    return torch.where(valid[:, None], v, torch.zeros((), device=x.device)).T.contiguous(), valid


def check_operand(s):
    """Bit-exact: hi and lo are split_bf16 of the gathered operand; padding and shifted-out columns hold +0."""
    c = s['c']
    ref, valid = operand_reference(s['x'], c['s'], c['pad'], c['PH'], c['PW'], c['shift'], c['ld'])
    for got, want in zip((s['hi'], s['lo']), _kernels().split_bf16(ref)):
        bits, wbits = got.bits(), want.view(torch.int16)
        assert torch.equal(bits, wbits), f'{c["name"]}: {int((bits != wbits).sum())} elements differ from split_bf16 of the gathered operand'
        assert (bits[:, ~valid] == 0).all(), f'{c["name"]}: a padding column is not +0'
    assert valid.any() and (~valid).any()
    return {}


def conv_inputs(c):
    g = _gen(c)
    N, cin, cout, H, W, k = c['N'], c['cin'], c['cout'], c['H'], c['W'], c['k']
    x = torch.randn(N, cin, H, W, device=DEV, generator=g).to(c['dtype'])
    w = (torch.randn(cout, cin // c['groups'], k, k, device=DEV, generator=g) / math.sqrt(cin // c['groups'] * k * k)).to(c['dtype'])
    if c['xcl']:
        x = x.contiguous(memory_format=torch.channels_last)
    OH, OW = (2 * H, 2 * W) if c['up'] == 2 else ((H - 2) // 2 + 1, (W - 2) // 2 + 1) if c['down'] == 2 else (H, W)
    dy = torch.randn(N, cout, OH, OW, device=DEV, generator=g).to(c['dtype'])
    if c['dycl']:
        dy = dy.contiguous(memory_format=torch.channels_last)
    return dict(c=c, x=x, w=w, dy=dy, kw=dict(up=c['up'], down=c['down'], padding=k // 2, groups=c['groups'], flip_weight=c['flip']))


def run_conv(s):
    """conv2d_resample forward and backward -> (y, dx, dw)."""
    from next3d_b200.torch_utils.ops import conv2d_resample as cr
    from oracle import ops as oo
    xg, wg = s['x'].clone().requires_grad_(), s['w'].clone().requires_grad_()
    y = cr.conv2d_resample(xg, wg, f=oo.setup_filter().to(DEV), **s['kw'])
    dx, dw = torch.autograd.grad(y, [xg, wg], s['dy'])
    return y.detach(), dx, dw


def check_conv(s):
    from next3d_b200 import kernels as K
    from oracle import ops as oo
    c = s['c']
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    p = case_plan(c, sms)
    w = p['wgrad']
    assert w['splits'] == K.wgrad_splits(c['groups'], w['grid'][1], c['cout'] // c['groups'], c['cin'] // c['groups'], p['Kp']), c['name']
    y, dx, dw = run_conv(s)
    assert y.dtype == dx.dtype == dw.dtype == c['dtype'] and dx.shape == s['x'].shape and dw.shape == s['w'].shape
    x64, w64 = s['x'].double().requires_grad_(), s['w'].double().requires_grad_()
    y64 = oo.conv2d_resample(x64, w64, f=oo.setup_filter().to(DEV, F64), **s['kw'])
    dx64, dw64 = torch.autograd.grad(y64, [x64, w64], s['dy'].double())
    pre = 'conv' if c['dtype'] == torch.float32 else 'conv16'
    errs = {f'{pre}.y': (range_rel_err(y, y64.detach()), 1.0), f'{pre}.dx': (range_rel_err(dx, dx64), 1.0),
            f'{pre}.dw': (range_rel_err(dw, dw64), wgrad_scale(w['longest']))}
    del x64, w64, y64, dx64, dw64
    for a, b in zip((y, dx, dw), run_conv(s)):
        assert torch.equal(a, b), f'{c["name"]}: a rerun is not bit-identical'
    return errs


def _storage(t, cl):
    """The elements of a dense 4-D tensor in storage order."""
    return (t.permute(0, 2, 3, 1) if cl else t).reshape(-1)


def setup_bias_act(c):
    """The tensors the autograd Function saves and the gradient launch reads, in the case's layout, with the edge elements placed."""
    from next3d_b200.torch_utils.ops import bias_act as BA
    g = _gen(c)
    dt, shape, dim = c['dtype'], c['shape'], c['dim']
    fmt = torch.channels_last if c['cl'] else torch.contiguous_format
    x = (torch.randn(shape, device=DEV, generator=g) * 2).to(dt)
    b = torch.randn(shape[dim], device=DEV, generator=g).to(dt) if dim is not None else None
    dy = torch.randn(shape, device=DEV, generator=g).to(dt)
    dyref = torch.randn(shape, device=DEV, generator=g).to(dt)
    bfull = b.double().reshape([-1 if i == dim else 1 for i in range(4)]).expand(shape) if b is not None else torch.zeros(shape, device=DEV, dtype=F64)
    marks = []
    for i, (what, pre, yv) in enumerate(edges(c)):
        at = tuple(int(v) for v in np.unravel_index(5 + 37 * i, shape))
        if what == 'zero':
            x[at] = -b[at[dim]] if b is not None else 0.0                 # x + b exactly 0
        else:
            x[at] = pre - bfull[at].item()
        marks.append((what, at, yv))
    x, dy, dyref = (t.contiguous(memory_format=fmt) for t in (x, dy, dyref))
    with torch.no_grad():
        y = BA.bias_act(x, b, dim=dim if dim is not None else 1, act=c['act'], alpha=c['alpha'], gain=c['gain'], clamp=c['clamp'])
    for what, at, yv in marks:
        if yv is not None:
            y[at] = yv                                                 # exactly +-clamp, or one ulp inside
    numel = math.prod(shape)
    return dict(c=c, x=x, b=b, bfull=bfull, y=y, dy=dy, dyref=dyref, marks=marks, dx=Guarded((numel,), dt))


def launch_bias_act(s):
    from next3d_b200 import _lib
    c = s['c']
    keep = saves_input(c['act'])
    b = s['b'] if keep else None
    size_b = step_b = 0
    if b is not None:
        size_b, step_b = b.shape[0], max(int(s['dy'].stride(c['dim'])), 1)
    _lib.check(_lib.lib.n3d_bias_act_grad(s['dy'].data_ptr(), _lib.ptr(b), _lib.ptr(s['x'] if keep else None),
                                          _lib.ptr(s['y'] if reads_output(c['act']) else None), _lib.ptr(s['dyref'] if c['grad'] == 2 else None),
                                          s['dx'].view.data_ptr(), 0 if c['dtype'] == torch.float32 else 1, math.prod(c['shape']), size_b, step_b,
                                          c['grad'], ACTS[c['act']][0], c['alpha'], c['gain'], c['clamp'], _lib.stream_ptr()), 'n3d_bias_act_grad')


def bias_act_reference(s):
    """fp64 grad mode 1 (dy * act'(x + b) * gain) or 2 (dy * dyref * act''(x + b) * gain), times the plugin's clamp mask."""
    from oracle import ops as oo
    c = s['c']
    act = c['act']
    xr = s['x'].double() + s['bfull']
    if act in ('elu', 'selu'):
        xr = torch.where(xr == 0, torch.full_like(xr, 1e-300), xr)      # the plugin's branch at the kink: yy >= 0
    xr.requires_grad_()
    yk = oo.bias_act(xr, None, act=act, alpha=c['alpha'], gain=c['gain'])
    d1, = torch.autograd.grad(yk.sum(), xr, create_graph=c['grad'] == 2)
    if c['grad'] == 2:
        d, = torch.autograd.grad(d1.sum(), xr)
        ref = s['dy'].double() * s['dyref'].double() * d
    else:
        ref = s['dy'].double() * d1.detach()
    cl = torch.tensor(c['clamp'], dtype=torch.float32)
    if c['clamp'] >= 0 and act != 'linear':                                 # linear saves no output: its gradient is not masked
        if act == 'swish':                                                  # the output recomputed in fp32 from x + b, as the kernel does
            x32 = s['x'].float() + s['bfull'].float()
            yr = torch.where(x32 < -80, torch.zeros_like(x32), x32 / (torch.exp(-x32) + 1) * c['gain'])
        else:
            yr = s['y'].float()
        ref = torch.where((yr > -cl) & (yr < cl), ref, torch.zeros_like(ref))
    return ref.detach()


def check_bias_act(s):
    c = s['c']
    if math.prod(c['shape']) == 0:
        return {}
    ref = bias_act_reference(s)
    got = s['dx'].view
    want = _storage(ref.contiguous(memory_format=torch.channels_last if c['cl'] else torch.contiguous_format), c['cl'])
    mask_out = _storage(((s['y'].float() <= -c['clamp']) | (s['y'].float() >= c['clamp'])).contiguous(
        memory_format=torch.channels_last if c['cl'] else torch.contiguous_format), c['cl']) if reads_output(c['act']) and c['clamp'] >= 0 else None
    if mask_out is not None:
        assert (got[mask_out].float() == 0).all(), f'{c["name"]}: an element whose saved output is on or outside +-clamp has a gradient'
    for what, at, yv in s['marks']:
        if what == 'ulp':                                                   # one ulp inside the clamp: the gradient passes
            assert (got[_flat(at, c)] != 0) == (ref[at] != 0), (c['name'], what, at)
    kind = f'ba{c["grad"]}.{"f32" if c["dtype"] == torch.float32 else "f16"}'
    return {kind: (range_rel_err(got, want), 1.0)}


def _flat(at, c):
    n, ch, h, w = at
    N, C, H, W = c['shape']
    return ((n * H + h) * W + w) * C + ch if c['cl'] else ((n * C + ch) * H + h) * W + w


SETUP = {'wgrad': setup_wgrad, 'operand': setup_operand, 'conv': conv_inputs, 'bias_act': setup_bias_act}
LAUNCH = {'wgrad': launch_wgrad, 'operand': launch_operand, 'conv': run_conv, 'bias_act': launch_bias_act}
CHECK = {'wgrad': check_wgrad, 'operand': check_operand, 'conv': check_conv, 'bias_act': check_bias_act}


def outputs(s):
    op = s['c']['op']
    if op == 'wgrad':
        return [s['dw']] + ([s['partial']] if s['partial'] else [])
    if op == 'operand':
        return [s['hi'], s['lo']]
    return [s['dx']] if op == 'bias_act' else []


def check_case(c):
    """Launch a case, check its guarded outputs and its errors against BOUNDS, and rerun it bit-identically."""
    s = SETUP[c['op']](c)
    if c['op'] != 'conv':
        LAUNCH[c['op']](s)
        torch.cuda.synchronize()
        for t in outputs(s):
            assert t.untouched_ok(), f'{c["name"]}: an element outside the output was written'
            assert t.written(), f'{c["name"]}: an owned element was not written'
    errs = CHECK[c['op']](s)
    record_errors('N3D_GRAD_ERRORS', [{'case': c['name'], 'kind': k, 'err': e, 'scale': sc, 'bound': BOUNDS[k] * sc} for k, (e, sc) in errs.items()])
    bad = {k: (e, BOUNDS[k] * sc) for k, (e, sc) in errs.items() if not e < BOUNDS[k] * sc}
    assert not bad, bad
    if outputs(s):
        assert rerun_identical(outputs(s), lambda: LAUNCH[c['op']](s)), f'{c["name"]}: a rerun is not bit-identical'


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_kernel_matches_fp64_reference(c):
    check_case(c)


@pytest.mark.gpu
def test_wgrad_operand_layout():
    """n3d_wgrad_operand at s 1 and 2, pads 0 and 1, shifts -1, 0, +1 of one 2x5x7x6 tensor, NCHW and channels_last: hi and lo bit for
    bit split_bf16 of the gathered operand, +0 in the padding, nothing written outside [C, ld], the same bits on a rerun."""
    for c in LAYOUT:
        check_case(c)


@pytest.mark.gpu
def test_launched_kernels_match_plan(tmp_path):
    """Every case under torch.profiler: the kernel instances it launched and their grids are the ones the mirror predicts at the
    device's SM count; numel 0 launches nothing."""
    pattern = re.compile(r'conv_wgrad_kernel<\d+>|wgrad_reduce_kernel|wgrad_operand_kernel|bias_act_grad_kernel<(?:float|__half)>')
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def run():
        expected = []
        for c in TABLE:                     # one case at a time: the production layers do not fit in memory together
            s = SETUP[c['op']](c)
            torch.cuda.synchronize()
            LAUNCH[c['op']](s)
            torch.cuda.synchronize()
            expected += [(c['name'], k, g) for k, g in launches(c, sms)]
            del s
        return expected

    expected, events = launched_kernels(run, pattern, tmp_path)
    for (who, kernel, grid), e in zip(expected, events):
        assert pattern.search(e['name']).group(0) == kernel, (who, e['name'], kernel)
        got = e.get('args', {}).get('grid')
        if got is not None:
            assert tuple(got) == tuple(grid), (who, kernel, got, grid)


@pytest.mark.gpu
def test_conv2d_resample_refuses_odd_down2():
    """down = 2 with a 3x3 kernel needs an even input: an odd one is refused with an error that names the op."""
    from next3d_b200.torch_utils.ops import conv2d_resample as cr
    from oracle import ops as oo
    w = torch.randn(8, 8, 3, 3, device=DEV)
    for H, W in [(7, 8), (8, 9)]:
        with pytest.raises(RuntimeError, match='conv2d_resample: down=2 with a 3x3 kernel needs an even input size'):
            cr.conv2d_resample(torch.randn(1, 8, H, W, device=DEV), w, f=oo.setup_filter().to(DEV), down=2, padding=1)
