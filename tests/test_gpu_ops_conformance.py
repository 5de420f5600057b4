"""The forward kernels of ops_basic.cu against an fp64 reference, over a table of launches that reaches every launch configuration their
entry points can select:

    n3d_bias_act        bias_act_kernel<float | __half>: the 4-wide vector loop when x and y are aligned, the scalar loop for the rest
    n3d_upfirdn2d       upfirdn2d_kernel<float | __half>, walking the output ox-fastest (y_strides[3] == 1) or c-fastest; a 1-D filter
                        is two launches, horizontal then vertical, each with gain sqrt(gain), as torch_utils.ops.upfirdn2d makes them
    n3d_filtered_lrelu  flrelu_up_kernel<...> into an fp32 scratch, then flrelu_down_kernel<...>

The entry points are called directly, so that every output (and filtered_lrelu's scratch) is a view into a larger allocation filled
with a NaN sentinel: the elements a launch owns must be written, every other element must keep the sentinel's bits.  Each case is then
rerun and must be bit-identical.

References, in fp64 on the device from the stored input values:
- bias_act: oracle.ops.bias_act of the fp32 sum x + b the kernel forms (b rounded to x's dtype first, as the wrapper does), so that
  only the activation, gain and clamp are left to compare.  The error is counted in ulps of the output dtype at the reference value;
  below the smallest normal fp32 number an absolute error up to that number is accepted (expf overflows there, and the result is 0).
- upfirdn2d: oracle.ops.upfirdn2d.  For fp16 on the separable route the intermediate image is rounded to fp16, as the port's two
  launches store it.
- filtered_lrelu: oracle.ops.filtered_lrelu.
- An fp16 output is compared with the fp64 result rounded to fp16 once: the kernels accumulate in fp32 and round once.
- The FIR ops are measured as max |got - ref| / R, R the same reference evaluated on |x| with |f| (and |b|): the sum of the absolute
  terms, the scale-free bound of a dot product.  Where R is 0 (whole border rows under padding) the output must be exactly 0.

The second table runs torch_utils.ops (bias_act, upfirdn2d, filter2d, upsample2d, downsample2d, filtered_lrelu) on NCHW, channels_last
and non-dense inputs: the values against the same references, and the output layout, which must be x.suggest_memory_format() as the
reference's plugins allocate it.

`bias_act_plan`, `upfirdn2d_plan` and `filtered_lrelu_plan` mirror the launch rules in plain Python.  The CPU test checks that the table
covers everything in COVERAGE; the profiler test checks on the GPU that each case launched the kernel instances and grids the mirror
predicts.  The refusal tests at the end need no GPU: bad arguments must be refused before any device call.
"""
import math
import re

import pytest
import torch

from tests.helpers import Guarded, cdiv, grid_stride, launched_kernels, lib, offset_view, record_errors, refused, rerun_identical

DEV = 'cuda'
SMS = 132                   # SM count the table is planned at (H100 SXM)
F32, F16, F64 = torch.float32, torch.float16, torch.float64
CL = torch.channels_last
SQRT2 = math.sqrt(2.0)
DTYPE_ID = {F32: 0, F16: 1}
TINY32 = torch.finfo(F32).tiny

# Element-wise bounds, measured over both tables (the kernel launches and torch_utils.ops) on an H100 80GB HBM3 (700 W power limit);
# the worst case is given beside each.  N3D_OPS_ERRORS=<file> appends every measured error to that file as JSON lines.
# bias_act, fp32: ulps at the reference value, at most 4x the worst case.
# bias_act, fp16: 1 ulp for every activation.  The kernel rounds an fp32 result that is within a few fp32 ulps of the reference, so it
# lands on one of the two fp16 values around the reference: at most 1 ulp from the reference rounded once.
# FIR ops: max |got - ref| / R, at most 4x the worst case.  An fp16 output differs from the rounded reference only where the fp32
# result crosses an fp16 rounding boundary: by one fp16 ulp of that element, at most 2^-10 R.
BOUNDS = {
    'ba.f32.linear': 2.4,       # Worst: 0.60 (ba_linear_f32_vec)
    'ba.f32.relu': 2.9,         # Worst: 0.73 (ba_relu_f32_vec)
    'ba.f32.lrelu': 4.6,        # Worst: 1.14 (ba_grid_scalar_lrelu)
    'ba.f32.tanh': 7.2,         # Worst: 1.80 (ba_tanh_f32_vec)
    'ba.f32.sigmoid': 8.4,      # Worst: 2.10 (ba_sigmoid_f32_vec)
    'ba.f32.elu': 5.9,          # Worst: 1.48 (ba_elu_f32_scalar)
    'ba.f32.selu': 6.5,         # Worst: 1.62 (ba_selu_f32_vec)
    'ba.f32.softplus': 6.6,     # Worst: 1.66 (ba_softplus_f32_scalar)
    'ba.f32.swish': 13.0,       # Worst: 3.26 (ba_grid_vec_swish)
    'ba.f16.linear': 1.0, 'ba.f16.relu': 1.0, 'ba.f16.lrelu': 1.0, 'ba.f16.elu': 1.0, 'ba.f16.selu': 1.0,    # Worst: 0 (each)
    'ba.f16.softplus': 1.0,     # Worst: 0
    'ba.f16.tanh': 1.0,         # Worst: 1 (ba_grid_vec_tanh_f16_cl)
    'ba.f16.sigmoid': 1.0,      # Worst: 1 (ba_sigmoid_f16_vec)
    'ba.f16.swish': 1.0,        # Worst: 1 (ba_swish_f16_vec)
    'fir.f32': 9e-7,            # Worst: 2.2e-7 (up_grid_1d8)
    'fir.f16': 3.3e-3,          # Worst: 8.3e-4 (up_grid_f16_cl)
    'flrelu.f32': 7.8e-7,       # Worst: 1.95e-7 (fl_grid)
    'flrelu.f16': 1.3e-5,       # Worst: 3.4e-6 (w_filtered_lrelu_cslice_cl_f16; 0 on every kernel-table case)
}

# name -> (cuda index, default alpha, default gain)                     torch_utils/ops/bias_act.py:23-33
ACTS = {'linear': (1, 0.0, 1.0), 'relu': (2, 0.0, SQRT2), 'lrelu': (3, 0.2, SQRT2), 'tanh': (4, 0.0, 1.0), 'sigmoid': (5, 0.0, 1.0),
        'elu': (6, 0.0, 1.0), 'selu': (7, 0.0, 1.0), 'softplus': (8, 0.0, 1.0), 'swish': (9, 0.0, SQRT2)}
# pre-activations placed in every bias_act case: the saturated regions of each activation
SATURATED = {'tanh': (10.0, -10.0, 20.0, -20.0), 'sigmoid': (30.0, -20.0, -40.0, -87.0, -100.0), 'elu': (-20.0, -50.0, -100.0),
             'selu': (-20.0, -50.0, -100.0), 'softplus': (21.0, 25.0, 30.0, 100.0, -30.0, -100.0),
             'swish': (41.0, 60.0, 100.0, -41.0, -60.0, -80.0, -100.0)}


def _dts(dt):
    return 'f32' if dt == F32 else 'f16'


def _kname(base, dt):
    return f'{base}<{"float" if dt == F32 else "__half"}>'


# ------------------------------------------------------------------------------------------------ the launch rules, mirrored
def bias_act_plan(numel, dtype, x_off, y_off, sms=SMS):
    """n3d_bias_act: nothing for numel 0; else grid_stride(ceil(numel / 4), sms, 8).  The vector loop takes numel // 4 items of 4
    elements when x and y (x_off / y_off elements past 64-byte aligned bases) are both 16-byte (fp32) or 8-byte (fp16) aligned; the
    scalar loop takes the rest (all of it when either is misaligned).  Each loop's grid-stride passes."""
    if numel == 0:
        return None
    vbytes = 4 * (4 if dtype == F32 else 2)
    esize = 4 if dtype == F32 else 2
    vec = (x_off * esize) % vbytes == 0 and (y_off * esize) % vbytes == 0
    grid = grid_stride(cdiv(numel, 4), sms, 8)
    nvec = numel // 4 if vec else 0
    nscalar = numel - 4 * nvec
    return dict(kernel=_kname('bias_act_kernel', dtype), grid=grid, vec=vec, nvec=nvec, nscalar=nscalar,
                vec_passes=cdiv(nvec, grid * 256), scalar_passes=cdiv(nscalar, grid * 256))


def upfirdn_out(H, W, fh, fw, up, down, pad):
    """Output size of one upfirdn2d launch: pad = (x0, x1, y0, y1), up / down = (x, y)."""
    return (H * up[1] + pad[2] + pad[3] - fh + down[1]) // down[1], (W * up[0] + pad[0] + pad[1] - fw + down[0]) // down[0]


def upfirdn2d_plan(N, C, H, W, f, up, down, pad, w_fastest, dtype, sms=SMS):
    """The n3d_upfirdn2d launches of one upfirdn2d: a 2-D filter ('2d', fh, fw) is one launch; a 1-D one ('1d', n) is a horizontal
    launch (1 x n, up / down / pad along x only) and then a vertical one (n x 1, along y only).  Each: the instance, the grid
    (grid_stride(N*C*outH*outW, sms, 16)), fh*fw*4 bytes of shared memory, the walk order (w_fastest: y_strides[3] == 1, given per
    launch) and the passes; plus the size of its output."""
    def one(h, w, fh, fw, u, d, p, wf):
        oh, ow = upfirdn_out(h, w, fh, fw, u, d, p)
        total = N * C * oh * ow
        grid = grid_stride(total, sms, 16)
        return dict(kernel=_kname('upfirdn2d_kernel', dtype), grid=grid, smem=fh * fw * 4, w_fastest=wf, passes=cdiv(total, grid * 256),
                    taps=(fh, fw), out=(oh, ow))
    if f[0] == '2d':
        return [one(H, W, f[1], f[2], up, down, pad, w_fastest[-1])]
    n = f[1]
    first = one(H, W, 1, n, (up[0], 1), (down[0], 1), (pad[0], pad[1], 0, 0), w_fastest[0])
    return [first, one(H, first['out'][1], n, 1, (1, up[1]), (1, down[1]), (0, 0, pad[2], pad[3]), w_fastest[-1])]


def _ftaps(f):
    """(fh, fw) of a filter spec as the filtered_lrelu wrapper passes it: None -> 1 x 1, a 1-D filter as its outer product."""
    if f is None:
        return 1, 1
    return (f[1], f[2]) if f[0] == '2d' else (f[1], f[1])


def filtered_lrelu_plan(N, C, H, W, fu, fd, up, down, pad, dtype, sms=SMS):
    """n3d_filtered_lrelu: flrelu_up_kernel over the N*C*upH*upW scratch, then flrelu_down_kernel over N*C*outH*outW, both
    grid_stride(., sms, 16)."""
    fuh, fuw = _ftaps(fu)
    fdh, fdw = _ftaps(fd)
    upH, upW = H * up + pad[2] + pad[3] - fuh + 1, W * up + pad[0] + pad[1] - fuw + 1
    outH, outW = (upH - fdh + down) // down, (upW - fdw + down) // down
    t1, t2 = N * C * upH * upW, N * C * outH * outW
    g1, g2 = grid_stride(t1, sms, 16), grid_stride(t2, sms, 16)
    return dict(up_kernel=_kname('flrelu_up_kernel', dtype), down_kernel=_kname('flrelu_down_kernel', dtype), up_grid=g1, down_grid=g2,
                up_passes=cdiv(t1, g1 * 256), down_passes=cdiv(t2, g2 * 256), upH=upH, upW=upW, outH=outH, outW=outW)


# ------------------------------------------------------------------------------------------------ the case table
def _ba(name, act, dtype, shape=(2, 6, 7, 8), cl=False, dim=1, xoff=0, yoff=0, gain=None, alpha=None, clamp=-1.0):
    """bias_act over a 4-D x stored NCHW or channels_last (cl), x and y starting xoff / yoff elements into aligned storage; dim None:
    no bias."""
    idx, dalpha, dgain = ACTS[act]
    return dict(op='bias_act', name=name, act=act, dtype=dtype, shape=shape, cl=cl, dim=dim, xoff=xoff, yoff=yoff,
                gain=dgain if gain is None else gain, alpha=dalpha if alpha is None else alpha, clamp=clamp)


_BA_SHAPES = [(2, 6, 7, 8), (1, 5, 7, 9), (2, 5, 3, 7), (1, 5, 3, 3)]       # numel % 4 == 0, 3, 2, 1
_BA_DIMS = [1, 0, 2, 3, None]
BIAS_ACT = [_ba(f'ba_{act}_{_dts(dt)}_{path}', act, dt, shape=_BA_SHAPES[(i + j) % 4], cl=(i + j) % 2 == 1,
                dim=_BA_DIMS[(i + 2 * j + (dt == F16)) % 5], xoff=j * (1 + i % 3), yoff=j * (1 + (i + 1) % 3),
                gain=0.7 if (i + j) % 3 == 0 else None, clamp=1.5 if (i + (dt == F16)) % 2 else -1.0)
            for i, act in enumerate(ACTS) for dt in (F32, F16) for j, path in enumerate(('vec', 'scalar'))] + [
    _ba('ba_lrelu_alpha_cl_dim3', 'lrelu', F32, cl=True, dim=3, alpha=0.05, gain=1.25),
    _ba('ba_lrelu_alpha_f16_dim2', 'lrelu', F16, dim=2, alpha=0.35, clamp=2.0),
    _ba('ba_swish_size_b1', 'swish', F32, shape=(3, 1, 6, 5), dim=1),
    _ba('ba_tanh_size_b1_cl_f16', 'tanh', F16, shape=(3, 1, 6, 5), cl=True, dim=1),
    _ba('ba_elu_cl_dim0', 'elu', F32, cl=True, dim=0),
    _ba('ba_selu_cl_dim2_f16', 'selu', F16, cl=True, dim=2),
    _ba('ba_sigmoid_x_misaligned', 'sigmoid', F32, xoff=2),
    _ba('ba_softplus_y_misaligned_f16', 'softplus', F16, yoff=3),
    _ba('ba_numel0', 'lrelu', F32, shape=(0, 6, 7, 8)),
    _ba('ba_grid_vec_swish', 'swish', F32, shape=(4, 33, 91, 97), dim=1),
    _ba('ba_grid_vec_tanh_f16_cl', 'tanh', F16, shape=(4, 33, 91, 97), cl=True, dim=1, clamp=0.9),
    _ba('ba_grid_scalar_lrelu', 'lrelu', F32, shape=(2, 17, 91, 97), cl=True, dim=3, xoff=1, yoff=1, clamp=1.5),
    _ba('ba_grid_scalar_sigmoid_f16', 'sigmoid', F16, shape=(2, 17, 91, 97), dim=2, xoff=1, yoff=3),
]


def _up(name, dtype, N, C, H, W, f, up=(1, 1), down=(1, 1), pad=(0, 0, 0, 0), flip=False, gain=1.0, xlay='nchw', ylay='nchw'):
    """upfirdn2d: f ('2d', fh, fw) or ('1d', n); up / down (x, y); pad (x0, x1, y0, y1).  xlay: nchw, cl, cslice (a channel slice),
    nslice (every other image), col2 (every other column), off1..off3 (starting 1-3 elements into the storage).  ylay: nchw, cl,
    cslice_cl (channels [2, C + 2) of a C + 4 channels_last buffer)."""
    return dict(op='upfirdn2d', name=name, dtype=dtype, N=N, C=C, H=H, W=W, f=f, up=tuple(up), down=tuple(down), pad=tuple(pad),
                flip=flip, gain=gain, xlay=xlay, ylay=ylay)


UPFIRDN = [
    _up('up_f4_nchw', F32, 2, 3, 9, 11, ('2d', 4, 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0),
    _up('up_f4_cl_f16', F16, 2, 5, 9, 11, ('2d', 4, 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_f1x1_cslice', F32, 2, 3, 7, 6, ('2d', 1, 1), xlay='cslice', gain=0.5),
    _up('up_f1x1_up4_cl_out', F16, 1, 4, 5, 6, ('2d', 1, 1), up=(4, 4), pad=(1, 2, 0, 3), xlay='nslice', ylay='cl'),
    _up('up_f35_up3x2_flip', F32, 2, 3, 8, 7, ('2d', 3, 5), up=(3, 2), pad=(2, 3, 1, 1), flip=True, gain=6.0, xlay='col2'),
    _up('up_f35_down3x2_f16_cslice_out', F16, 2, 6, 13, 17, ('2d', 3, 5), down=(3, 2), pad=(1, 2, 2, 0), xlay='cl', ylay='cslice_cl'),
    _up('up_f4_up4_down2', F32, 1, 3, 6, 5, ('2d', 4, 4), up=(4, 4), down=(2, 2), pad=(3, 2, 3, 2), gain=16.0, xlay='off1'),
    _up('up_f4_up2_down3x2_f16', F16, 2, 2, 11, 9, ('2d', 4, 4), up=(2, 2), down=(3, 2), pad=(1, 2, 2, 1), gain=4.0, xlay='off2'),
    _up('up_negpad_x0', F32, 2, 3, 9, 10, ('2d', 4, 4), pad=(-2, 1, 1, 1), xlay='off3', ylay='cl'),
    _up('up_negpad_x1_f16', F16, 2, 3, 9, 10, ('2d', 3, 5), pad=(1, -3, 1, 1), flip=True),
    _up('up_negpad_y0', F32, 1, 4, 9, 10, ('2d', 3, 5), pad=(2, 2, -2, 1), ylay='cslice_cl'),
    _up('up_negpad_y1_f16', F16, 1, 4, 9, 10, ('2d', 4, 4), up=(2, 2), pad=(1, 1, 2, -3), gain=4.0, xlay='cslice', ylay='cl'),
    _up('up_widepad_zero_rows', F32, 2, 3, 5, 6, ('2d', 3, 5), pad=(7, 6, 5, 4)),
    _up('up_widepad_zero_rows_f16_cl', F16, 2, 3, 5, 6, ('2d', 4, 4), up=(2, 2), pad=(6, 5, 7, 4), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_out_h1', F32, 2, 3, 4, 9, ('2d', 4, 4), down=(1, 2), pad=(1, 1, 0, 0)),
    _up('up_out_w1_f16', F16, 2, 3, 9, 4, ('2d', 3, 5), pad=(0, 1, 1, 1), ylay='cl'),
    _up('up_in_h1', F32, 3, 2, 1, 12, ('2d', 1, 1), up=(2, 2), pad=(0, 1, 0, 1)),
    _up('up_in_w1_cl', F16, 3, 2, 12, 1, ('2d', 4, 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_f32x32', F32, 1, 2, 40, 36, ('2d', 32, 32), pad=(16, 15, 16, 15), flip=True, gain=2.0),
    _up('up_f32x32_f16_cl', F16, 1, 3, 20, 24, ('2d', 32, 32), up=(2, 2), down=(2, 2), pad=(16, 15, 16, 15), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_1d1', F32, 2, 3, 7, 9, ('1d', 1), up=(2, 2), pad=(0, 1, 1, 0), gain=4.0),
    _up('up_1d4_f16_cl', F16, 2, 3, 7, 9, ('1d', 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_1d8_down2', F32, 2, 3, 16, 14, ('1d', 8), down=(2, 2), pad=(3, 3, 3, 3), flip=True, xlay='nslice'),
    _up('up_1d8_up3x2_f16', F16, 1, 4, 9, 8, ('1d', 8), up=(3, 2), pad=(4, 3, 4, 3), gain=6.0, xlay='col2'),
    _up('up_1d12_down3x2_cslice_out', F32, 2, 5, 20, 18, ('1d', 12), down=(3, 2), pad=(5, 5, 6, 4), gain=2.0, ylay='cslice_cl'),
    _up('up_1d12_negpad_f16', F16, 2, 3, 16, 15, ('1d', 12), up=(2, 2), pad=(-1, 3, 5, -2), gain=4.0, flip=True, xlay='off1'),
    _up('up_grid', F32, 2, 3, 200, 200, ('2d', 4, 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0),
    _up('up_grid_f16_cl', F16, 2, 3, 200, 200, ('2d', 4, 4), up=(2, 2), pad=(2, 1, 2, 1), gain=4.0, xlay='cl', ylay='cl'),
    _up('up_grid_1d8', F32, 1, 4, 200, 200, ('1d', 8), up=(2, 2), pad=(4, 3, 4, 3), gain=4.0),
]


def _fl(name, dtype, N, C, H, W, fu, fd, up, down, pad, flip=False, gain=SQRT2, slope=0.2, clamp=None, bias=True):
    """filtered_lrelu: fu / fd None, ('2d', fh, fw) or ('1d', n); pad (x0, x1, y0, y1)."""
    return dict(op='filtered_lrelu', name=name, dtype=dtype, N=N, C=C, H=H, W=W, fu=fu, fd=fd, up=up, down=down, pad=tuple(pad),
                flip=flip, gain=gain, slope=slope, clamp=clamp, bias=bias)


F44, F35, F1D4, F1D8 = ('2d', 4, 4), ('2d', 3, 5), ('1d', 4), ('1d', 8)
FLRELU = [
    _fl('fl_u1_d1', F32, 2, 3, 8, 9, F35, F44, 1, 1, (2, 1, 1, 2)),
    _fl('fl_u1_d2_f16', F16, 2, 3, 10, 9, F44, F44, 1, 2, (2, 1, 2, 1), clamp=0.6),
    _fl('fl_u1_d4', F32, 2, 3, 12, 14, None, F1D8, 1, 4, (3, 4, 4, 3), bias=False),
    _fl('fl_u2_d1_funone', F32, 2, 3, 8, 7, None, F44, 2, 1, (1, 2, 1, 2)),
    _fl('fl_u2_d2_funone_fdnone', F32, 2, 3, 8, 7, None, None, 2, 2, (0, 1, 0, 1), slope=0.0),     # samples the input pixels
    _fl('fl_u2_d4_f16', F16, 1, 4, 9, 10, F1D4, F1D8, 2, 4, (3, 2, 3, 2), flip=True, gain=1.3),
    _fl('fl_u4_d1_funone_f16', F16, 2, 3, 6, 5, None, F35, 4, 1, (1, 0, 2, 2), clamp=0.8),
    _fl('fl_u4_d2', F32, 1, 3, 6, 7, F1D8, F44, 4, 2, (5, 4, 5, 4), clamp=1.0, flip=True),
    _fl('fl_u4_d4_funone', F32, 2, 2, 5, 6, None, F1D4, 4, 4, (0, 3, 1, 2), slope=0.0, bias=False),
    _fl('fl_fd_none_down2_negpad', F32, 2, 3, 9, 8, F35, None, 2, 2, (-1, 2, 1, -2), gain=0.9),
    _fl('fl_1d_both_flip_f16', F16, 2, 3, 10, 11, F1D8, F1D8, 2, 2, (6, 5, 6, 5), flip=True, clamp=0.5, bias=False),
    _fl('fl_nonsquare_both', F32, 1, 4, 9, 9, F35, F35, 2, 1, (2, 2, 1, 3)),
    _fl('fl_1d4_fu_fd_none_negpad_f16', F16, 2, 2, 9, 8, F1D4, None, 1, 1, (-1, 0, 0, -1), slope=0.0, gain=2.0),
    _fl('fl_grid', F32, 1, 4, 200, 200, F44, None, 2, 1, (2, 1, 2, 1)),
    _fl('fl_grid_f16', F16, 1, 2, 300, 300, None, None, 2, 1, (0, 0, 0, 0), clamp=1.0),
]

CASES = BIAS_ACT + UPFIRDN + FLRELU
CASE_IDS = [c['name'] for c in CASES]


def _wf(lay):
    return lay == 'nchw'


def launches(c, sms=SMS):
    """[(kernel, grid)] of a case in launch order."""
    if c['op'] == 'bias_act':
        p = bias_act_plan(math.prod(c['shape']), c['dtype'], c['xoff'], c['yoff'], sms)
        return [] if p is None else [(p['kernel'], p['grid'])]
    if c['op'] == 'upfirdn2d':
        return [(p['kernel'], p['grid']) for p in case_plan(c, sms)]
    p = case_plan(c, sms)
    return [(p['up_kernel'], p['up_grid']), (p['down_kernel'], p['down_grid'])]


def _w_fastest(c):
    """y_strides[3] == 1 of each launch: NCHW outputs (and the intermediate of an NCHW output) walk ox fastest; channels_last ones
    walk c fastest unless C is 1."""
    wf = _wf(c['ylay']) or c['C'] == 1
    return (wf, wf) if c['f'][0] == '1d' else (wf,)


def case_plan(c, sms=SMS):
    if c['op'] == 'bias_act':
        return bias_act_plan(math.prod(c['shape']), c['dtype'], c['xoff'], c['yoff'], sms)
    if c['op'] == 'upfirdn2d':
        return upfirdn2d_plan(c['N'], c['C'], c['H'], c['W'], c['f'], c['up'], c['down'], c['pad'], _w_fastest(c), c['dtype'], sms)
    return filtered_lrelu_plan(c['N'], c['C'], c['H'], c['W'], c['fu'], c['fd'], c['up'], c['down'], c['pad'], c['dtype'], sms)


def _of(op, cs):
    return [(c, p) for c, p in cs if c['op'] == op]


def _fkind(f):
    if f is None:
        return 'none'
    if f[0] == '1d':
        return '1d<8' if f[1] < 8 else '1d>=8'
    return '2d' if f[1] == f[2] else '2d-nonsquare'


def _zero_rows(c):
    """Padding wider than the filter on a leading side: whole output rows / columns read only zeros."""
    fh, fw = (c['f'][1], c['f'][2]) if c['f'][0] == '2d' else (c['f'][1], c['f'][1])
    return c['pad'][2] >= fh or c['pad'][0] >= fw


COVERAGE = {
    # bias_act
    'bias_act: every activation x fp32 / fp16 x vector / scalar loop':
        lambda cs: {(c['act'], c['dtype'], p['vec']) for c, p in _of('bias_act', cs) if p} == {(a, d, v) for a in ACTS for d in (F32, F16) for v in (False, True)},
    'bias_act: numel % 4 of 0, 1, 2, 3 on the vector loop': lambda cs: {math.prod(c['shape']) % 4 for c, p in _of('bias_act', cs) if p and p['vec']} == {0, 1, 2, 3},
    'bias_act: numel % 4 of 0, 1, 2, 3 on the scalar loop': lambda cs: {math.prod(c['shape']) % 4 for c, p in _of('bias_act', cs) if p and not p['vec']} == {0, 1, 2, 3},
    'bias_act: no bias, and a bias along dims 0-3 in NCHW and channels_last':
        lambda cs: {(c['dim'], c['cl']) for c, p in _of('bias_act', cs)} >= {(None, False), (None, True)} | {(d, cl) for d in range(4) for cl in (False, True)},
    'bias_act: step_b 1 and > 1': lambda cs: {_step_b(c) == 1 for c, p in _of('bias_act', cs) if c['dim'] is not None} == {False, True},
    'bias_act: size_b 1': lambda cs: any(c['dim'] is not None and c['shape'][c['dim']] == 1 for c, p in _of('bias_act', cs)),
    'bias_act: gain other than the default': lambda cs: any(c['gain'] != ACTS[c['act']][2] for c, p in _of('bias_act', cs)),
    'bias_act: lrelu alpha other than 0.2': lambda cs: any(c['act'] == 'lrelu' and c['alpha'] != 0.2 for c, p in _of('bias_act', cs)),
    'bias_act: clamp off and on, each in fp32 and fp16': lambda cs: {(c['clamp'] >= 0, c['dtype']) for c, p in _of('bias_act', cs)} == {(a, d) for a in (False, True) for d in (F32, F16)},
    'bias_act: saturated inputs with clamp off for tanh, sigmoid, elu, selu, softplus, swish':
        lambda cs: {c['act'] for c, p in _of('bias_act', cs) if c['clamp'] < 0 and p} >= set(SATURATED),
    'bias_act: x misaligned alone, y misaligned alone, both':
        lambda cs: {(c['xoff'] % 4 != 0, c['yoff'] % 4 != 0) for c, p in _of('bias_act', cs)} >= {(True, False), (False, True), (True, True)},
    'bias_act: > 1 pass of the vector loop in fp32 and fp16': lambda cs: {c['dtype'] for c, p in _of('bias_act', cs) if p and p['vec_passes'] > 1} == {F32, F16},
    'bias_act: > 1 pass of the scalar loop in fp32 and fp16': lambda cs: {c['dtype'] for c, p in _of('bias_act', cs) if p and p['scalar_passes'] > 1} == {F32, F16},
    'bias_act: numel 0': lambda cs: any(p is None for c, p in _of('bias_act', cs)),
    # upfirdn2d
    'upfirdn2d: fp32 / fp16 x w_fastest 0 / 1':
        lambda cs: {(c['dtype'], q['w_fastest']) for c, p in _of('upfirdn2d', cs) for q in p} == {(d, w) for d in (F32, F16) for w in (False, True)},
    'upfirdn2d: filters 1x1, 4x4, 3x5, 32x32; 1-D 1, 4, 8, 12':
        lambda cs: {c['f'] for c, p in _of('upfirdn2d', cs)} >= {('2d', 1, 1), F44, F35, ('2d', 32, 32), ('1d', 1), F1D4, F1D8, ('1d', 12)},
    'upfirdn2d: 1024 taps is the largest launch': lambda cs: max(q['smem'] for c, p in _of('upfirdn2d', cs) for q in p) == 4096,
    'upfirdn2d: flip 0 / 1 and a gain other than 1': lambda cs: {c['flip'] for c, p in _of('upfirdn2d', cs)} == {False, True} and any(c['gain'] != 1 for c, p in _of('upfirdn2d', cs)),
    'upfirdn2d: up (1, 1), (2, 2), (4, 4), (3, 2)': lambda cs: {c['up'] for c, p in _of('upfirdn2d', cs)} >= {(1, 1), (2, 2), (4, 4), (3, 2)},
    'upfirdn2d: down (2, 2) and (3, 2)': lambda cs: {c['down'] for c, p in _of('upfirdn2d', cs)} >= {(2, 2), (3, 2)},
    'upfirdn2d: up and down together': lambda cs: any(c['up'] != (1, 1) and c['down'] != (1, 1) for c, p in _of('upfirdn2d', cs)),
    'upfirdn2d: negative padding on each side alone':
        lambda cs: all(any(c['pad'][k] < 0 and all(c['pad'][j] >= 0 for j in range(4) if j != k) for c, p in _of('upfirdn2d', cs)) for k in range(4)),
    'upfirdn2d: padding wider than the filter (whole zero rows)': lambda cs: any(_zero_rows(c) for c, p in _of('upfirdn2d', cs)),
    'upfirdn2d: outH 1 and outW 1': lambda cs: {(q['out'][0] == 1, q['out'][1] == 1) for c, p in _of('upfirdn2d', cs) for q in p[-1:]} >= {(True, False), (False, True)},
    'upfirdn2d: H 1 and W 1': lambda cs: any(c['H'] == 1 for c, p in _of('upfirdn2d', cs)) and any(c['W'] == 1 for c, p in _of('upfirdn2d', cs)),
    'upfirdn2d: every input layout': lambda cs: {c['xlay'] for c, p in _of('upfirdn2d', cs)} == {'nchw', 'cl', 'cslice', 'nslice', 'col2', 'off1', 'off2', 'off3'},
    'upfirdn2d: an output in a channel slice of a wider channels_last buffer, 2-D and 1-D filters':
        lambda cs: {c['f'][0] for c, p in _of('upfirdn2d', cs) if c['ylay'] == 'cslice_cl'} == {'2d', '1d'},
    'upfirdn2d: > 1 pass, 2-D filter in fp32 and fp16 and the separable route':
        lambda cs: {(c['dtype'], c['f'][0]) for c, p in _of('upfirdn2d', cs) if any(q['passes'] > 1 for q in p)} >= {(F32, '2d'), (F16, '2d'), (F32, '1d')},
    # filtered_lrelu
    'filtered_lrelu: up 1, 2, 4 x down 1, 2, 4': lambda cs: {(c['up'], c['down']) for c, p in _of('filtered_lrelu', cs)} == {(u, d) for u in (1, 2, 4) for d in (1, 2, 4)},
    'filtered_lrelu: fu None, 2-D, non-square 2-D, 1-D < 8 and >= 8 taps':
        lambda cs: {_fkind(c['fu']) for c, p in _of('filtered_lrelu', cs)} == {'none', '2d', '2d-nonsquare', '1d<8', '1d>=8'},
    'filtered_lrelu: fd None, 2-D, non-square 2-D, 1-D < 8 and >= 8 taps':
        lambda cs: {_fkind(c['fd']) for c, p in _of('filtered_lrelu', cs)} == {'none', '2d', '2d-nonsquare', '1d<8', '1d>=8'},
    'filtered_lrelu: fu None at up 2 and 4': lambda cs: {c['up'] for c, p in _of('filtered_lrelu', cs) if c['fu'] is None} >= {2, 4},
    'filtered_lrelu: asymmetric and negative padding':
        lambda cs: any(c['pad'][0] != c['pad'][1] for c, p in _of('filtered_lrelu', cs)) and any(min(c['pad']) < 0 for c, p in _of('filtered_lrelu', cs)),
    'filtered_lrelu: flip_filter, slope 0 and 0.2, gain other than sqrt 2':
        lambda cs: any(c['flip'] for c, p in _of('filtered_lrelu', cs)) and {c['slope'] for c, p in _of('filtered_lrelu', cs)} == {0.0, 0.2}
        and any(c['gain'] != SQRT2 for c, p in _of('filtered_lrelu', cs)),
    'filtered_lrelu: clamp None and active, bias None and present':
        lambda cs: {c['clamp'] is None for c, p in _of('filtered_lrelu', cs)} == {False, True} and {c['bias'] for c, p in _of('filtered_lrelu', cs)} == {False, True},
    'filtered_lrelu: fp16': lambda cs: any(c['dtype'] == F16 for c, p in _of('filtered_lrelu', cs)),
    'filtered_lrelu: > 1 pass in each launch, fp32 and fp16':
        lambda cs: {c['dtype'] for c, p in _of('filtered_lrelu', cs) if p['up_passes'] > 1 and p['down_passes'] > 1} == {F32, F16},
}


def _step_b(c):
    """x.stride(dim) of a bias_act case's x (the wrapper's step_b)."""
    N, C, H, W = c['shape']
    strides = (H * W * C, 1, W * C, C) if c['cl'] else (C * H * W, H * W, W, 1)
    return max(strides[c['dim']], 1)


def case_bytes(c):
    """Device memory of a case: inputs, guarded outputs and about six fp64 copies of the largest image (reference, R, their inputs)."""
    if c['op'] == 'bias_act':
        n = math.prod(c['shape'])
        return n * (2 * 4 + 6 * 8)
    if c['op'] == 'upfirdn2d':
        p = case_plan(c)
        big = max([c['N'] * c['C'] * c['H'] * c['W'] * 2] + [c['N'] * (c['C'] + 4) * q['out'][0] * q['out'][1] for q in p])
        big *= max(c['up'][0] * c['up'][1], 1)                       # the zero-inserted image of the reference
        return big * (2 * 4 + 6 * 8)
    p = case_plan(c)
    big = max(c['N'] * c['C'] * c['H'] * c['W'] * c['up'] ** 2, c['N'] * c['C'] * p['upH'] * p['upW'])
    return big * (4 + 4 + 6 * 8)


def test_case_table_covers_every_launch_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rules, at <= 512 MB per case."""
    planned = [(c, case_plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(CASE_IDS + WRAP_IDS)) == len(CASE_IDS) + len(WRAP_IDS)
    big = {c['name']: case_bytes(c) / 2 ** 20 for c in CASES if case_bytes(c) > 512 * 2 ** 20}
    assert not big, big


def test_mirror_examples():
    """CPU: the mirrors on hand-computed launches."""
    p = bias_act_plan(4 * 270336 + 5, F32, 0, 0)          # ceil(numel / 4) > 132 * 8 * 256: the grid is capped, two vector passes
    assert (p['grid'], p['vec'], p['nvec'], p['nscalar'], p['vec_passes'], p['scalar_passes']) == (1056, True, 270337, 1, 2, 1)
    p = bias_act_plan(13, F16, 0, 2)                          # y 4 bytes into its storage: not 8-byte aligned
    assert (p['grid'], p['vec'], p['nscalar']) == (1, False, 13)
    assert bias_act_plan(13, F16, 4, 4)['vec'] and not bias_act_plan(13, F32, 2, 2)['vec']
    h, v = upfirdn2d_plan(1, 3, 10, 12, ('1d', 8), (2, 1), (1, 2), (3, 4, 2, 5), (True, False), F32)
    assert h['out'] == (10, (24 + 7 - 8 + 1)) and v['out'] == ((10 + 7 - 8 + 2) // 2, 24) and (h['taps'], v['taps']) == ((1, 8), (8, 1))
    p = filtered_lrelu_plan(1, 2, 8, 8, None, F44, 2, 2, (1, 2, 1, 2), F32)
    assert (p['upH'], p['upW'], p['outH'], p['outW']) == (19, 19, 8, 8)


# ------------------------------------------------------------------------------------------------ errors
def ulp(v, dtype):
    """The spacing of `dtype` at |v| (fp64), at least its spacing at the smallest normal number."""
    fi = torch.finfo(dtype)
    _, e = torch.frexp(v.abs().clamp_min(fi.tiny))
    return fi.eps * torch.exp2((e - 1).to(F64))            # |v| in [2^(e-1), 2^e)


def ulp_err(got, ref, dtype):
    """max over elements of |got - ref| / ulp(ref), ref the fp64 value (rounded to fp16 first for fp16 outputs); where |ref| lies below
    the smallest normal fp32 number, an absolute error up to that number is not counted.  NaN counts as infinite."""
    want = ref.to(F16).double() if dtype == F16 else ref
    d = (got.double() - want).abs()
    d = torch.where(ref.abs() < TINY32, (d - TINY32).clamp_min(0), d)
    e = d / ulp(ref, dtype)
    e = torch.nan_to_num(e, nan=math.inf)
    return e.max().item() if e.numel() else 0.0


def fir_err(got, ref, R, dtype):
    """max over elements of |got - ref| / R (ref rounded to fp16 first for fp16 outputs); an element with R == 0 must be exactly 0."""
    want = ref.to(F16).double() if dtype == F16 else ref
    d = torch.nan_to_num((got.double() - want).abs(), nan=math.inf)
    e = torch.where(R > 0, d / R.clamp_min(1e-300), torch.where(d == 0, torch.zeros_like(d), torch.full_like(d, math.inf)))
    return e.max().item() if e.numel() else 0.0


# ------------------------------------------------------------------------------------------------ inputs, outputs, launches
def _gen(c, table):
    return torch.Generator(device=DEV).manual_seed(3000 + [t['name'] for t in table].index(c['name']) + (0 if table is CASES else 500))


def make_input(shape, dtype, lay, g, scale=1.0):
    """A 4-D input of logical shape `shape` in one of the layouts of the table (see _up)."""
    N, C, H, W = shape
    rnd = lambda *s: (torch.randn(*s, device=DEV, generator=g) * scale).to(dtype)      # noqa: E731
    if lay == 'nchw':
        return rnd(N, C, H, W)
    if lay == 'cl':
        return rnd(N, C, H, W).contiguous(memory_format=CL)
    if lay == 'cslice':
        return rnd(N, C + 3, H, W)[:, 1:C + 1]
    if lay == 'cslice_cl':
        return rnd(N, C + 4, H, W).contiguous(memory_format=CL)[:, 2:C + 2]
    if lay == 'nslice':
        return rnd(2 * N, C, H, W)[::2]
    if lay == 'col2':
        return rnd(N, C, H, 2 * W)[..., ::2]
    k = int(lay[3:])
    n = N * C * H * W
    return offset_view(rnd(n + 64), k * torch.tensor([], dtype=dtype).element_size())[:n].view(N, C, H, W)


def make_output(shape, dtype, lay):
    """(Guarded, the logical NCHW view the launch writes) for an output layout: nchw, cl, cslice_cl."""
    N, C, H, W = shape
    if lay == 'nchw':
        t = Guarded((N, C, H, W), dtype)
        return t, t.view
    if lay == 'cl':
        t = Guarded((N, H, W, C), dtype)
        return t, t.view.permute(0, 3, 1, 2)
    t = Guarded((N, H, W, C + 4), dtype, own=slice(2, C + 2))
    return t, t.view[..., 2:C + 2].permute(0, 3, 1, 2)


def _filter(spec, g):
    """A filter of mixed sign for a spec: ('2d', fh, fw) or ('1d', n); None stays None."""
    if spec is None:
        return None
    shape = (spec[1], spec[2]) if spec[0] == '2d' else (spec[1],)
    f = torch.randn(*shape, device=DEV, generator=g) + 0.5
    return f / f.sum().abs()


def setup_case(c):
    g = _gen(c, CASES)
    s = dict(c=c)
    if c['op'] == 'bias_act':
        dt, shape = c['dtype'], c['shape']
        N, C, H, W = shape
        n = math.prod(shape)
        store = offset_view((torch.randn(n + 64, device=DEV, generator=g) * 2).to(dt), c['xoff'] * (4 if dt == F32 else 2))[:n]
        sat = SATURATED.get(c['act'], ())
        for i, v in enumerate(sat[:n]):
            store[(3 + 11 * i) % n] = v
        s['x'] = store.view(N, H, W, C).permute(0, 3, 1, 2) if c['cl'] else store.view(shape)
        s['b'] = (torch.randn(shape[c['dim']], device=DEV, generator=g) * 0.5).to(dt) if c['dim'] is not None else None
        s['y'] = Guarded((n + c['yoff'],), dt, own=slice(c['yoff'], None))
        return s
    if c['op'] == 'upfirdn2d':
        N, C, H, W = c['N'], c['C'], c['H'], c['W']
        s['x'] = make_input((N, C, H, W), c['dtype'], c['xlay'], g)
        s['f'] = _filter(c['f'], g)
        p = case_plan(c)
        s['outs'] = []
        mid_lay = 'nchw' if c['ylay'] == 'nchw' else 'cl'
        for i, q in enumerate(p):
            lay = c['ylay'] if i == len(p) - 1 else mid_lay
            s['outs'].append(make_output((N, C) + q['out'], c['dtype'], lay))
        return s
    N, C, H, W = c['N'], c['C'], c['H'], c['W']
    p = case_plan(c)
    s['x'] = make_input((N, C, H, W), c['dtype'], 'nchw', g)
    s['fu'], s['fd'] = _filter(c['fu'], g), _filter(c['fd'], g)
    s['b'] = (torch.randn(C, device=DEV, generator=g) * 0.5).to(c['dtype']) if c['bias'] else None
    s['y'] = Guarded((N, C, p['outH'], p['outW']), c['dtype'])
    s['tmp'] = Guarded((N * C * p['upH'] * p['upW'],), F32)
    return s


def upfirdn2d_call(x, f2d, y, up, down, pad, flip, gain):
    """One n3d_upfirdn2d launch of x into the (possibly strided) view y, as torch_utils.ops.upfirdn2d._launch makes it."""
    L = lib()
    N, C, H, W = x.shape
    fh, fw = f2d.shape
    oh, ow = y.shape[2:]
    xs, ys = (L.I64 * 4)(*x.stride()), (L.I64 * 4)(*y.stride())
    return L.lib.n3d_upfirdn2d(x.data_ptr(), f2d.data_ptr(), y.data_ptr(), DTYPE_ID.get(x.dtype, 2), N, C, H, W, xs, ys, fh, fw, up[0], up[1],
                               down[0], down[1], pad[0], pad[1], pad[2], pad[3], int(flip), float(gain), oh, ow, L.stream_ptr())


def _as_2d(f):
    return None if f is None else (torch.outer(f, f) if f.ndim == 1 else f).contiguous()


def launch_case(s):
    L = lib()
    c = s['c']
    if c['op'] == 'bias_act':
        b = s['b']
        size_b, step_b = (b.shape[0], max(int(s['x'].stride(c['dim'])), 1)) if b is not None else (0, 0)
        L.check(L.lib.n3d_bias_act(s['x'].data_ptr(), L.ptr(b), s['y'].view[c['yoff']:].data_ptr(), DTYPE_ID[c['dtype']], math.prod(c['shape']),
                                   size_b, step_b, ACTS[c['act']][0], c['alpha'], c['gain'], c['clamp'], L.stream_ptr()), 'n3d_bias_act')
    elif c['op'] == 'upfirdn2d':
        f, up, down, pad = s['f'], c['up'], c['down'], c['pad']
        if c['f'][0] == '2d':
            L.check(upfirdn2d_call(s['x'], f, s['outs'][0][1], up, down, pad, c['flip'], c['gain']), 'n3d_upfirdn2d')
        else:                                   # the separable route of torch_utils.ops.upfirdn2d._forward
            gs = math.sqrt(c['gain'])
            mid = s['outs'][0][1]
            L.check(upfirdn2d_call(s['x'], f[None, :].contiguous(), mid, (up[0], 1), (down[0], 1), (pad[0], pad[1], 0, 0), c['flip'], gs), 'n3d_upfirdn2d')
            L.check(upfirdn2d_call(mid, f[:, None].contiguous(), s['outs'][1][1], (1, up[1]), (1, down[1]), (0, 0, pad[2], pad[3]), c['flip'], gs),
                    'n3d_upfirdn2d')
    else:
        p = case_plan(c)
        fu2, fd2 = _as_2d(s['fu']), _as_2d(s['fd'])
        fuh, fuw = _ftaps(c['fu'])
        fdh, fdw = _ftaps(c['fd'])
        px0, px1, py0, py1 = c['pad']
        L.check(L.lib.n3d_filtered_lrelu(s['x'].data_ptr(), L.ptr(fu2), L.ptr(fd2), L.ptr(s['b']), s['y'].view.data_ptr(), s['tmp'].view.data_ptr(),
                                         DTYPE_ID[c['dtype']], c['N'], c['C'], c['H'], c['W'], fuh, fuw, fdh, fdw, c['up'], c['down'],
                                         px0, px1, py0, py1, float(c['gain']), float(c['slope']), float(c['clamp'] if c['clamp'] is not None else -1.0),
                                         int(c['flip']), p['outH'], p['outW'], L.stream_ptr()), 'n3d_filtered_lrelu')
        s['keep'] = (fu2, fd2)                  # the filters must outlive the launch


def outputs(s):
    op = s['c']['op']
    if op == 'bias_act':
        return [s['y']]
    if op == 'upfirdn2d':
        return [t for t, _ in s['outs']]
    return [s['y'], s['tmp']]


# ------------------------------------------------------------------------------------------------ the fp64 references
def bias_act_reference(x, b, dim, act, alpha, gain, clamp):
    """oracle.ops.bias_act in fp64 of the fp32 sum x + b (b already in x's dtype)."""
    from oracle import ops as oo
    pre = x.float()
    if b is not None:
        pre = pre + b.float().reshape([-1 if i == dim else 1 for i in range(x.ndim)])
    return oo.bias_act(pre.double(), None, act=act, alpha=alpha, gain=gain, clamp=clamp if clamp >= 0 else None)


def fir_reference(x, f, up, down, pad, flip, gain, dtype):
    """(ref, R) of upfirdn2d in fp64: the oracle on the stored x and f, and on |x| with |f|.  For fp16 on the separable route the
    intermediate image is rounded to fp16, as the two launches store it."""
    from oracle import ops as oo
    x64, f64 = x.double(), f.double()
    R = oo.upfirdn2d(x64.abs(), f64.abs(), up=list(up), down=list(down), padding=list(pad), flip_filter=flip, gain=abs(gain))
    if f.ndim == 1 and dtype == F16:
        gs = math.sqrt(gain)
        mid = oo.upfirdn2d(x64, f64[None, :], up=[up[0], 1], down=[down[0], 1], padding=[pad[0], pad[1], 0, 0], flip_filter=flip, gain=gs)
        ref = oo.upfirdn2d(mid.to(F16).double(), f64[:, None], up=[1, up[1]], down=[1, down[1]], padding=[0, 0, pad[2], pad[3]],
                           flip_filter=flip, gain=gs)
    else:
        ref = oo.upfirdn2d(x64, f64, up=list(up), down=list(down), padding=list(pad), flip_filter=flip, gain=gain)
    return ref, R


def flrelu_reference(x, fu, fd, b, up, down, pad, gain, slope, clamp, flip):
    """(ref, R) of filtered_lrelu in fp64: the oracle on the stored values, and on |x|, |fu|, |fd|, |b| without the clamp."""
    from oracle import ops as oo
    d = lambda t: None if t is None else t.double()             # noqa: E731
    a = lambda t: None if t is None else t.double().abs()       # noqa: E731
    ref = oo.filtered_lrelu(d(x), d(fu), d(fd), d(b), up=up, down=down, padding=list(pad), gain=gain, slope=slope, clamp=clamp, flip_filter=flip)
    R = oo.filtered_lrelu(a(x), a(fu), a(fd), a(b), up=up, down=down, padding=list(pad), gain=gain, slope=slope, clamp=None, flip_filter=flip)
    return ref, R


def check_case(s):
    """-> {bound kind: error}; asserts the sentinel and written-element checks first."""
    c = s['c']
    for t in outputs(s):
        assert t.untouched_ok(), f'{c["name"]}: an element outside the output was written'
        assert t.written(), f'{c["name"]}: an owned element was not written'
    if c['op'] == 'bias_act':
        if math.prod(c['shape']) == 0:
            return {}
        ref = bias_act_reference(s['x'], s['b'], c['dim'], c['act'], c['alpha'], c['gain'], c['clamp'])
        ref = (ref.permute(0, 2, 3, 1) if c['cl'] else ref).reshape(-1)       # storage order
        return {f'ba.{_dts(c["dtype"])}.{c["act"]}': ulp_err(s['y'].view[c['yoff']:], ref, c['dtype'])}
    if c['op'] == 'upfirdn2d':
        ref, R = fir_reference(s['x'], s['f'], c['up'], c['down'], c['pad'], c['flip'], c['gain'], c['dtype'])
        return {f'fir.{_dts(c["dtype"])}': fir_err(s['outs'][-1][1], ref, R, c['dtype'])}
    ref, R = flrelu_reference(s['x'], s['fu'], s['fd'], s['b'], c['up'], c['down'], c['pad'], c['gain'], c['slope'], c['clamp'], c['flip'])
    return {f'flrelu.{_dts(c["dtype"])}': fir_err(s['y'].view, ref, R, c['dtype'])}


def _assert_bounds(name, errs):
    record_errors('N3D_OPS_ERRORS', [{'case': name, 'kind': k, 'err': e, 'bound': BOUNDS[k]} for k, e in errs.items()])
    bad = {k: (e, BOUNDS[k]) for k, e in errs.items() if not e <= BOUNDS[k]}
    assert not bad, (name, bad)


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_kernel_matches_fp64_reference(c):
    s = setup_case(c)
    launch_case(s)
    torch.cuda.synchronize()
    _assert_bounds(c['name'], check_case(s))
    assert rerun_identical(outputs(s), lambda: launch_case(s)), f'{c["name"]}: a rerun is not bit-identical'


@pytest.mark.gpu
def test_launched_kernels_match_plan(tmp_path):
    """Every case under torch.profiler: the kernel instances it launched and their grids are the ones the mirror predicts at the
    device's SM count; numel 0 launches nothing."""
    pattern = re.compile(r'bias_act_kernel<(?:float|__half)>|upfirdn2d_kernel<(?:float|__half)>|flrelu_up_kernel<(?:float|__half)>|'
                         r'flrelu_down_kernel<(?:float|__half)>')
    sms = torch.cuda.get_device_properties(0).multi_processor_count

    def run():
        expected = []
        for c in CASES:
            s = setup_case(c)
            torch.cuda.synchronize()
            launch_case(s)
            torch.cuda.synchronize()
            expected += [(c['name'], k, g) for k, g in launches(c, sms)]
            del s
        return expected

    expected, events = launched_kernels(run, pattern, tmp_path)
    for (who, kernel, grid), e in zip(expected, events):
        assert pattern.search(e['name']).group(0) == kernel, (who, e['name'], kernel)
        got = e.get('args', {}).get('grid')
        if got is not None:
            assert list(got) == [grid, 1, 1], (who, kernel, got, grid)


# ------------------------------------------------------------------------------------------------ torch_utils.ops
def _w(name, op, dtype, lay, shape=(2, 5, 12, 10), **kw):
    return dict(op=op, name=name, dtype=dtype, lay=lay, shape=shape, **kw)


WRAP = [
    _w('w_bias_act_nchw', 'bias_act', F32, 'nchw', act='lrelu', dim=1),
    _w('w_bias_act_cl_f16', 'bias_act', F16, 'cl', act='swish', dim=1, clamp=2.0),
    _w('w_bias_act_cslice_cl', 'bias_act', F32, 'cslice_cl', act='tanh', dim=1),
    _w('w_bias_act_nslice_dim2_f16', 'bias_act', F16, 'nslice', act='softplus', dim=2),
    _w('w_upfirdn2d_cl_1d8_f16', 'upfirdn2d', F16, 'cl', f=F1D8, up=2, down=1, pad=[4, 3, 4, 3], gain=4.0),
    _w('w_upfirdn2d_cslice_cl', 'upfirdn2d', F32, 'cslice_cl', f=F44, up=[3, 2], down=[1, 2], pad=[2, 1, 1, 2], gain=6.0),
    _w('w_upfirdn2d_col2_flip', 'upfirdn2d', F32, 'col2', f=F35, up=1, down=2, pad=[1, 1, 1, 1], flip=True),
    _w('w_upfirdn2d_cslice_cl_1d12', 'upfirdn2d', F32, 'cslice_cl', f=('1d', 12), up=1, down=[2, 1], pad=[5, 6, 5, 6]),
    _w('w_filter2d_cl', 'filter2d', F32, 'cl', f=F35, pad=1),
    _w('w_filter2d_nchw_f16', 'filter2d', F16, 'nchw', f=F44, pad=0),
    _w('w_upsample2d_cslice_cl_f16', 'upsample2d', F16, 'cslice_cl', f=F44),
    _w('w_upsample2d_nchw_1d8', 'upsample2d', F32, 'nchw', f=F1D8),
    _w('w_downsample2d_cl', 'downsample2d', F32, 'cl', f=F44),
    _w('w_downsample2d_nslice_1d12_f16', 'downsample2d', F16, 'nslice', f=('1d', 12)),
    _w('w_filtered_lrelu_cl', 'filtered_lrelu', F32, 'cl', fu=None, fd=F44, up=2, down=2, pad=[1, 2, 1, 2]),
    _w('w_filtered_lrelu_cslice_cl_f16', 'filtered_lrelu', F16, 'cslice_cl', fu=F1D8, fd=F1D4, up=2, down=1, pad=[5, 4, 5, 4], clamp=0.7),
    _w('w_filtered_lrelu_nchw_1d', 'filtered_lrelu', F32, 'nchw', fu=F1D4, fd=None, up=4, down=2, pad=[2, 1, 2, 1], flip=True),
]
WRAP_IDS = [c['name'] for c in WRAP]


def suggested_format(x):
    """x.suggest_memory_format() of the C++ API, as PyTorch restates it in Python for its own decompositions."""
    from torch._prims_common import suggest_memory_format
    return suggest_memory_format(x)


def _wrapper_fir_args(c):
    """(up, down, pad, gain) of the upfirdn2d a wrapper op makes, restated from torch_utils/ops/upfirdn2d.py:279-389."""
    f = c['f']
    fw = fh = f[1] if f[0] == '1d' else None
    if f[0] == '2d':
        fh, fw = f[1], f[2]
    if c['op'] == 'upfirdn2d':
        up = (c['up'], c['up']) if isinstance(c['up'], int) else tuple(c['up'])
        down = (c['down'], c['down']) if isinstance(c['down'], int) else tuple(c['down'])
        return up, down, tuple(c['pad']), c.get('gain', 1.0)
    if c['op'] == 'filter2d':
        p = c['pad']
        return (1, 1), (1, 1), (p + fw // 2, p + (fw - 1) // 2, p + fh // 2, p + (fh - 1) // 2), 1.0
    if c['op'] == 'upsample2d':
        return (2, 2), (1, 1), ((fw + 1) // 2, (fw - 2) // 2, (fh + 1) // 2, (fh - 2) // 2), 4.0
    return (1, 1), (2, 2), ((fw - 1) // 2, (fw - 2) // 2, (fh - 1) // 2, (fh - 2) // 2), 1.0


def test_suggest_memory_format_matches_torch():
    """CPU: the ops' restatement of suggest_memory_format against PyTorch's own on non-dense views: channel, batch, row and column
    slices of NCHW and channels_last tensors, size-1 dims among them, and transposed views."""
    from next3d_b200.torch_utils.ops._layout import suggest_memory_format
    views = []
    for shape in [(2, 5, 6, 7), (1, 5, 6, 7), (2, 1, 6, 7), (2, 5, 1, 7), (2, 5, 6, 1), (3, 1, 1, 1), (1, 4, 1, 1), (1, 1, 6, 7)]:
        for fmt in (torch.contiguous_format, CL):
            N, C, H, W = shape
            t = torch.empty(2 * N, C + 2, 2 * H, 2 * W).contiguous(memory_format=fmt)
            views += [t[::2, 1:C + 1, :H, :W], t[:N, :C, ::2, :W], t[:N, :C, :H, ::2], t[:N, 2:, :H, 1:W + 1]]
    views += [torch.empty(2, 5, 6, 7).transpose(2, 3)[..., :5], torch.empty(2, 5, 6, 7).transpose(1, 3)[:, :6]]
    views = [v for v in views if not (v.is_contiguous() or v.is_contiguous(memory_format=CL))]
    assert len(views) > 50
    for v in views:
        assert suggest_memory_format(v) == suggested_format(v), (tuple(v.shape), v.stride())
    assert {suggest_memory_format(v) for v in views} == {torch.contiguous_format, CL}


@pytest.mark.gpu
@pytest.mark.parametrize('c', WRAP, ids=WRAP_IDS)
def test_torch_utils_ops_values_and_layout(c):
    """torch_utils.ops on NCHW, channels_last and non-dense inputs: the values against the fp64 references, and an output in
    x.suggest_memory_format()."""
    from next3d_b200.torch_utils import ops
    g = _gen(c, WRAP)
    dt = c['dtype']
    x = make_input(c['shape'], dt, c['lay'], g, scale=2.0 if c['op'] == 'bias_act' else 1.0)
    with torch.no_grad():
        if c['op'] == 'bias_act':
            b = torch.randn(c['shape'][c['dim']], device=DEV, generator=g) * 0.5
            kw = dict(act=c['act'], clamp=c.get('clamp'))
            y = ops.bias_act.bias_act(x, b, dim=c['dim'], **kw)
            idx, alpha, gain = ACTS[c['act']]
            ref = bias_act_reference(x, b.to(dt), c['dim'], c['act'], alpha, gain, c.get('clamp') if c.get('clamp') is not None else -1.0)
            errs = {f'ba.{_dts(dt)}.{c["act"]}': ulp_err(y, ref, dt)}
        elif c['op'] == 'filtered_lrelu':
            fu, fd = _filter(c['fu'], g), _filter(c['fd'], g)
            b = (torch.randn(c['shape'][1], device=DEV, generator=g) * 0.5).to(dt)
            kw = dict(up=c['up'], down=c['down'], padding=c['pad'], clamp=c.get('clamp'), flip_filter=c.get('flip', False))
            y = ops.filtered_lrelu.filtered_lrelu(x, fu, fd, b, **kw)
            ref, R = flrelu_reference(x, fu, fd, b, c['up'], c['down'], c['pad'], SQRT2, 0.2, c.get('clamp'), c.get('flip', False))
            errs = {f'flrelu.{_dts(dt)}': fir_err(y, ref, R, dt)}
        else:
            f = _filter(c['f'], g)
            U = ops.upfirdn2d
            if c['op'] == 'upfirdn2d':
                y = U.upfirdn2d(x, f, up=c['up'], down=c['down'], padding=c['pad'], flip_filter=c.get('flip', False), gain=c.get('gain', 1.0))
            elif c['op'] == 'filter2d':
                y = U.filter2d(x, f, padding=c['pad'])
            elif c['op'] == 'upsample2d':
                y = U.upsample2d(x, f)
            else:
                y = U.downsample2d(x, f)
            up, down, pad, gain = _wrapper_fir_args(c)
            ref, R = fir_reference(x, f, up, down, pad, c.get('flip', False), gain, dt)
            errs = {f'fir.{_dts(dt)}': fir_err(y, ref, R, dt)}
    assert y.dtype == dt and y.shape == ref.shape, (c['name'], y.dtype, y.shape, ref.shape)
    fmt = suggested_format(x)
    assert y.is_contiguous(memory_format=fmt), (c['name'], fmt, y.stride())
    _assert_bounds(c['name'], errs)


# ------------------------------------------------------------------------------------------------ refusals (CPU, nothing launched)
def test_bias_act_refuses_bad_arguments():
    L = lib()
    x, y, b = torch.zeros(64), torch.zeros(64), torch.zeros(4)
    call = lambda act=3, dtype=0, bp=b.data_ptr(), size_b=4: L.lib.n3d_bias_act(x.data_ptr(), bp, y.data_ptr(), dtype, 64, size_b, 1, act,  # noqa: E731
                                                                                 0.2, 1.0, -1.0, None)
    assert L.lib.n3d_bias_act(None, None, None, 0, 0, 0, 0, 3, 0.2, 1.0, -1.0, None) == 0      # numel 0: an empty tensor's NULL pointer
    refused(L.lib.n3d_bias_act(None, None, y.data_ptr(), 0, 64, 0, 0, 3, 0.2, 1.0, -1.0, None), 'null pointer')
    refused(call(act=0), 'act 0 out of range')
    refused(call(act=10), 'act 10 out of range')
    refused(call(dtype=2), 'unsupported dtype 2')
    refused(call(size_b=0), 'bad bias geometry')


def test_upfirdn2d_refuses_bad_arguments():
    L = lib()
    x, y, f = torch.zeros(4 * 8 * 8), torch.zeros(4 * 64 * 64), torch.zeros(1025)
    strides = (L.I64 * 4)(256, 64, 8, 1)

    def call(fh=4, fw=4, up=(1, 1), down=(1, 1), out=(5, 5), dtype=0):
        return L.lib.n3d_upfirdn2d(x.data_ptr(), f.data_ptr(), y.data_ptr(), dtype, 1, 4, 8, 8, strides, strides, fh, fw, up[0], up[1],
                                   down[0], down[1], 0, 0, 0, 0, 0, 1.0, out[0], out[1], None)
    refused(call(fh=25, fw=41), 'filter 25x41 not supported')
    refused(call(fh=1, fw=1025, out=(8, 1)), 'filter 1x1025 not supported')
    refused(call(up=(0, 1)), 'bad up/down factors')
    refused(call(down=(1, 0)), 'bad up/down factors')
    refused(call(out=(5, 6)), 'output size 5x6, expected 5x5')
    refused(call(out=(4, 5)), 'output size 4x5, expected 5x5')
    refused(call(dtype=2), 'unsupported dtype 2')


def test_filtered_lrelu_refuses_bad_arguments():
    L = lib()
    x, y, tmp, f = torch.zeros(4 * 8 * 8), torch.zeros(4 * 64 * 64), torch.zeros(4 * 64 * 64), torch.zeros(1025)

    def call(fu=(4, 4), fd=(4, 4), up=2, down=2, out=(7, 7)):
        return L.lib.n3d_filtered_lrelu(x.data_ptr(), f.data_ptr(), f.data_ptr(), None, y.data_ptr(), tmp.data_ptr(), 0, 1, 4, 8, 8, fu[0], fu[1],
                                        fd[0], fd[1], up, down, 1, 2, 1, 2, 1.4, 0.2, -1.0, 0, out[0], out[1], None)
    assert (16 + 3 - 4 + 1 - 4 + 2) // 2 == 7                   # the output size of the call's default arguments
    refused(call(fd=(20, 4)), 'upsampled image smaller than the down filter')
    refused(call(out=(7, 8)), 'bad output size')
    refused(call(fu=(33, 32), out=(0, 0)), 'bad filter / factors')
    refused(call(fd=(1, 1025), out=(0, 0)), 'bad filter / factors')
