"""The fp16 instances of conv_gemm (N3DConvGemm.f16 = 1) and the fp16 single outputs of the conv, split-K and FIR-up epilogues, modulate
and resize, against the contract in include/next3d_b200.h.

The convolution reference is the fp64 product of exactly the fp16 operands the kernel gets (an fp16 x fp16 product is exact in
fp64), so what is left is the fp32 accumulation order and the fp32 epilogue.  Wherever a launch also writes the fp32 output of the same
epilogue values, an fp16 single output must equal fp16(fp32 output * style) bit for bit: both are formed from the same fp32 value, one
store rounded to fp16.  Every fp16 output is also held to the fp64 value within half an fp16 ulp plus the fp32 error.

Every output is a view into a larger allocation filled with a NaN sentinel (tests/helpers.Guarded): the elements a launch owns must
be written, all others must keep the sentinel's bits.  Every case is rerun and must be bit-identical.

The launch rule is the bf16 suite's mirror (tests/test_gpu_conv_conformance.plan / transposed_plan) with f16=True.  The CPU test
checks that the case table reaches everything in COVERAGE, including every SR launch the engine issues in fp16 mode
(engine_sr_launches); the profiler tests check that each case, and the engine itself, ran the conv_gemm_f16_kernel<block_n, block_k>
and grid the mirror predicts.
"""
import ctypes as C
import math
import re

import pytest
import torch
import torch.nn.functional as F

from tests.helpers import Guarded, grid_stride, launched_kernels, lib, record_errors, refused, rerun_identical
from tests.test_gpu_conv_conformance import (Expected, _f32_path, _place, _place_slice, _split_paths, block_k_for, conv_reference,
                                             epilogue_reference, plan, reachable_instances, transposed_plan)
from tests.test_gpu_fir_conformance import fir_up_plan

DEV = 'cuda'
SMS = 132                   # SM count the tables are planned at (H100 SXM)

# Range-relative bounds, max |got - ref| / max |ref| over the owned elements, each at most 4x the worst case measured over the table
# on an H100 SXM 80 GB (700 W power limit), which is given beside it.  N3D_CONV16_ERRORS=<file> appends every measured error to that
# file as JSON lines.
BOUNDS = {'raw': 6.5e-6,            # mode 1 and transposed raw sums; worst 1.74e-6 (multi_item_transposed)
          'splitk.raw': 1.7e-6,     # split-K partial sums; worst 4.2e-7 (splitk3)
          'f32': 3.4e-5,            # fp32 output of the conv epilogue; worst 8.5e-6 (sr8x_b0conv1_rgb256)
          'splitk.f32': 2.9e-6,     # fp32 output of n3d_splitk_epilogue after the split-K partial sums; worst 7.4e-7 (splitk3)
          'subnormal.f32': 2.2e-6,  # every activation an fp16 subnormal (a flushed operand would be an error of order 1); worst 5.5e-7
          'large.f32': 3.6e-6,      # activations near +-65504; worst 9.2e-7
          'rgb': 5.6e-6,            # fused ToRGB image; worst 1.4e-6 (sr8x_b0conv1_rgb256)
          'f16': 6e-4,              # an fp16 output against the fp64 value: half an fp16 ulp (2^-11 = 4.9e-4 of the value) plus the
                                    # fp32 error; worst 4.43e-4 (bn128_cluster_pingpong)
          'glue.f16': 6e-4}         # the fp16 outputs of a fir-up launch without an fp32 output against fp64: the same half ulp;
                                    # worst 3.3e-4 (up16_no_f32)


# ------------------------------------------------------------------------------------------------ the case table
def _case(name, N, Cin, Cout, MH, MW, **kw):
    """taps: '3x3', '1x1', 's2' (stride-2 taps over parity sub-images), 'tr10' (one transposed parity class, mode 1) or 'transposed'
    (the whole n3d_conv_transposed_gemm launch).  values: 'normal', 'subnormal' (every activation an fp16 subnormal), 'large'
    (activations near +-65504) or 'outedge' (styles that take v * s past 65504 and into the fp16 subnormal range).  f32=False: no
    fp32 output (the fp16 outputs are then held to fp64 only)."""
    c = dict(name=name, N=N, Cin=Cin, Cout=Cout, MH=MH, MW=MW, taps='3x3', mode=0, splits=1, epi='full', noise='shared', outs=None,
             f32=None, rgb=None, epi_noise='sample', values='normal', clamp=2.0)
    c.update(kw)
    transposed = c['taps'] == 'transposed'
    if c['mode'] == 1 or transposed:
        c['epi'], c['noise'] = 'none', None
    if c['outs'] is None:           # default: an fp16 output of its own and one into the second half of a concat buffer
        c['outs'] = [] if c['mode'] == 1 or transposed else [dict(cstride=Cout, coff=0), dict(cstride=2 * Cout, coff=Cout)]
    if c['f32'] is None and not transposed:
        c['f32'] = dict(cstride=Cout, coff=0, nchw=False, acc=False)
    c['f32'] = c['f32'] or None
    return c


TORGB = dict(epi='torgb', noise=None, outs=[], taps='1x1')     # ToRGBLayer as the engine issues it: linear, bias, clamp, NCHW +=
RGB_ENGINE = dict(ch=3, nchw=False, acc=True)                  # block0's fused ToRGB (block1's is NCHW)
CASES = [
    # the SR launches of the 8XDC head (32 -> 256 -> 128 channels) and the 4X head (32 -> 128 -> 64), each at a reduced size with the
    # engine's selection (see engine_sr_launches)
    _case('sr8x_b0conv0_transposed', 1, 32, 256, 64, 64, taps='transposed'),
    _case('sr8x_b0conv1_rgb256', 1, 256, 256, 32, 32, rgb=RGB_ENGINE, outs=[dict(cstride=256, coff=0)]),     # two 128-wide n-tiles
    _case('sr8x_b1conv0_transposed', 1, 256, 128, 16, 16, taps='transposed'),
    _case('sr8x_b1conv1_rgb128_cluster', 1, 128, 128, 64, 64, rgb=dict(ch=3, nchw=True, acc=True), outs=[]),   # the last layer
    _case('sr4x_b0conv0', 2, 32, 128, 64, 64, outs=[dict(cstride=128, coff=0)]),
    _case('sr4x_b0conv1_rgb128', 1, 128, 128, 32, 32, rgb=RGB_ENGINE, outs=[dict(cstride=128, coff=0)]),
    _case('sr4x_b1conv0_transposed', 2, 128, 64, 64, 64, taps='transposed'),
    _case('sr4x_b1conv1_rgb64', 1, 64, 64, 32, 32, rgb=dict(ch=3, nchw=True, acc=True), outs=[]),
    # clusters with a pad tile and two fp16 outputs (one into a concat buffer); narrow tiles
    _case('pad_tile_cluster', 5, 128, 128, 104, 16, outs=[dict(cstride=128, coff=0), dict(cstride=256, coff=128)]),
    _case('bn16_concat', 2, 64, 16, 16, 16, outs=[dict(cstride=24, coff=8)]),
    _case('bn32_bk32', 1, 96, 40, 8, 16),
    # several work items per CTA (cluster): both consumer warpgroups and the ring's wrap-around, as at the SR's full sizes
    _case('multi_item_cluster', 2, 128, 128, 128, 128),
    _case('multi_item_rgb128', 1, 128, 128, 256, 256, rgb=dict(ch=3, nchw=True, acc=True), outs=[]),
    _case('multi_item_bn64', 2, 64, 64, 128, 128),
    _case('multi_item_transposed', 2, 256, 128, 64, 64, taps='transposed'),
    # every other instance: (16, 32) at TN 8, (32, 64) at TN 2 with a Cin tail, (64, 32) staged, 96 / 128 unclustered and clustered
    _case('bn16_bk32_tn8_sample', 9, 32, 16, 4, 4, noise='sample', f32=dict(cstride=17, coff=1, nchw=False, acc=False)),
    _case('bn32_bk64_tn2_cin40', 3, 40, 40, 8, 8, f32=dict(cstride=44, coff=4, nchw=False, acc=False), outs=[dict(cstride=44, coff=4)]),
    _case('bn64_bk32_sample_staged_nchw', 2, 32, 64, 64, 64, noise='sample', f32=dict(cstride=64, coff=0, nchw=True, acc=False)),
    _case('bn96_bk32_rgb_unclustered', 1, 32, 96, 8, 16, rgb=dict(ch=3, nchw=True, acc=True), outs=[dict(cstride=96, coff=0)]),
    _case('bn96_bk64_rgb_unclustered', 1, 64, 96, 8, 16, rgb=dict(ch=1, nchw=False, acc=False), outs=[dict(cstride=96, coff=0)]),
    _case('bn96_bk32_rgb_cluster_pad', 3, 32, 96, 8, 16, rgb=dict(ch=4, nchw=True, acc=False), outs=[dict(cstride=96, coff=0)]),
    _case('bn96_bk64_rgb_cluster', 2, 64, 96, 16, 16, rgb=dict(ch=4, nchw=False, acc=False), outs=[dict(cstride=192, coff=96)]),
    _case('bn128_bk32_rgb_unclustered', 1, 32, 128, 8, 16, rgb=dict(ch=1, nchw=False, acc=False), outs=[dict(cstride=128, coff=0)]),
    _case('bn128_bk64_rgb_unclustered', 1, 64, 128, 8, 16, rgb=dict(ch=4, nchw=True, acc=True), outs=[dict(cstride=128, coff=0)]),
    _case('rgb192_cluster_two_tiles', 2, 64, 192, 16, 16, rgb=dict(ch=1, nchw=True, acc=False), outs=[dict(cstride=192, coff=0)]),
    _case('rgb40_four_channels', 2, 80, 40, 16, 16, rgb=dict(ch=4, nchw=False, acc=True), outs=[dict(cstride=48, coff=8)]),
    # clusters: pad tiles, f32 accumulate (which takes no fp16 outputs), stride 2, TN 2, several items per cluster at block_k 64
    _case('bn128_cluster_pad_accumulate', 33, 24, 200, 8, 16, f32=dict(cstride=200, coff=0, nchw=False, acc=True), outs=[], noise='sample'),
    _case('bn128_cluster_stride2_pad', 5, 8, 128, 40, 40, taps='s2', noise='sample'),
    _case('bn128_cluster_tn2_pad', 129, 40, 128, 8, 8, noise='sample'),
    _case('bn96_cluster_torgb1x1_accumulate', 8, 80, 96, 32, 32, **TORGB, f32=dict(cstride=96, coff=0, nchw=False, acc=True)),
    _case('bn128_cluster_pingpong', 299, 8, 128, 8, 16),
    _case('bn96_cluster_multi_item_bk64', 200, 16, 96, 8, 16, outs=[dict(cstride=96, coff=0)]),
    # unclustered ping-pong (an odd count of items per CTA), TN > 1
    _case('bn32_pingpong_staged', 135, 16, 48, 8, 16, noise='sample', outs=[dict(cstride=48, coff=0), dict(cstride=56, coff=8)]),
    # 1x1 ToRGB launches at 4^2 and 8^2 (TN 8 and 2, N not a multiple of TN, NCHW accumulate)
    _case('torgb1x1_4x4', 9, 64, 3, 4, 4, **TORGB, f32=dict(cstride=3, coff=0, nchw=True, acc=True)),
    _case('torgb1x1_8x8', 5, 32, 3, 8, 8, **TORGB, f32=dict(cstride=3, coff=0, nchw=True, acc=True)),
    # fp16 store paths: uint4 and scalar, on their own and into a concat buffer; no fp32 output beside them
    _case('f16_uint4_own_and_concat', 2, 64, 24, 8, 16, outs=[dict(cstride=24, coff=0), dict(cstride=40, coff=8)]),
    _case('f16_scalar_own_and_concat', 2, 64, 12, 8, 16, outs=[dict(cstride=12, coff=0), dict(cstride=20, coff=4)]),
    _case('f16_only_no_f32', 2, 48, 32, 16, 16, f32=False, noise='sample'),
    # split-K through n3d_splitk_epilogue: 9 slices, 3 slices, 2 uneven slices (5 + 4 of 9 K steps)
    _case('splitk9', 2, 64, 64, 4, 4, mode=1, splits=9, epi_noise='shared'),
    _case('splitk3', 3, 80, 40, 8, 8, mode=1, splits=3),
    _case('splitk2_uneven', 2, 24, 72, 8, 8, mode=1, splits=2),
    # raw output of one transposed-conv parity class: every other output pixel belongs to another class
    _case('transposed_class10_raw', 2, 40, 64, 12, 13, mode=1, taps='tr10', f32=dict(cstride=64, coff=0, nchw=False, acc=False)),
    # fp16 value edges
    _case('subnormal_activations', 2, 64, 64, 16, 16, values='subnormal', clamp=-1.0),
    _case('large_activations', 2, 64, 64, 16, 16, values='large', clamp=-1.0),
    _case('output_edges', 2, 64, 64, 16, 16, values='outedge'),
    _case('output_edges_splitk', 2, 64, 32, 4, 4, mode=1, splits=3, values='outedge'),
]
CASE_IDS = [c['name'] for c in CASES]


def _plan(c, sms=SMS, cluster_slots=SMS // 2):
    if c['taps'] == 'transposed':
        return transposed_plan(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], sms, cluster_slots, f16=True)
    return plan(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], c['splits'], bool(c['rgb']), sms, cluster_slots, f16=True)


def selection(p):
    """What the engine inventory compares: (block_n, block_k, cluster, item_tiles, grouped)."""
    return p['block_n'], p['block_k'], p['cluster'], p['item_tiles'], p['grouped']


def engine_sr_launches(module, N, sms=SMS, cluster_slots=SMS // 2):
    """The fp16 SR launches Engine._superresolution issues, in order, for SR module '8XDC' / '4X' and batch N: the SR input is resized
    (or modulated) to r0 = 128, block0 runs at res0 = 2 r0 (8XDC, conv0 transposed) or r0 (4X), block1 at 2 res0 (conv0 transposed),
    and each conv1 carries the fused ToRGB.  -> [(what, shape, plan)]; a transposed conv's FIR-up follows it as ('fir_up', (N, H2, W2,
    C), fir_up_plan)."""
    from next3d_b200 import config
    cfg = config.GeneratorConfig(img_resolution={'8XDC': 512, '4X': 256}[module])
    c0, c1 = config.sr_channels(cfg)
    r0, cin = 128, cfg.plane_ch
    res0 = 2 * r0 if module == '8XDC' else r0
    convs = [('transposed', (N, cin, c0, r0, r0)) if module == '8XDC' else ('conv', (N, cin, c0, r0, r0)),
             ('rgb', (N, c0, c0, res0, res0)), ('transposed', (N, c0, c1, res0, res0)), ('rgb', (N, c1, c1, 2 * res0, 2 * res0))]
    out = []
    for what, (n, ci, co, h, w) in convs:
        if what == 'transposed':
            out.append((what, (n, ci, co, h, w), transposed_plan(n, ci, co, h, w, sms, cluster_slots, f16=True)))
            out.append(('fir_up', (n, 2 * h, 2 * w, co), fir_up_plan(n, 2 * h, 2 * w, co, sms)))
        else:
            out.append((what, (n, ci, co, h, w), plan(n, ci, co, h, w, rgb=what == 'rgb', sms=sms, cluster_slots=cluster_slots, f16=True)))
    return out


def engine_selections():
    """Every (selection, kind) of the engine's fp16 SR convolutions over both SR modules and N 1, 2, 4, 8."""
    return {(selection(p), what) for m in ('8XDC', '4X') for n in (1, 2, 4, 8) for what, _, p in engine_sr_launches(m, n) if what != 'fir_up'}


def _full_epilogue(c):
    return c['mode'] == 0 and c['epi'] == 'full' and c['noise'] is not None and bool(c['outs'])


def _kind(c):
    return 'transposed' if c['taps'] == 'transposed' else 'rgb' if c['rgb'] else 'conv'


def _odd3(n):
    return n >= 3 and n % 2 == 1


def _store_paths(c):
    """(fp16 store path, into a concat buffer) of each fp16 output of the case."""
    return {(next(iter(_split_paths(dict(outs=[o])))).replace('split', 'f16'), o['cstride'] > c['Cout'] and o['coff'] != 0) for o in c['outs']}


COVERAGE = {
    'every reachable fp16 instance (all 10) in mode 0 with the full epilogue':
        lambda cs: {(p['block_n'], p['block_k']) for c, p in cs if _full_epilogue(c) or (c['rgb'] and c['outs'])} == reachable_instances(True),
    'block_n 96 clustered': lambda cs: any(p['block_n'] == 96 and p['cluster'] == 2 and c['mode'] == 0 for c, p in cs),
    'block_n 96 unclustered': lambda cs: any(p['block_n'] == 96 and p['cluster'] == 1 and c['mode'] == 0 for c, p in cs),
    'block_n 128 clustered': lambda cs: any(p['block_n'] == 128 and p['cluster'] == 2 and c['mode'] == 0 for c, p in cs),
    'block_n 128 unclustered': lambda cs: any(p['block_n'] == 128 and p['cluster'] == 1 and c['mode'] == 0 for c, p in cs),
    'TN 1, 2 and 8': lambda cs: {1, 2, 8} <= {p.get('TN') for c, p in cs},
    'TN 2 and 8 with N not a multiple of TN': lambda cs: {2, 8} <= {p['TN'] for c, p in cs if 'TN' in p and c['N'] % p['TN']},
    'clustered TN 2': lambda cs: any(p.get('TN') == 2 and p['cluster'] == 2 for c, p in cs),
    'pad tile with f32_accumulate': lambda cs: any(p['pad'] and c['f32'] and c['f32']['acc'] for c, p in cs),
    'pad tile in a stride-2 launch': lambda cs: any(p['pad'] and c['taps'] == 's2' for c, p in cs),
    'odd count >= 3 of items per CTA, unclustered':
        lambda cs: any(p['cluster'] == 1 and p['block_n'] <= 64 and _odd3(p['items_per_cta']) for c, p in cs),
    'odd count >= 3 of items per cluster': lambda cs: any(p['cluster'] == 2 and _odd3(p['items_per_cta']) for c, p in cs),
    'several items per CTA at block_k 64 on block_n 96 and 128 (6 stages)':
        lambda cs: {p['block_n'] for c, p in cs if p['block_k'] == 64 and p['items_per_cta'] >= 2 and p['stages'] == 6} >= {96, 128},
    'split-K S 9, 3 and 2': lambda cs: {9, 3, 2} <= {c['splits'] for c, p in cs},
    'split-K with uneven slices': lambda cs: any(c['splits'] > 1 and (9 * -(-c['Cin'] // p['block_k'])) % c['splits'] for c, p in cs),
    'mode-1 raw output of one transposed parity class': lambda cs: any(c['taps'] == 'tr10' and c['mode'] == 1 for c, p in cs),
    '1x1 ToRGB launches at 4x4 and 8x8': lambda cs: {4, 8} <= {c['MH'] for c, p in cs if c['epi'] == 'torgb' and c['f32']['nchw']},
    'stride-2 taps': lambda cs: any(c['taps'] == 's2' for c, p in cs),
    'Cin 8, 24, 40': lambda cs: {8, 24, 40} <= {c['Cin'] for c, p in cs},
    # block_k 32 is chosen only for Cin % 64 == 32 in fp16 (the ring always holds 4 stages of 64), so a Cin tail (Cin % block_k != 0)
    # exists at block_k 64 only; test_block_k32_has_no_cin_tail_in_fp16 checks that
    'Cin tails at block_k 64, and block_k 32': lambda cs: any(c['Cin'] % 64 not in (0, 32) and p['block_k'] == 64 for c, p in cs)
        and any(p['block_k'] == 32 for c, p in cs),
    'Cout % 16 != 0 on narrow tiles': lambda cs: any(c['Cout'] % 16 and p['block_n'] <= 64 and c['Cout'] > 16 for c, p in cs),
    'Cout % 16 != 0 on wide tiles': lambda cs: any(c['Cout'] % 16 and p['block_n'] >= 96 for c, p in cs),
    'fp16 stores: 256-bit, uint4, scalar, each on its own and into a concat buffer':
        lambda cs: {(k, cat) for k in ('f16_256', 'f16_uint4', 'f16_scalar') for cat in (False, True)} <= set().union(*(_store_paths(c) for c, p in cs)),
    'two fp16 outputs in one launch': lambda cs: any(len(c['outs']) == 2 and c['mode'] == 0 for c, p in cs),
    'fp32 stores: 256-bit, float4, scalar, NCHW, NCHW accumulate':
        lambda cs: {'f32_256', 'f32_float4', 'f32_scalar', 'nchw', 'nchw_accumulate'} <= {_f32_path(c) for c, p in cs},
    'fp16 outputs without an fp32 output': lambda cs: any(c['outs'] and c['f32'] is None and c['mode'] == 0 for c, p in cs),
    'per-sample noise, staged (TN 1)': lambda cs: any(c['noise'] == 'sample' and p['TN'] == 1 and p['cluster'] == 1 for c, p in cs if 'TN' in p),
    'per-sample noise, unstaged (TN > 1)': lambda cs: any(c['noise'] == 'sample' and p['TN'] > 1 for c, p in cs if 'TN' in p),
    'per-sample noise, clustered': lambda cs: any(c['noise'] == 'sample' and p['cluster'] == 2 for c, p in cs),
    'per-sample noise through the split-K epilogue': lambda cs: any(c['splits'] > 1 and c['epi_noise'] == 'sample' for c, p in cs),
    'fused ToRGB with 1, 3, 4 channels': lambda cs: {1, 3, 4} <= {c['rgb']['ch'] for c, p in cs if c['rgb']},
    'fused ToRGB over one and two n-tiles': lambda cs: {1, 2} <= {p['item_tiles'] for c, p in cs if c['rgb']},
    'subnormal and large activations, output edges through the conv and split-K epilogues':
        lambda cs: {'subnormal', 'large'} <= {c['values'] for c, p in cs} and {c['splits'] > 1 for c, p in cs if c['values'] == 'outedge'} == {False, True},
    'every fp16 SR launch of the engine (both SR modules, N 1, 2, 4, 8)':
        lambda cs: engine_selections() <= {(selection(p), _kind(c)) for c, p in cs},
}


def test_case_table_covers_every_sr_launch_form():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rule."""
    planned = [(c, _plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(reachable_instances(True)) == 10
    assert len(set(CASE_IDS)) == len(CASE_IDS)


def test_block_k32_has_no_cin_tail_in_fp16():
    """CPU: fp16 launches take block_k 32 exactly for Cin % 64 == 32, at every block_n."""
    assert all(block_k_for(cin, bn, f16=True) == (32 if cin % 64 == 32 else 64) for bn in (16, 32, 64, 96, 128) for cin in range(8, 520, 8))


def test_engine_sr_launches_use_the_large_selections():
    """CPU: the engine's first SR convolution runs conv_gemm_f16_kernel<128, 32> (8XDC transposed, grouped; 4X 3x3), clustered, at
    every batch size."""
    for n in (1, 2, 4, 8):
        assert selection(engine_sr_launches('8XDC', n)[0][2]) == (128, 32, 2, 1, True)
        assert selection(engine_sr_launches('4X', n)[0][2]) == (128, 32, 2, 1, False)


# ------------------------------------------------------------------------------------------------ one case
def _taps(c):
    from next3d_b200 import kernels as K
    return {'3x3': K.taps_conv3x3, '1x1': K.taps_conv1x1, 's2': K.taps_stride2, 'tr10': lambda: K.taps_transposed(1, 0),
            'transposed': K.taps_conv3x3}[c['taps']]()


def _geometry(c):
    """(NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW) of a case."""
    N, MH, MW = c['N'], c['MH'], c['MW']
    if c['taps'] == 's2':           # parity sub-images of a 2 MH x 2 MW input padded by the FIR: [4N, MH + 1, MW + 1]
        return 4 * N, MH + 1, MW + 1, N, 1, 0, 1, 0, MH, MW
    if c['taps'] == 'tr10':         # class (1, 0) of a stride-2 transposed conv of an MH x (MW - 1) input
        H, W = MH, MW - 1
        return N, H, W, 0, 2, 1, 2, 0, 2 * H + 1, 2 * W + 1
    if c['taps'] == 'transposed':
        return N, MH, MW, 0, 2, 0, 2, 0, 2 * MH + 1, 2 * MW + 1
    return N, MH, MW, 0, 1, 0, 1, 0, MH, MW


def _seeded(c):
    return torch.Generator(device=DEV).manual_seed(3000 + CASE_IDS.index(c['name']))


def _operands(c, g, NI, AH, AW, T, ntaps):
    """fp16 activations and weights of the case's value class (the weights scaled so that the outputs are normal fp16/fp32 values)."""
    Cin, Cout = c['Cin'], c['Cout']
    x = torch.randn(NI, AH, AW, Cin, device=DEV, generator=g)
    w = torch.randn(T, Cout, Cin, device=DEV, generator=g) / math.sqrt(Cin * ntaps)
    if c['values'] == 'subnormal':      # |a| in [2^-18, 2^-14): subnormal after the rounding, none zero
        x = torch.sign(x + 1e-3) * (2.0 ** -14) * (0.06 + 0.93 * torch.rand(x.shape, device=DEV, generator=g))
        w = w * 2.0 ** 14
    elif c['values'] == 'large':        # |a| in [32752, 65504]
        x = torch.sign(x + 1e-3) * 65504.0 * (0.5 + 0.5 * torch.rand(x.shape, device=DEV, generator=g))
        w = w * 2.0 ** -8
    return x.half(), w.half()


def _styles(c, g, n):
    N, Cout = c['N'], c['Cout']
    if c['values'] != 'outedge':
        return [torch.randn(N, Cout, device=DEV, generator=g) for _ in range(n)]
    # |v| <= 2 (the clamp): these take v * s past 65504 (to 65504 or inf by round-to-nearest) and into the fp16 subnormal range
    edge = torch.tensor([7e4, -7e4, 4e4, -3.3e4, 1e5, 3.3e4, 1e-5, -3e-6, 6e-8, -1e-9, 1.0, -2e4], device=DEV)
    idx = torch.arange(N * Cout, device=DEV).reshape(N, Cout)
    return [edge[(idx + k) % len(edge)] * (1 + 0.05 * torch.rand(N, Cout, device=DEV, generator=g)) for k in range(n)]


def setup_case(c):
    """Operands, epilogue vectors, guarded outputs and their fp64 references."""
    g = _seeded(c)
    N, Cin, Cout = c['N'], c['Cin'], c['Cout']
    NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW = geo = _geometry(c)
    taps = _taps(c)
    T = max(t[3] for t in taps) + 1
    a, w = _operands(c, g, NI, AH, AW, T, len(taps))
    s = dict(c=c, taps=taps, a=a, w=w, geo=geo, priors=[])
    if c['taps'] == 'transposed':
        s['raw'] = Expected((N, OH, OW, Cout), torch.float32)
        s['raw'].own[:] = True
        s['raw'].expect = _transposed_reference(a, w)
        return s
    if c['epi'] == 'full':
        s.update(dcoef=torch.rand(N, Cout, device=DEV, generator=g) + 0.5, bias=torch.randn(Cout, device=DEV, generator=g) * 0.5,
                 gain=math.sqrt(2), slope=0.2, clamp=c['clamp'])
    elif c['epi'] == 'torgb':
        s.update(dcoef=None, bias=torch.randn(Cout, device=DEV, generator=g), gain=1.0, slope=1.0, clamp=1.5)
    else:
        s.update(dcoef=None, bias=None, gain=1.0, slope=1.0, clamp=-1.0)
    s['noise'], s['noise_nstride'] = None, 0
    if c['noise'] == 'shared':
        s['noise'] = torch.randn(OH, OW, device=DEV, generator=g) * 0.3
    elif c['noise'] == 'sample':
        s['noise'], s['noise_nstride'] = torch.randn(N, OH, OW, device=DEV, generator=g) * 0.3, OH * OW
    s['styles'] = _styles(c, g, len(c['outs']))
    s['outs'] = [Expected((N, OH, OW, o['cstride']), torch.float16) for o in c['outs']]
    f = c['f32']
    s['f32'] = None
    if f is not None:
        shape = (N, f['cstride'], OH, OW) if f['nchw'] else (N, OH, OW, f['cstride'])
        s['f32'] = Expected(((c['splits'],) if c['splits'] > 1 else ()) + shape, torch.float32)
    r = c['rgb']
    if r:
        s['rgb_w'] = torch.randn(r['ch'], Cout, device=DEV, generator=g)
        s['rgb_s'] = torch.randn(N, Cout, device=DEV, generator=g) / math.sqrt(Cout)
        s['rgb_b'] = torch.randn(r['ch'], device=DEV, generator=g)
        s['rgb'] = Expected((N, r['ch'], OH, OW) if r['nchw'] else (N, OH, OW, r['ch']), torch.float32)
    if c['splits'] > 1:             # second pass: n3d_splitk_epilogue with the full epilogue into fresh guarded fp16 / fp32 outputs
        s.update(dcoef=torch.rand(N, Cout, device=DEV, generator=g) + 0.5, bias=torch.randn(Cout, device=DEV, generator=g) * 0.5,
                 gain=math.sqrt(2), slope=0.2, clamp=2.0)
        per_sample = c['epi_noise'] == 'sample'
        s['noise'] = torch.randn(*((N,) if per_sample else ()), OH, OW, device=DEV, generator=g) * 0.3
        s['noise_nstride'] = OH * OW if per_sample else 0
        s['epi_styles'] = _styles(c, g, 2)
        s['epi_outs'] = [Expected((N, OH, OW, cs), torch.float16) for cs in (Cout, 2 * Cout)]
        s['epi_f32'] = Expected((N, OH, OW, Cout), torch.float32)
    yv = torch.nonzero(torch.arange(c['MH'], device=DEV) * oy_mul + oy_off < OH).flatten()
    xv = torch.nonzero(torch.arange(c['MW'], device=DEV) * ox_mul + ox_off < OW).flatten()
    oy = torch.arange(c['MH'], device=DEV) * oy_mul + oy_off
    ox = torch.arange(c['MW'], device=DEV) * ox_mul + ox_off
    _expect(s, yv, xv, oy, ox)
    return s


def _transposed_reference(a, w):
    """fp64 conv_transpose2d(stride 2) of the fp16 operands: a [N,H,W,Cin], w [9,Cout,Cin] -> [N, 2H+1, 2W+1, Cout];
    out[2p+a, 2q+b] = sum W[ky,kx] x[p-(ky-a)/2, q-(kx-b)/2]."""
    x = a.double().permute(0, 3, 1, 2)
    k = w.double().reshape(3, 3, w.shape[1], w.shape[2])
    return F.conv_transpose2d(x, k.permute(3, 2, 0, 1), stride=2).permute(0, 2, 3, 1).contiguous()


def _expect(s, yv, xv, oy, ox):
    c = s['c']
    p = _plan(c)
    N, MH, MW = c['N'], c['MH'], c['MW']
    NI, AH, AW, a_img_mul, *_, OH, OW = s['geo']
    ref = lambda **kw: conv_reference(s['a'], None, s['w'], s['w'], s['taps'], N, MH, MW, a_img_mul, 1, **kw)      # noqa: E731
    epi = lambda acc: epilogue_reference(acc, oy, ox, OW, s['dcoef'], s['bias'], s['noise'], s['noise_nstride'], s['gain'],  # noqa: E731
                                         s['slope'], s['clamp'])
    f = c['f32']
    if c['splits'] > 1:
        nsteps = len(s['taps']) * -(-c['Cin'] // p['block_k'])
        per = -(-nsteps // c['splits'])
        total = 0
        for k in range(c['splits']):
            part = ref(block_k=p['block_k'], k_steps=(k * per, (k + 1) * per))
            _place_slice(s['f32'], k, part, yv, xv, oy, ox)
            total = total + part
        v = epi(total)
        for t, sty, coff in zip(s['epi_outs'], s['epi_styles'], (0, c['Cout'])):
            _place(t, v * sty.double()[:, None, None, :], yv, xv, oy, ox, coff, False)
        _place(s['epi_f32'], v, yv, xv, oy, ox, 0, False)
        return
    acc = ref()
    v = acc if c['mode'] == 1 else epi(acc)
    for t, sty, o in zip(s['outs'], s['styles'], c['outs']):
        _place(t, v * sty.double()[:, None, None, :], yv, xv, oy, ox, o['coff'], False)
    g = _seeded(c)
    if f is not None:
        prior = None
        if f['acc']:                # accumulating output: finite prior content in the owned region
            _place(s['f32'], v, yv, xv, oy, ox, f['coff'], f['nchw'])
            s['f32'].view[s['f32'].own] = torch.randn(int(s['f32'].own.sum()), device=DEV, generator=g)
            prior = s['f32'].view.clone()
            s['priors'].append((s['f32'], prior))
        _place(s['f32'], v, yv, xv, oy, ox, f['coff'], f['nchw'], prior)
    r = c['rgb']
    if r:
        img = torch.einsum('nyxo,no,co->nyxc', v, s['rgb_s'].double(), s['rgb_w'].double()) + s['rgb_b'].double()
        img = img.clamp(-2.0, 2.0)
        prior = None
        if r['acc']:
            _place(s['rgb'], img, yv, xv, oy, ox, 0, r['nchw'])
            s['rgb'].view[s['rgb'].own] = torch.randn(int(s['rgb'].own.sum()), device=DEV, generator=g)
            prior = s['rgb'].view.clone()
            s['priors'].append((s['rgb'], prior))
        _place(s['rgb'], img, yv, xv, oy, ox, 0, r['nchw'], prior)


def outputs(s):
    c = s['c']
    if c['taps'] == 'transposed':
        return [s['raw']]
    out = list(s['outs']) + [t for t in (s['f32'], s.get('rgb')) if t is not None]
    if c['splits'] > 1:
        out += list(s['epi_outs']) + [s['epi_f32']]
    return out


def launch_case(s):
    from next3d_b200 import kernels as K
    c = s['c']
    for t, prior in s['priors']:        # an accumulating output starts from its prior content
        t.view.copy_(prior)
    if c['taps'] == 'transposed':
        K.conv_transposed_gemm(s['a'], None, s['w'], None, c['N'], c['MH'], c['MW'], s['raw'].view, nprod=1)
        return
    NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW = s['geo']
    mode0 = c['mode'] == 0
    outs = [K.make_split_out(t.view, None, sty if mode0 else None, o['cstride'], o['coff'], f16=True)
            for t, sty, o in zip(s['outs'], s['styles'], c['outs'])]
    f = c['f32']
    kw = {}
    if f is not None:
        kw = dict(out_f32=s['f32'].view, f32_cstride=f['cstride'], f32_coff=f['coff'], f32_nchw=f['nchw'], f32_accumulate=f['acc'])
    if c['rgb']:
        r = c['rgb']
        kw['rgb'] = dict(out=s['rgb'].view, weight=s['rgb_w'], style=s['rgb_s'], bias=s['rgb_b'], clamp=2.0, nchw=r['nchw'], accumulate=r['acc'])
    if c['splits'] > 1:
        kw.update(splits=c['splits'], split_stride=s['f32'].view[0].numel())
    K.conv_gemm(s['a'], None, s['w'], None, s['taps'], c['N'], c['MH'], c['MW'], a_img_mul=a_img_mul, nprod=1, mode=c['mode'],
                dcoef=s['dcoef'] if mode0 else None, bias=s['bias'] if mode0 else None, noise=s['noise'] if mode0 else None,
                noise_nstride=s['noise_nstride'] if mode0 else 0, gain=s['gain'], slope=s['slope'], clamp=s['clamp'], outs=outs,
                oy_mul=oy_mul, oy_off=oy_off, ox_mul=ox_mul, ox_off=ox_off, OH=OH, OW=OW, **kw)
    if c['splits'] > 1:
        Cout = c['Cout']
        eouts = [K.make_split_out(t.view, None, sty, cs, coff, f16=True)
                 for t, sty, (cs, coff) in zip(s['epi_outs'], s['epi_styles'], ((Cout, 0), (2 * Cout, Cout)))]
        K.splitk_epilogue(s['f32'].view, s['dcoef'], s['bias'], s['noise'], s['gain'], s['slope'], s['clamp'], outs=eouts,
                          out_f32=s['epi_f32'].view, f32_cstride=Cout, f32_coff=0, noise_nstride=s['noise_nstride'])


def _err(got, g):
    ref = g.expect[g.own]
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def _nhwc(view, f):
    """The channels [coff, coff + Cout) of an fp32 output, NHWC."""
    v = view.permute(0, 2, 3, 1) if f.get('nchw') else view
    return v[..., f['coff']:]


def check_case(s):
    """-> {output: (bound kind, range-relative error)}; asserts the sentinel, written-element and fp16 bit-identity checks."""
    c = s['c']
    Cout = c['Cout']
    errs = {}
    pre = c['values'] + '.' if c['values'] in ('subnormal', 'large') else ''

    def guarded(name, g, accumulate=False):
        assert g.untouched_ok(), f'{c["name"]}.{name}: an element outside the output was written'
        assert accumulate or g.written(), f'{c["name"]}.{name}: an owned element was not written'

    def f16(name, t, sty, coff, f32):
        """An fp16 output: fp16(fp32 output * style) bit for bit where the fp32 output exists, and within the f16 bound of fp64."""
        guarded(name, t)
        got = t.view[..., coff:coff + Cout]
        if f32 is not None:
            want = (f32[..., :Cout] * sty[:, None, None, :]).half()
            assert torch.equal(got.view(torch.int16), want.view(torch.int16)), \
                (c['name'], name, 'not fp16(fp32 output * style)', int((got.view(torch.int16) != want.view(torch.int16)).sum()))
        if c['values'] != 'outedge':
            errs[name] = ('f16', _err(t.view[t.own].double(), t))

    if c['taps'] == 'transposed':
        guarded('raw', s['raw'])
        errs['raw'] = ('raw', _err(s['raw'].view[s['raw'].own].double(), s['raw']))
        return errs
    f = c['f32']
    if s['f32'] is not None:
        acc = f['acc']
        guarded('f32', s['f32'], acc)
        kind = ('splitk.raw' if c['splits'] > 1 else 'raw') if c['mode'] == 1 else pre + 'f32'
        errs['f32'] = (kind, _err(s['f32'].view[s['f32'].own].double(), s['f32']))
    f32 = _nhwc(s['f32'].view, f) if s['f32'] is not None and c['mode'] == 0 and not f['acc'] else None
    for k, (t, sty, o) in enumerate(zip(s['outs'], s['styles'], c['outs'])):
        f16(f'out{k}', t, sty, o['coff'], f32)
    if c['rgb']:
        guarded('rgb', s['rgb'], c['rgb']['acc'])
        errs['rgb'] = ('rgb', _err(s['rgb'].view[s['rgb'].own].double(), s['rgb']))
    if c['splits'] > 1:
        guarded('splitk_epilogue.f32', s['epi_f32'])
        errs['splitk_epilogue.f32'] = ('splitk.f32', _err(s['epi_f32'].view[s['epi_f32'].own].double(), s['epi_f32']))
        for k, (t, sty, coff) in enumerate(zip(s['epi_outs'], s['epi_styles'], (0, Cout))):
            f16(f'splitk_epilogue.out{k}', t, sty, coff, s['epi_f32'].view)
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_conv_gemm_f16_matches_fp64_contract(c):
    s = setup_case(c)
    if c['values'] == 'subnormal':
        assert bool(((s['a'] != 0) & (s['a'].abs() < 2.0 ** -14)).all())
    launch_case(s)
    torch.cuda.synchronize()
    errs = check_case(s)
    record_errors('N3D_CONV16_ERRORS', [{'case': c['name'], 'output': k, 'kind': kind, 'err': e, 'bound': BOUNDS[kind]}
                                        for k, (kind, e) in errs.items()])
    bad = {k: (kind, e) for k, (kind, e) in errs.items() if not e < BOUNDS[kind]}
    assert not bad, bad
    assert rerun_identical(outputs(s), lambda: launch_case(s)), f'{c["name"]}: a rerun is not bit-identical'


def _check_launch(name, e, p):
    m = re.search(r'conv_gemm_f16_kernel<(\d+), (\d+)>', e['name'])
    assert m and (int(m.group(1)), int(m.group(2))) == (p['block_n'], p['block_k']), (name, e['name'], p)
    grid = e.get('args', {}).get('grid')
    if grid is not None:
        assert list(grid) == [p['grid'], 1, 1], (name, grid, p)
    cl = e.get('args', {}).get('cluster')
    if cl is not None:
        assert list(cl)[0] == p['cluster'], (name, cl, p)


@pytest.mark.gpu
def test_launched_f16_instance_matches_plan(tmp_path):
    """Every case under torch.profiler: it launched the conv_gemm_f16_kernel<block_n, block_k>, grid and cluster the mirror predicts
    (transposed launches included)."""
    setups = [setup_case(c) for c in CASES]
    torch.cuda.synchronize()

    def run():
        for s in setups:
            launch_case(s)
        return CASES                        # one conv_gemm_f16_kernel launch per case

    _, events = launched_kernels(run, r'conv_gemm_f16_kernel', tmp_path)
    props = torch.cuda.get_device_properties(0)
    for c, e in zip(CASES, events):
        _check_launch(c['name'], e, _plan(c, props.multi_processor_count, props.multi_processor_count // 2))


@pytest.mark.gpu
@pytest.mark.parametrize('name', ['tiny512', 'full512'])
def test_engine_sr_launches_match_mirror(name, tmp_path, monkeypatch):
    """G.synthesis in fp16 mode under torch.profiler: its conv_gemm_f16_kernel launches are the engine_sr_launches the table reaches,
    with the predicted instance and grid, and its fir_up_* launches (backbone and SR) the kernel and grid fir_up_plan predicts."""
    from next3d_b200 import kernels as K
    from tests.test_gpu_sr_fp16 import _setup
    G, cfg, sd, ws, cam, v, noise = _setup(name)
    N = ws.shape[0]
    props = torch.cuda.get_device_properties(0)
    sms = props.multi_processor_count
    expect = engine_sr_launches(cfg.sr_module, N, sms, sms // 2)
    fir_calls = []
    fir_up = K.fir_up_epilogue

    def recording_fir_up(raw, C_, *a, **kw):
        fir_calls.append((raw.shape[0], raw.shape[1] - 1, raw.shape[2] - 1, C_))
        return fir_up(raw, C_, *a, **kw)

    monkeypatch.setattr(K, 'fir_up_epilogue', recording_fir_up)
    G.sr_precision = 'fp16'

    def synth():
        fir_calls.clear()
        with torch.no_grad():
            G.synthesis(ws, cam, v, noise_mode='const', sampler_noise=noise)
        torch.cuda.synchronize()

    def run_convs():
        synth()
        return [x for x in expect if x[0] != 'fir_up']

    def run_firs():
        synth()
        return list(fir_calls)

    convs, events = launched_kernels(run_convs, r'conv_gemm_f16_kernel', tmp_path)
    for (what, shape, p), e in zip(convs, events):
        _check_launch(f'{name}: {what} {shape}', e, p)
    covered = {(selection(_plan(c)), _kind(c)) for c in CASES}
    assert all((selection(p), what) in covered for what, _, p in convs)
    calls, events = launched_kernels(run_firs, r'fir_up_stream_kernel|fir_up_epilogue_kernel', tmp_path)
    assert calls[-2:] == [shape for what, shape, _ in expect if what == 'fir_up'], calls[-2:]
    for shape, e in zip(calls, events):
        p = fir_up_plan(*shape, sms)
        assert re.search(p['kernel'], e['name']), (shape, e['name'], p)
        grid = e.get('args', {}).get('grid')
        if grid is not None:
            assert list(grid) == [p['grid'], 1, 1], (shape, grid, p)


# ------------------------------------------------------------------------------------------------ fp16 single outputs of the glue kernels
@pytest.mark.gpu
@pytest.mark.parametrize('HW,C', [(16, 256), (32, 128), (8, 64), (128, 128), (64, 256)])     # the last two: the streamed kernel
def test_fir_up_epilogue_f16_output(HW, C):
    """n3d_fir_up_epilogue with one fp16 single and one split bf16 output: the fp16 one is fp16(fp32 output * style) bit for bit, the
    split one is unchanged by the other's format."""
    from next3d_b200 import kernels as K
    g = torch.Generator().manual_seed(HW * C)
    N = 2
    raw = torch.randn(N, 2 * HW + 1, 2 * HW + 1, C, generator=g).to(DEV)
    dcoef, bias = (torch.rand(N, C, generator=g) + 0.5).to(DEV), (torch.randn(C, generator=g) * 0.1).to(DEV)
    noise = (torch.randn(2 * HW, 2 * HW, generator=g) * 0.1).to(DEV)
    s0, s1 = (torch.rand(N, C, generator=g) + 0.5).to(DEV), (torch.rand(N, C, generator=g) + 0.5).to(DEV)
    f32 = Guarded((N, 2 * HW, 2 * HW, C))
    h16 = Guarded((N, 2 * HW, 2 * HW, C), dtype=torch.float16)
    hi, lo = Guarded((N, 2 * HW, 2 * HW, C), dtype=torch.bfloat16), Guarded((N, 2 * HW, 2 * HW, C), dtype=torch.bfloat16)
    outs = [K.make_split_out(h16.view, None, s0, C, 0, f16=True), K.make_split_out(hi.view, lo.view, s1, C, 0)]
    K.fir_up_epilogue(raw, C, dcoef, bias, noise, 2 ** 0.5, 0.2, 1.5, outs=outs, out_f32=f32.view, f32_cstride=C)
    torch.cuda.synchronize()
    for t in (f32, h16, hi, lo):
        assert t.untouched_ok() and t.written()
    assert torch.equal(h16.view, (f32.view * s0[:, None, None, :]).half())
    split = hi.view.float() + lo.view.float()
    assert ((split - f32.view * s1[:, None, None, :]).abs().max() / (f32.view * s1[:, None, None, :]).abs().max()).item() < 2e-5


@pytest.mark.gpu
def test_modulate_f16():
    from next3d_b200 import kernels as K
    g = torch.Generator().manual_seed(7)
    x = torch.randn(2, 16, 16, 32, generator=g).to(DEV)
    s = (torch.rand(2, 32, generator=g) + 0.5).to(DEV)
    out = Guarded((2, 16, 16, 32), dtype=torch.float16)
    K.modulate_f16(x, s, out.view)
    torch.cuda.synchronize()
    assert out.untouched_ok() and out.written()
    assert torch.equal(out.view, (x * s[:, None, None, :]).half())


@pytest.mark.gpu
@pytest.mark.parametrize('C', [32, 12])        # the wide (warp per pixel) and the scalar kernel
def test_resize_aa_f16(C):
    """n3d_resize_aa_f16 = fp16(n3d_resize_aa's fp32 result * style), bit for bit (the 64^2 -> 128^2 SR input)."""
    from next3d_b200 import kernels as K
    g = torch.Generator().manual_seed(C)
    src = torch.randn(2, 64, 64, C, generator=g).to(DEV)
    s = (torch.rand(2, C, generator=g) + 0.5).to(DEV)
    f32 = torch.empty(2, 128, 128, C, device=DEV)
    K.resize_aa(src, f32)
    out = Guarded((2, 128, 128, C), dtype=torch.float16)
    K.resize_aa_f16(src, out.view, style=s)
    torch.cuda.synchronize()
    assert out.untouched_ok() and out.written()
    assert torch.equal(out.view, (f32 * s[:, None, None, :]).half())


# The planned glue table.  fir_up: (N, H2, W2, C) output size, fp16 outputs (cstride, coff), an fp32 output or not, noise;
# modulate: (N, H, W, C), one fp16 output (cstride, coff), style or NULL; resize: (N, SH, SW, C) -> (DH, DW), boxes, style or NULL.
# values 'outedge': styles past 65504 and into the fp16 subnormal range.
def _glue(name, kind, N, H, W, Cc, **kw):
    g = dict(name=name, kind=kind, N=N, H=H, W=W, C=Cc, outs=[(Cc, 0)], f32=True, noise='shared', style=True, values='normal',
             DH=None, DW=None, boxes=False)
    g.update(kw)
    return g


GLUE = [
    # fir-up: the engine's SR selections (8XDC N 1 / 2: TR 32 / 64 at 256 channels, TR 64 / 128 at 128; 4X N 1: S 4), plus S 8 and 16
    _glue('up16_stream_tr32_c256', 'fir_up', 1, 256, 256, 256, outs=[(256, 0), (512, 256)]),
    _glue('up16_stream_tr64_c128', 'fir_up', 1, 512, 512, 128, noise='sample'),
    _glue('up16_stream_tr128_c128', 'fir_up', 2, 512, 512, 128, outs=[(128, 0), (128, 0)]),
    _glue('up16_tiled_s4_c64', 'fir_up', 1, 256, 256, 64, outs=[(64, 0), (128, 64)]),
    _glue('up16_tiled_s8', 'fir_up', 2, 256, 264, 128),
    _glue('up16_tiled_s16', 'fir_up', 4, 256, 264, 128, noise='sample'),
    _glue('up16_no_f32', 'fir_up', 2, 18, 10, 12, outs=[(12, 0), (24, 12)], f32=False, noise='sample'),
    _glue('up16_outedge', 'fir_up', 2, 16, 24, 32, outs=[(32, 0), (64, 32)], values='outedge'),
    _glue('splitk16_outedge', 'splitk', 2, 8, 12, 32, outs=[(32, 0), (64, 32)], values='outedge'),
    # modulate: C 4, 12, 32, a concat output, NULL style, several grid-stride passes
    _glue('mod16_c4', 'modulate', 2, 5, 7, 4),
    _glue('mod16_c12_concat', 'modulate', 2, 6, 5, 12, outs=[(20, 4)]),
    _glue('mod16_c32_nostyle', 'modulate', 3, 4, 6, 32, style=False),
    _glue('mod16_c32_concat_grid', 'modulate', 4, 128, 128, 64, outs=[(96, 32)]),
    _glue('mod16_outedge', 'modulate', 2, 8, 8, 12, values='outedge'),
    # resize: the wide kernel at every C / 4, its strong-minification branch, the scalar kernel at C 3 and 12, boxes, NULL style
    *[_glue(f'resize16_wide_c{4 * q}', 'resize', 1, 64, 64, 4 * q, DH=128, DW=128) for q in (1, 2, 4, 8, 16, 32)],
    _glue('resize16_minify_c32', 'resize', 1, 256, 256, 32, DH=24, DW=24),
    _glue('resize16_minify_c8_boxes', 'resize', 2, 256, 256, 8, DH=40, DW=40, boxes=True),
    _glue('resize16_scalar_c3', 'resize', 2, 64, 64, 3, DH=128, DW=128, style=False),
    _glue('resize16_scalar_c12_boxes', 'resize', 2, 40, 48, 12, DH=64, DW=56, boxes=True),
    _glue('resize16_wide_c32_boxes_nostyle', 'resize', 2, 48, 40, 32, DH=72, DW=64, boxes=True, style=False),
    _glue('resize16_outedge', 'resize', 1, 32, 32, 12, DH=48, DW=48, values='outedge'),
]
GLUE_IDS = [g['name'] for g in GLUE]


def glue_plan(g, sms=SMS):
    """Kernel and grid of a glue launch."""
    N, H, W, Cc = g['N'], g['H'], g['W'], g['C']
    if g['kind'] == 'fir_up':
        return fir_up_plan(N, H, W, Cc, sms)
    if g['kind'] == 'splitk':
        return dict(kernel='splitk_epilogue_kernel', grid=grid_stride(N * H * W * Cc // 4, sms, 16))
    if g['kind'] == 'modulate':
        work = N * H * W * Cc // 4
        return dict(kernel='modulate_split_kernel', work=work, grid=grid_stride(work, sms, 16))
    wide = Cc % 4 == 0 and Cc <= 128 and 32 % (Cc // 4) == 0
    DH, DW = g['DH'], g['DW']
    ntaps = (math.ceil(H / DH) * 2 + 1) * (math.ceil(W / DW) * 2 + 1)          # at least the taps of the window, up to rounding
    return dict(kernel='resize_aa_kernel' if wide else 'resize_aa_scalar_kernel', wide=wide, minify=wide and Cc <= 32 and ntaps >= 64,
                grid=grid_stride(N * DH * DW * (8 if wide else Cc), sms, 16))


GLUE_COVERAGE = {
    'fir-up streamed at TR 32, 64, 128': lambda gs: {p['TR'] for g, p in gs if p.get('streamed')} == {32, 64, 128},
    'fir-up register-tiled at S 4, 8, 16': lambda gs: {p['S'] for g, p in gs if g['kind'] == 'fir_up' and not p['streamed']} >= {4, 8, 16},
    "fir-up at the engine's SR selections": lambda gs: {(p['kernel'], p.get('TR'), p.get('S')) for m in ('8XDC', '4X') for n in (1, 2, 4, 8)
                                                       for what, _, p in engine_sr_launches(m, n) if what == 'fir_up'}
        <= {(p['kernel'], p.get('TR'), p.get('S')) for g, p in gs if g['kind'] == 'fir_up'},
    'fir-up: a concat output, two fp16 outputs, no fp32 output':
        lambda gs: any(len(g['outs']) == 2 and g['outs'][1][1] == g['C'] for g, p in gs if g['kind'] == 'fir_up')
        and any(not g['f32'] for g, p in gs if g['kind'] == 'fir_up'),
    'modulate at C 4, 12, 32, a concat output, NULL style, several grid-stride passes':
        lambda gs: {4, 12, 32} <= {g['C'] for g, p in gs if g['kind'] == 'modulate'}
        and any(g['outs'][0][1] > 0 for g, p in gs if g['kind'] == 'modulate') and any(not g['style'] for g, p in gs if g['kind'] == 'modulate')
        and any(p['work'] > 256 * p['grid'] for g, p in gs if g['kind'] == 'modulate'),
    'resize: the wide kernel at every C / 4': lambda gs: {1, 2, 4, 8, 16, 32} <= {g['C'] // 4 for g, p in gs if p.get('wide')},
    'resize: strong minification': lambda gs: any(p.get('minify') for g, p in gs),
    'resize: the scalar kernel at C 3 and 12': lambda gs: {3, 12} <= {g['C'] for g, p in gs if g['kind'] == 'resize' and not p['wide']},
    'resize: boxes on both kernels, NULL style': lambda gs: {p['wide'] for g, p in gs if g['kind'] == 'resize' and g['boxes']} == {False, True}
        and any(not g['style'] for g, p in gs if g['kind'] == 'resize'),
    'output edges through fir-up, split-K, modulate and resize': lambda gs: {g['kind'] for g, p in gs if g['values'] == 'outedge'}
        == {'fir_up', 'splitk', 'modulate', 'resize'},
}


def test_glue_table_covers_every_launch_configuration():
    """CPU: the glue table reaches everything listed in GLUE_COVERAGE."""
    planned = [(g, glue_plan(g)) for g in GLUE]
    missing = [k for k, ok in GLUE_COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(GLUE_IDS)) == len(GLUE_IDS)


def _glue_styles(g, gen, n):
    N, Cc = g['N'], g['C']
    if g['values'] == 'outedge':
        edge = torch.tensor([7e4, -7e4, 4e4, -3.3e4, 1e5, 3.3e4, 1e-5, -3e-6, 6e-8, -1e-9, 1.0, -2e4], device=DEV)
        idx = torch.arange(N * Cc, device=DEV).reshape(N, Cc)
        return [edge[(idx + k) % len(edge)] for k in range(n)]
    return [torch.rand(N, Cc, device=DEV, generator=gen) + 0.5 for _ in range(n)]


def _boxes(g, N, SH, SW, DH, DW):
    """Source and destination windows per image (y0, y1, x0, x1): the destination one inside the image, so pixels outside it keep
    the sentinel."""
    src = torch.tensor([[2 + n, SH - 3 * n, 1 + 2 * n, SW - n] for n in range(N)], dtype=torch.int32, device=DEV)
    dst = torch.tensor([[3 + n, DH - 2 - n, 2 * n, DW - 5 + n] for n in range(N)], dtype=torch.int32, device=DEV)
    return src, dst


def setup_glue(g):
    gen = torch.Generator(device=DEV).manual_seed(4000 + GLUE_IDS.index(g['name']))
    N, H, W, Cc = g['N'], g['H'], g['W'], g['C']
    s = dict(g=g)
    if g['kind'] in ('fir_up', 'splitk'):
        s['x'] = (torch.randn(N, H + 1, W + 1, Cc, device=DEV, generator=gen) if g['kind'] == 'fir_up'
                  else torch.randn(3, N, H, W, Cc, device=DEV, generator=gen) / math.sqrt(3))
        s['dcoef'] = torch.rand(N, Cc, device=DEV, generator=gen) + 0.5
        s['bias'] = torch.randn(Cc, device=DEV, generator=gen) * 0.5
        s['noise'] = (torch.randn(N, H, W, device=DEV, generator=gen) if g['noise'] == 'sample' else torch.randn(H, W, device=DEV, generator=gen)) * 0.3
        s['noise_nstride'] = H * W if g['noise'] == 'sample' else 0
        s['styles'] = _glue_styles(g, gen, len(g['outs']))
        s['outs'] = [Guarded((N, H, W, cs), torch.float16, slice(co, co + Cc)) for cs, co in g['outs']]
        s['f32'] = Guarded((N, H, W, Cc)) if g['f32'] else None
    elif g['kind'] == 'modulate':
        s['x'] = torch.randn(N, H, W, Cc, device=DEV, generator=gen)
        s['styles'] = _glue_styles(g, gen, 1) if g['style'] else [None]
        (cs, co), = g['outs']
        s['outs'] = [Guarded((N, H, W, cs), torch.float16, slice(co, co + Cc))]
        s['f32'] = None
    else:
        DH, DW = g['DH'], g['DW']
        s['x'] = torch.randn(N, H, W, Cc, device=DEV, generator=gen)
        s['styles'] = _glue_styles(g, gen, 1) if g['style'] else [None]
        s['boxes'] = _boxes(g, N, H, W, DH, DW) if g['boxes'] else (None, None)
        own = torch.ones(N, DH, DW, 1, dtype=torch.bool, device=DEV)
        if g['boxes']:
            own[:] = False
            for n, (y0, y1, x0, x1) in enumerate(s['boxes'][1].tolist()):
                own[n, y0:y1, x0:x1] = True
        s['outs'] = [Guarded((N, DH, DW, Cc), torch.float16, own)]
        s['f32'] = None
    return s


def launch_glue(s):
    from next3d_b200 import kernels as K
    g = s['g']
    if g['kind'] in ('fir_up', 'splitk'):
        outs = [K.make_split_out(t.view, None, sty, cs, co, f16=True) for t, sty, (cs, co) in zip(s['outs'], s['styles'], g['outs'])]
        kw = dict(outs=outs, out_f32=s['f32'].view if s['f32'] else None, f32_cstride=g['C'] if s['f32'] else 0, noise_nstride=s['noise_nstride'])
        if g['kind'] == 'fir_up':
            K.fir_up_epilogue(s['x'], g['C'], s['dcoef'], s['bias'], s['noise'], math.sqrt(2), 0.2, 2.0, **kw)
        else:
            K.splitk_epilogue(s['x'], s['dcoef'], s['bias'], s['noise'], math.sqrt(2), 0.2, 2.0, **kw)
    elif g['kind'] == 'modulate':
        (cs, co), = g['outs']
        K.modulate_f16(s['x'], s['styles'][0], s['outs'][0].view, cs, co)
    else:
        K.resize_aa_f16(s['x'], s['outs'][0].view, *s['boxes'], style=s['styles'][0])


def _fir_up_reference(s):
    """fp64 FIR-up (upfirdn2d, gain 4) and the mode-0 epilogue of the whole (small) launch -> [N, H2, W2, C]."""
    from oracle import ops as oo
    g = s['g']
    f64 = oo.setup_filter().to(DEV, torch.float64)
    acc = oo.upfirdn2d(s['x'].permute(0, 3, 1, 2).double(), f64, padding=1, gain=4).permute(0, 2, 3, 1)
    noise = s['noise'].double() if g['noise'] == 'sample' else s['noise'].double()[None]
    v = acc * s['dcoef'].double()[:, None, None, :] + noise[..., None] + s['bias'].double()
    return (torch.where(v > 0, v, 0.2 * v) * math.sqrt(2)).clamp(-2.0, 2.0)


def check_glue(s):
    """-> {output: range-relative error against fp64}; asserts the sentinel, written-element and fp16 bit-identity checks."""
    from next3d_b200 import kernels as K
    g = s['g']
    Cc = g['C']
    errs = {}
    for k, t in enumerate(s['outs'] + ([s['f32']] if s['f32'] is not None else [])):
        assert t.untouched_ok(), (g['name'], k, 'an element outside the output was written')
        assert t.written(), (g['name'], k, 'an owned element was not written')
    if g['kind'] == 'resize':                   # n3d_resize_aa's fp32 result: the fp16 one's reference
        base = Guarded(s['outs'][0].view.shape, torch.float32, s['outs'][0].own)
        K.resize_aa(s['x'], base.view, src_box=s['boxes'][0], dst_box=s['boxes'][1])
        torch.cuda.synchronize()
        f32 = base.view
    elif g['kind'] == 'modulate':
        f32 = s['x']
    else:
        f32 = s['f32'].view if s['f32'] is not None else None
    if g['kind'] == 'fir_up' and f32 is None:
        ref = _fir_up_reference(s)
    for k, (t, sty) in enumerate(zip(s['outs'], s['styles'])):
        co = g['outs'][k][1] if g['kind'] != 'resize' else 0
        got = t.view[..., co:co + Cc]
        scale = sty[:, None, None, :] if sty is not None else 1.0
        if f32 is not None:
            want = (f32 * scale).half()
            own = t.own.expand_as(got) if isinstance(t.own, torch.Tensor) else torch.ones_like(got, dtype=torch.bool)
            diff = (got.view(torch.int16) != want.view(torch.int16)) & own
            assert not bool(diff.any()), (g['name'], k, 'not fp16(fp32 result * style)', int(diff.sum()))
        else:
            want64 = ref * (sty.double()[:, None, None, :] if sty is not None else 1.0)
            errs[f'out{k}'] = ((got.double() - want64).abs().max() / want64.abs().max()).item()
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('g', GLUE, ids=GLUE_IDS)
def test_glue_f16_outputs(g, monkeypatch):
    """Each glue launch: its fp16 outputs are fp16(fp32 result * style) bit for bit (fir-up and split-K: their own fp32 output;
    modulate: x; resize: n3d_resize_aa's fp32 result), or within glue.f16 of fp64 where there is no fp32 output; pixels outside the
    paste window keep the sentinel; a rerun, and for the streamed FIR-up a rerun under N3D_FIR_STREAM=0, is bit-identical."""
    monkeypatch.delenv('N3D_FIR_STREAM', raising=False)
    s = setup_glue(g)
    launch_glue(s)
    torch.cuda.synchronize()
    errs = check_glue(s)
    record_errors('N3D_CONV16_ERRORS', [{'case': g['name'], 'output': k, 'kind': 'glue.f16', 'err': e, 'bound': BOUNDS['glue.f16']}
                                        for k, e in errs.items()])
    bad = {k: e for k, e in errs.items() if not e < BOUNDS['glue.f16']}
    assert not bad, bad
    outs = s['outs'] + ([s['f32']] if s['f32'] is not None else [])
    rerun = lambda: rerun_identical(outs, lambda: launch_glue(s))         # noqa: E731
    assert rerun(), f'{g["name"]}: a rerun is not bit-identical'
    if glue_plan(g, torch.cuda.get_device_properties(0).multi_processor_count).get('streamed'):
        monkeypatch.setenv('N3D_FIR_STREAM', '0')
        assert rerun(), f'{g["name"]}: the register-tiled kernel is not bit-identical to the streamed one'


@pytest.mark.gpu
def test_launched_glue_kernel_matches_plan(tmp_path, monkeypatch):
    """Every glue case under torch.profiler: the kernel it launched and its grid are the ones glue_plan predicts."""
    monkeypatch.delenv('N3D_FIR_STREAM', raising=False)
    pattern = re.compile(r'fir_up_stream_kernel|fir_up_epilogue_kernel|splitk_epilogue_kernel|modulate_split_kernel|resize_aa_kernel|'
                         r'resize_aa_scalar_kernel')

    def run():
        for g in GLUE:
            s = setup_glue(g)
            launch_glue(s)
            torch.cuda.synchronize()
            del s
        return GLUE                         # one launch per case

    _, events = launched_kernels(run, pattern, tmp_path)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for g, e in zip(GLUE, events):
        p = glue_plan(g, sms)
        assert pattern.search(e['name']).group(0) == p['kernel'], (g['name'], e['name'], p)
        grid = e.get('args', {}).get('grid')
        if grid is not None:
            assert list(grid) == [p['grid'], 1, 1], (g['name'], grid, p)


# ------------------------------------------------------------------------------------------------ argument checks (CPU, nothing launched)
def _desc16(nprod=1):
    L = lib()
    a = torch.zeros(1, 8, 16, 64, dtype=torch.float16)
    w = torch.zeros(1, 16, 64, dtype=torch.float16)
    p = L.ConvGemm()
    p.a_hi, p.w_hi = a.data_ptr(), w.data_ptr()
    p.NI, p.AH, p.AW, p.Cin = a.shape
    p.T, p.Cout = 1, 16
    p.N, p.MH, p.MW = 1, 8, 16
    p.ntaps = 1
    p.taps[0] = L.ConvTap(0, 0, 0, 0)
    p.nprod, p.f16 = nprod, 1
    p.gain, p.slope, p.clamp = 1.0, 1.0, -1.0
    p.oy_mul, p.ox_mul, p.OH, p.OW = 1, 1, 8, 16
    return p, (a, w)


def test_conv_gemm_f16_refuses_nprod3():
    p, keep = _desc16(nprod=3)
    refused(lib().lib.n3d_conv_gemm(C.byref(p), None), 'fp16 operands take nprod 1')


@pytest.mark.parametrize('operand_f16,out_f16', [(1, 0), (0, 1)])
def test_conv_gemm_refuses_mixed_output_form(operand_f16, out_f16):
    L = lib()
    p, keep = _desc16()
    p.f16 = operand_f16
    o = torch.zeros(1, 8, 16, 16, dtype=torch.float16)
    p.out[0] = L.SplitOut(o.data_ptr(), o.data_ptr(), None, 16, 0, out_f16)
    refused(L.lib.n3d_conv_gemm(C.byref(p), None), 'n3d_conv_gemm: output 0 must be')


def test_fir_up_epilogue_refuses_bad_output_form():
    L = lib()
    raw = torch.zeros(1, 5, 5, 4)
    o = torch.zeros(1, 4, 4, 4, dtype=torch.float16)
    arr = (L.SplitOut * 2)()
    arr[0] = L.SplitOut(o.data_ptr(), None, None, 4, 0, 2)
    refused(L.lib.n3d_fir_up_epilogue(raw.data_ptr(), 1, 4, 4, 4, None, None, None, 0, 1.0, 1.0, -1.0, arr, None, 0, 0, None),
            'f16 must be 0')
