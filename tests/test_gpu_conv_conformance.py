"""conv_gemm against the N3DConvGemm contract (include/next3d_b200.h), in fp64, over a table of small launches that reaches every
kernel instance, work schedule and epilogue path `launch_conv` (next3d_b200/csrc/conv_gemm.cu) can select.

The reference multiplies exactly the operands the kernel gets: hi*hi + hi*lo + lo*hi for nprod 3 and hi*hi for nprod 1, as fp64
products (a bf16 x bf16 product is exact in fp64).  What is left between kernel and reference is the fp32 accumulation order and the
fp32 epilogue, so the bounds below are far tighter than the ~2^-16 of the split scheme itself.

Every output is a view into a larger allocation filled with a NaN sentinel: the elements a launch owns must be written (and match),
every other element -- guard bands, the other half of a concat buffer, channels outside [coff, coff + Cout), pixels another parity
class owns -- must keep the sentinel's bits.

`plan` mirrors the launch rule of `launch_conv` in plain Python.  The CPU test checks that the table covers every configuration
listed in COVERAGE; the profiler test checks on the GPU that each case ran the kernel instance (and grid) `plan` predicts.

The alignment tests at the end need no GPU: descriptors over CPU tensors at 4-byte offsets must be refused before any device call.
"""
import ctypes as C
import math
import re

import pytest
import torch

from tests.helpers import Guarded, launched_kernels, lib, offset_view, refused

DEV = 'cuda'

# Range-relative error bounds per output kind, max |got - ref| / max |ref| over the owned elements, each at most 4x the worst case
# measured over the table on an H100 SXM 80 GB (700 W power limit), which is given beside it.
BOUNDS = {
    'raw': 4e-6,        # mode 1 / split-K partial sums.  Worst: 9.9e-7 (splitk3, 3 x 9 x 80 products)
    'f32': 3.5e-5,      # mode-0 fp32 output.  Worst: 9.7e-6 (bn32_bk32_cin160: fp32 accumulation of 3 x 9 x 160 products; the clamp at 2
                        # keeps the output range at 2 while the accumulator reaches ~5, so the same absolute error is larger relative)
    'split': 2.5e-5,    # hi + lo of a split bf16 output (the split itself rounds at 2^-18 of the value).  Worst: 7.5e-6 (rgb32.out0)
    'rgb': 9e-6,        # fused ToRGB image.  Worst: 2.5e-6 (rgb192_cluster)
}

# ------------------------------------------------------------------------------------------------ the launch rule, mirrored
# Constants of conv_gemm.cu: kBlockM, kMinTiles, kMinTilesSplit, kMinStages, kMaxBlockN, kStageArrays, kXStride, kStoreBoxBytes,
# and from them the epilogue area of a warpgroup (kEpiBytes) and the stage-ring bytes (kRingBytes).  test_mirror_constants_match_source
# reads them from the source.
BLOCK_M, MIN_TILES, MIN_TILES_SPLIT, MIN_STAGES, MAX_BLOCK_N = 128, 64, 128, 4, 128
STAGE_ARRAYS, X_STRIDE, STORE_BOX_BYTES = 8, 36, 64 * 32 * 4
EPI_BYTES = max(STAGE_ARRAYS * MAX_BLOCK_N * 4 + 64 * X_STRIDE * 4 + 64 * 4 * 4, 2 * STORE_BOX_BYTES)
RING_BYTES = 227 * 1024 - 2 * EPI_BYTES - 1024 - 256
BLOCK_NS = (16, 32, 64, 96, 128)


def _pow2_ceil(v):
    p = 1
    while p < v:
        p <<= 1
    return p


def tile_geometry(N, MH, MW):
    """(TW, TH, TN, M tiles) of one sub-problem: TW up to 16 wide, then TH, then TN images (TW * TH * TN == kBlockM)."""
    TW = min(16, _pow2_ceil(MW))
    TH = min(BLOCK_M // TW, _pow2_ceil(MH))
    TN = BLOCK_M // (TW * TH)
    return TW, TH, TN, -(-MW // TW) * -(-MH // TH) * -(-N // TN)


def widest_block_n(Cout, tiles_m, splits=1):
    """The widest wgmma N not above Cout (96 only where it divides Cout rounded to 16), halved while the launch has fewer than
    kMinTiles (kMinTilesSplit under split-K) tiles."""
    cout16 = -(-Cout // 16) * 16
    bn = next(c for c in (128, 96, 64, 32, 16) if c <= cout16 and (c != 96 or cout16 % 96 == 0))
    min_tiles = MIN_TILES_SPLIT if splits > 1 else MIN_TILES
    while bn > 32 and tiles_m * splits * -(-Cout // bn) < min_tiles:
        bn = 32 if bn == 96 else bn // 2
    return bn


def block_k_for(Cin, bn, f16=False):
    """block_k rule of launch_conv: 32-channel stages for Cin % 64 == 32 or where 64-channel stages leave < kMinStages in the ring.
    A bf16 stage holds the hi and lo tiles of A and B, an fp16 stage (f16) one of each."""
    tiles_per_stage = 1 if f16 else 2
    return 32 if Cin % 64 == 32 or RING_BYTES // (tiles_per_stage * (BLOCK_M + bn) * 64 * 2) < MIN_STAGES else 64


def stages_for(bn, bk, f16=False):
    """Stages of the ring (kMaxStages 8 at most)."""
    return min(8, RING_BYTES // ((1 if f16 else 2) * (BLOCK_M + bn) * bk * 2))


def plan(N, Cin, Cout, MH, MW, splits=1, rgb=False, sms=132, cluster_slots=66, f16=False):
    """What launch_conv (conv_gemm.cu) selects for a one-sub-problem n3d_conv_gemm launch: tile geometry, block_n (widest wgmma N
    not above Cout, halved while the launch has fewer than kMinTiles tiles; the fused ToRGB takes the narrowest width holding all
    channels, else 128-wide n-tiles in turn), block_k, 2-CTA clusters (block_n >= 96, no split-K, >= 2 M tiles), work items and the
    grid.  sms / cluster_slots: SMs and cudaOccupancyMaxActiveClusters of the device (132 and 66 on the H100 SXM).  f16: fp16
    operands (N3DConvGemm.f16)."""
    TW, TH, TN, tiles_m = tile_geometry(N, MH, MW)
    bn = widest_block_n(Cout, tiles_m, splits)
    item_tiles = 1
    if rgb:
        cout16 = -(-Cout // 16) * 16
        bn = next((w for w in BLOCK_NS if w >= cout16), MAX_BLOCK_N)
        item_tiles = -(-Cout // bn)
    tiles_n = -(-Cout // bn)
    cluster = 2 if splits == 1 and bn >= 96 and tiles_m >= 2 else 1
    units = -(-tiles_m // cluster) * tiles_n * splits // item_tiles
    slots = sms if cluster == 1 else cluster_slots
    bk = block_k_for(Cin, bn, f16)
    return dict(block_n=bn, block_k=bk, stages=stages_for(bn, bk, f16), cluster=cluster, TW=TW, TH=TH, TN=TN, tiles_m=tiles_m,
                tiles_n=tiles_n, item_tiles=item_tiles, units=units, grid=cluster * min(units, slots), items_per_cta=-(-units // slots),
                pad=cluster == 2 and tiles_m % 2 == 1, grouped=False)


def transposed_plan(N, Cin, Cout, H, W, sms=132, cluster_slots=66, f16=False):
    """What n3d_conv_transposed_gemm selects for a stride-2 transposed 3x3 conv of an H x W input: nine sub-problems (the four
    parity-class interiors H x W, two row strips 1 x W, two column strips H x 1, the corner 1 x 1), block_n from the sum of their M
    tiles, a 2-CTA cluster where block_n >= 96 and the largest sub-problem has >= 2 M tiles, the four interleaved classes grouped into
    one unit per (M tile, n-tile) when they have more items than the launch has CTA (cluster) slots, and the grid."""
    sub_m = [tile_geometry(N, mh, mw)[3] for mh, mw in [(H, W)] * 4 + [(1, W)] * 2 + [(H, 1)] * 2 + [(1, 1)]]
    tiles_m = sum(sub_m)
    bn = widest_block_n(Cout, tiles_m)
    tiles_n = -(-Cout // bn)
    cluster = 2 if bn >= 96 and max(sub_m) >= 2 else 1
    slots = sms if cluster == 1 else cluster_slots
    units_grouped = -(-sub_m[0] // cluster) * tiles_n
    groups = units_grouped if 4 * units_grouped > slots else 0
    total_items = 4 * units_grouped + sum(-(-m // cluster) * tiles_n for m in sub_m[4:])
    units = total_items - 3 * groups
    bk = block_k_for(Cin, bn, f16)
    return dict(block_n=bn, block_k=bk, stages=stages_for(bn, bk, f16), cluster=cluster, tiles_m=tiles_m, tiles_n=tiles_n, item_tiles=1,
                units=units, grid=cluster * min(units, slots), items_per_cta=-(-units // slots), pad=cluster == 2 and any(m % 2 for m in sub_m),
                grouped=groups > 0)


def reachable_instances(f16=False):
    """(block_n, block_k) pairs the rule can produce: every block_n with a Cin that is / is not 32 mod 64 (8 for bf16 operands, all
    10 for fp16, whose stages are half the size)."""
    return {(bn, block_k_for(cin, bn, f16)) for bn in BLOCK_NS for cin in (32, 64)}


def source_constants():
    """The integer constants of conv_gemm.cu (`constexpr int k... = <expr>;`), each evaluated in terms of the ones before it."""
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'next3d_b200', 'csrc', 'conv_gemm.cu')).read()
    env = {}
    for name, expr in re.findall(r'^constexpr int (k\w+) = ([^;]+);', src, re.M):
        cond = re.fullmatch(r'(.+?) ([<>]=?) (.+?) \? (.+?) : (.+)', expr.strip())
        if cond:                            # c ? a : b
            expr = f'(({cond[4]}) if ({cond[1]}) {cond[2]} ({cond[3]}) else ({cond[5]}))'
        env[name] = int(eval(expr, {'__builtins__': {}}, dict(env)))
    return env


# ------------------------------------------------------------------------------------------------ the case table
def _case(name, N, Cin, Cout, MH, MW, **kw):
    c = dict(name=name, N=N, Cin=Cin, Cout=Cout, MH=MH, MW=MW, taps='3x3', nprod=3, mode=0, splits=1, epi='full', noise='shared',
             outs=None, f32=None, rgb=None, epi_noise='sample')     # epi_noise: noise of the split-K epilogue pass
    c.update(kw)
    if c['mode'] == 1:
        c['epi'], c['noise'] = 'none', None
    if c['outs'] is None:           # default: a split output of its own and one into the second half of a concat buffer
        c['outs'] = [] if c['mode'] == 1 or c['rgb'] else [dict(cstride=Cout, coff=0), dict(cstride=2 * Cout, coff=Cout)]
    if c['f32'] is None and not c['rgb']:
        c['f32'] = dict(cstride=Cout, coff=0, nchw=False, acc=False)
    c['f32'] = c['f32'] or None
    return c


TORGB = dict(epi='torgb', noise=None, outs=[], taps='1x1')     # ToRGBLayer as the engine issues it: linear, bias, clamp, NCHW +=
CASES = [
    # every reachable (block_n, block_k) instance in mode 0 with the full epilogue
    _case('bn16_bk64_nprod1', 2, 64, 16, 16, 16, nprod=1, noise='sample'),
    _case('bn16_bk32_24x3', 3, 96, 16, 24, 3, outs=[dict(cstride=20, coff=4)]),
    _case('bn32_bk64_5x37_cout40', 2, 64, 40, 5, 37, f32=dict(cstride=40, coff=0, nchw=True, acc=False)),
    _case('bn32_bk32_cin160', 2, 160, 32, 16, 8, f32=dict(cstride=41, coff=1, nchw=False, acc=False)),
    _case('bn64_bk64_cout72', 17, 48, 72, 16, 16, f32=dict(cstride=80, coff=4, nchw=False, acc=False)),
    _case('bn64_bk32_cin32', 64, 32, 64, 8, 16, outs=[dict(cstride=80, coff=8)]),
    _case('bn96_bk32_rgb_unclustered', 1, 40, 96, 8, 16, rgb=dict(ch=3, nchw=True, acc=True), outs=[dict(cstride=96, coff=0)]),
    _case('bn128_bk32_rgb_unclustered', 1, 8, 128, 8, 16, rgb=dict(ch=1, nchw=False, acc=False), outs=[dict(cstride=128, coff=0)],
          f32=dict(cstride=128, coff=0, nchw=False, acc=False)),
    # clusters: pad tiles, f32 accumulate (which takes no split outputs), stride 2, TN 2, several items per cluster
    _case('bn128_cluster_pad_accumulate', 33, 24, 200, 8, 16, f32=dict(cstride=200, coff=0, nchw=False, acc=True), outs=[], noise='sample'),
    _case('bn128_cluster_stride2_pad', 5, 8, 128, 40, 40, taps='s2', noise='sample'),
    _case('bn128_cluster_tn2_pad', 129, 40, 128, 8, 8, noise='sample'),
    _case('bn96_cluster_torgb1x1_accumulate', 8, 80, 96, 32, 32, **TORGB, f32=dict(cstride=96, coff=0, nchw=False, acc=True)),
    _case('bn128_cluster_pingpong', 299, 8, 128, 8, 16, nprod=1),
    # unclustered ping-pong (several items per CTA, block_n <= 64), TN > 1 with the full epilogue
    _case('bn32_pingpong_staged', 135, 16, 48, 8, 16, noise='sample'),
    _case('bn32_tn8_unstaged', 9, 48, 32, 4, 4, noise='sample'),
    # 1x1 ToRGB launches at 4^2 and 8^2 (TN 8 and 2, N not a multiple of TN, NCHW accumulate)
    _case('torgb1x1_4x4', 9, 64, 3, 4, 4, **TORGB, f32=dict(cstride=3, coff=0, nchw=True, acc=True)),
    _case('torgb1x1_8x8', 5, 32, 3, 8, 8, **TORGB, f32=dict(cstride=3, coff=0, nchw=True, acc=True), nprod=1),
    # fused ToRGB: every width class, 1 / 3 / 4 channels, NHWC / NCHW, with and without accumulate
    _case('rgb16', 2, 24, 16, 16, 16, rgb=dict(ch=1, nchw=False, acc=False)),
    _case('rgb32', 2, 40, 32, 16, 8, rgb=dict(ch=3, nchw=True, acc=True), outs=[dict(cstride=32, coff=0)]),
    _case('rgb40', 2, 80, 40, 16, 16, rgb=dict(ch=4, nchw=False, acc=True), outs=[dict(cstride=48, coff=8)]),
    _case('rgb96_cluster_pad', 3, 48, 96, 8, 16, rgb=dict(ch=3, nchw=True, acc=False)),
    _case('rgb192_cluster', 2, 64, 192, 16, 16, rgb=dict(ch=4, nchw=True, acc=False), outs=[dict(cstride=192, coff=0)],
          f32=dict(cstride=192, coff=0, nchw=False, acc=False)),
    _case('rgb256_cluster_pad', 3, 32, 256, 8, 16, rgb=dict(ch=3, nchw=False, acc=True)),
    # split-K through n3d_splitk_epilogue: 9 slices, 3 slices, 2 uneven slices (5 + 4 of 9 K steps)
    _case('splitk9', 2, 64, 64, 4, 4, mode=1, splits=9, epi_noise='shared'),
    _case('splitk3', 3, 80, 40, 8, 8, mode=1, splits=3),
    _case('splitk2_uneven', 2, 24, 72, 8, 8, mode=1, splits=2),
    # raw output of one transposed-conv parity class: every other output pixel belongs to another class
    _case('transposed_class10_raw', 2, 40, 64, 12, 13, mode=1, taps='tr10', f32=dict(cstride=64, coff=0, nchw=False, acc=False)),
]
CASE_IDS = [c['name'] for c in CASES]
# (block_n, block_k, stages, cluster, grid) `plan` gives each case at 132 SMs: the mirror is shared with the fp16 suite, and a change
# to it must leave these as they are
BF16_PLANS = {
    'bn16_bk64_nprod1': (16, 64, 5, 1, 4), 'bn16_bk32_24x3': (16, 32, 8, 1, 3), 'bn32_bk64_5x37_cout40': (32, 64, 4, 1, 12),
    'bn32_bk32_cin160': (32, 32, 8, 1, 2), 'bn64_bk64_cout72': (64, 64, 4, 1, 68), 'bn64_bk32_cin32': (64, 32, 8, 1, 64),
    'bn96_bk32_rgb_unclustered': (96, 32, 6, 1, 1), 'bn128_bk32_rgb_unclustered': (128, 32, 6, 1, 1),
    'bn128_cluster_pad_accumulate': (128, 32, 6, 2, 68), 'bn128_cluster_stride2_pad': (128, 32, 6, 2, 76),
    'bn128_cluster_tn2_pad': (128, 32, 6, 2, 66), 'bn96_cluster_torgb1x1_accumulate': (96, 32, 6, 2, 64),
    'bn128_cluster_pingpong': (128, 32, 6, 2, 132), 'bn32_pingpong_staged': (32, 64, 4, 1, 132), 'bn32_tn8_unstaged': (32, 64, 4, 1, 2),
    'torgb1x1_4x4': (16, 64, 5, 1, 2), 'torgb1x1_8x8': (16, 32, 8, 1, 3), 'rgb16': (16, 64, 5, 1, 4), 'rgb32': (32, 64, 4, 1, 2),
    'rgb40': (64, 64, 4, 1, 4), 'rgb96_cluster_pad': (96, 32, 6, 2, 4), 'rgb192_cluster': (128, 32, 6, 2, 4),
    'rgb256_cluster_pad': (128, 32, 6, 2, 4), 'splitk9': (32, 64, 4, 1, 18), 'splitk3': (32, 64, 4, 1, 12),
    'splitk2_uneven': (32, 64, 4, 1, 6), 'transposed_class10_raw': (32, 64, 4, 1, 8),
}


def _taps(c):
    from next3d_b200 import kernels as K
    return {'3x3': K.taps_conv3x3, '1x1': K.taps_conv1x1, 's2': K.taps_stride2, 'tr10': lambda: K.taps_transposed(1, 0)}[c['taps']]()


def _geometry(c):
    """(NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW) of a case."""
    N, MH, MW = c['N'], c['MH'], c['MW']
    if c['taps'] == 's2':           # parity sub-images of a 2 MH x 2 MW input padded by the FIR: [4N, MH + 1, MW + 1]
        return 4 * N, MH + 1, MW + 1, N, 1, 0, 1, 0, MH, MW
    if c['taps'] == 'tr10':         # class (1, 0) of a stride-2 transposed conv of an MH x (MW - 1) input
        H, W = MH, MW - 1
        return N, H, W, 0, 2, 1, 2, 0, 2 * H + 1, 2 * W + 1
    return N, MH, MW, 0, 1, 0, 1, 0, MH, MW


def _plan(c):
    return plan(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], c['splits'], bool(c['rgb']))


def _full_epilogue(c):
    return c['mode'] == 0 and c['epi'] == 'full' and c['noise'] is not None and bool(c['outs'])


def _f32_path(c):
    """Store path of the fp32 output (conv_gemm.cu epilogue): 256-bit, float4 or scalar; NCHW has its own."""
    f = c['f32']
    if f is None:
        return None
    if f['nchw']:
        return 'nchw_accumulate' if f['acc'] else 'nchw'
    if f['cstride'] % 8 == 0 and f['coff'] % 8 == 0:
        return 'f32_256'
    return 'f32_float4' if f['cstride'] % 4 == 0 and f['coff'] % 4 == 0 else 'f32_scalar'


def _split_paths(c):
    paths = set()
    for o in c['outs']:
        if o['cstride'] % 16 == 0 and o['coff'] % 16 == 0:
            paths.add('split_256')
        else:
            paths.add('split_uint4' if o['cstride'] % 8 == 0 and o['coff'] % 8 == 0 else 'split_scalar')
    return paths


COVERAGE = {
    'every reachable instance in mode 0 with the full epilogue':
        lambda cs: {(p['block_n'], p['block_k']) for c, p in cs if _full_epilogue(c) or (c['rgb'] and c['outs'])} == reachable_instances(),
    'block_n 96 clustered': lambda cs: any(p['block_n'] == 96 and p['cluster'] == 2 and c['mode'] == 0 for c, p in cs),
    'block_n 96 unclustered': lambda cs: any(p['block_n'] == 96 and p['cluster'] == 1 and c['mode'] == 0 for c, p in cs),
    'block_n 128 clustered': lambda cs: any(p['block_n'] == 128 and p['cluster'] == 2 and c['mode'] == 0 for c, p in cs),
    'block_n 128 unclustered': lambda cs: any(p['block_n'] == 128 and p['cluster'] == 1 and c['mode'] == 0 for c, p in cs),
    'pad tile with f32_accumulate': lambda cs: any(p['pad'] and c['f32'] and c['f32']['acc'] for c, p in cs),
    'pad tile in a stride-2 launch': lambda cs: any(p['pad'] and c['taps'] == 's2' for c, p in cs),
    'TN 1, 2 and 8': lambda cs: {1, 2, 8} <= {p['TN'] for c, p in cs},
    'clustered TN 2': lambda cs: any(p['TN'] == 2 and p['cluster'] == 2 for c, p in cs),
    'N not a multiple of TN': lambda cs: any(p['TN'] > 1 and c['N'] % p['TN'] for c, p in cs),
    'odd count >= 3 of items per CTA, unclustered':
        lambda cs: any(p['cluster'] == 1 and p['block_n'] <= 64 and p['items_per_cta'] >= 3 and p['items_per_cta'] % 2 for c, p in cs),
    'odd count >= 3 of items per cluster': lambda cs: any(p['cluster'] == 2 and p['items_per_cta'] >= 3 and p['items_per_cta'] % 2 for c, p in cs),
    'split-K S 9, 3 and 2': lambda cs: {9, 3, 2} <= {c['splits'] for c, p in cs},
    'split-K with uneven slices': lambda cs: any(c['splits'] > 1 and (9 * -(-c['Cin'] // p['block_k'])) % c['splits'] for c, p in cs),
    'Cout % 16 != 0 on narrow tiles': lambda cs: any(c['Cout'] % 16 and p['block_n'] <= 64 and c['Cout'] > 16 for c, p in cs),
    'Cout % 16 != 0 on wide tiles': lambda cs: any(c['Cout'] % 16 and p['block_n'] >= 96 for c, p in cs),
    'Cin 8, 24, 40, 48, 80, 160': lambda cs: {8, 24, 40, 48, 80, 160} <= {c['Cin'] for c, p in cs},
    'channel tails at both block_k': lambda cs: {p['block_k'] for c, p in cs if c['Cin'] % 16} == {32, 64},
    'MW < 16, MW not a power of two, MH != MW':
        lambda cs: {(5, 37), (24, 3)} <= {(c['MH'], c['MW']) for c, p in cs},
    'fp32 stores: 256-bit, float4, scalar, NCHW, NCHW accumulate':
        lambda cs: {'f32_256', 'f32_float4', 'f32_scalar', 'nchw', 'nchw_accumulate'} <= {_f32_path(c) for c, p in cs},
    'split stores: 256-bit, uint4, scalar': lambda cs: {'split_256', 'split_uint4', 'split_scalar'} <= set().union(*(_split_paths(c) for c, p in cs)),
    'fused ToRGB at Cout 16, 32, 40, 96, 192, 256': lambda cs: {16, 32, 40, 96, 192, 256} <= {c['Cout'] for c, p in cs if c['rgb']},
    'fused ToRGB with 1, 3, 4 channels': lambda cs: {1, 3, 4} <= {c['rgb']['ch'] for c, p in cs if c['rgb']},
    'fused ToRGB NHWC / NCHW x accumulate or not':
        lambda cs: {(a, b) for a in (0, 1) for b in (0, 1)} <= {(int(c['rgb']['nchw']), int(c['rgb']['acc'])) for c, p in cs if c['rgb']},
    'fused ToRGB with a partial second n-tile': lambda cs: any(c['rgb'] and p['item_tiles'] == 2 and c['Cout'] % 128 for c, p in cs),
    '1x1 ToRGB launches at 4x4 and 8x8': lambda cs: {4, 8} <= {c['MH'] for c, p in cs if c['epi'] == 'torgb' and c['f32']['nchw']},
    'nprod 1 on several instances': lambda cs: len({(p['block_n'], p['block_k']) for c, p in cs if c['nprod'] == 1}) >= 3,
    'per-sample noise, staged (TN 1)': lambda cs: any(c['noise'] == 'sample' and p['TN'] == 1 and p['cluster'] == 1 for c, p in cs),
    'per-sample noise, unstaged (TN > 1)': lambda cs: any(c['noise'] == 'sample' and p['TN'] > 1 for c, p in cs),
    'per-sample noise, clustered': lambda cs: any(c['noise'] == 'sample' and p['cluster'] == 2 for c, p in cs),
    'per-sample noise through the split-K epilogue': lambda cs: any(c['splits'] > 1 and c['epi_noise'] == 'sample' for c, p in cs),
}


def test_case_table_covers_every_launch_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rule."""
    planned = [(c, _plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(reachable_instances()) == 8
    assert (96, 64) not in reachable_instances() and (128, 64) not in reachable_instances()
    assert len(set(CASE_IDS)) == len(CASE_IDS)


def test_mirror_constants_match_source():
    """CPU: the mirror's constants are conv_gemm.cu's, and EPI_BYTES / RING_BYTES follow from them as kEpiBytes / kRingBytes do."""
    k = source_constants()
    assert (k['kBlockM'], k['kMinTiles'], k['kMinTilesSplit'], k['kMinStages'], k['kMaxBlockN']) == (BLOCK_M, MIN_TILES, MIN_TILES_SPLIT,
                                                                                                   MIN_STAGES, MAX_BLOCK_N)
    assert (k['kStageArrays'], k['kXStride'], k['kStoreBoxBytes']) == (STAGE_ARRAYS, X_STRIDE, STORE_BOX_BYTES)
    assert k['kMaxStages'] == 8
    assert max(k['kStageArrays'] * k['kMaxBlockN'] * 4 + 64 * k['kXStride'] * 4 + 64 * 4 * 4, 2 * k['kStoreBoxBytes']) == EPI_BYTES
    assert k['kEpiBytes'] == EPI_BYTES and k['kRingBytes'] == RING_BYTES


def test_plan_is_unchanged_for_bf16():
    """CPU: the bf16 selections of the table, pinned (instance, stages, cluster, grid), so that a change of the shared mirror shows."""
    got = {c['name']: (p['block_n'], p['block_k'], p['stages'], p['cluster'], p['grid']) for c in CASES for p in [_plan(c)]}
    assert got == BF16_PLANS, {k: (v, BF16_PLANS.get(k)) for k, v in got.items() if BF16_PLANS.get(k) != v}


# ------------------------------------------------------------------------------------------------ the fp64 reference
def conv_reference(a_hi, a_lo, w_hi, w_lo, taps, N, MH, MW, a_img_mul=0, nprod=3, block_k=None, k_steps=None):
    """acc[n, y, x, o] = sum_taps sum_i A[n + img_off * a_img_mul, y + dy, x + dx, i] * W[wtap, o, i] in fp64, A = 0 outside the
    image, with the kernel's products: hi*hi + hi*lo + lo*hi (nprod 3) or hi*hi (nprod 1).  k_steps = (begin, end): only K steps
    [begin, end) of the tap-major order of (tap, block_k-channel chunk) steps (one split-K slice)."""
    NI, AH, AW, Cin = a_hi.shape
    dev = a_hi.device
    ahi, alo = a_hi.double(), (a_lo.double() if nprod == 3 else None)
    whi, wlo = w_hi.double(), w_lo.double()
    wb = whi + wlo if nprod == 3 else whi              # hi*hi + hi*lo = hi * (hi + lo), exact in fp64
    chunks = -(-Cin // block_k) if block_k else 1
    acc = torch.zeros(N, MH, MW, w_hi.shape[1], dtype=torch.float64, device=dev)
    for step in range(len(taps) * chunks):
        if k_steps is not None and not (k_steps[0] <= step < k_steps[1]):
            continue
        dy, dx, io, wt = taps[step // chunks]
        ch = slice(0, Cin) if chunks == 1 else slice((step % chunks) * block_k, min(Cin, (step % chunks + 1) * block_k))
        ys, xs = torch.arange(MH, device=dev) + dy, torch.arange(MW, device=dev) + dx
        inside = (((ys >= 0) & (ys < AH))[:, None] & ((xs >= 0) & (xs < AW))[None, :]).double()[None, :, :, None]
        img = torch.arange(N, device=dev) + io * a_img_mul
        yc, xc = ys.clamp(0, AH - 1), xs.clamp(0, AW - 1)
        a = ahi[img][:, yc][:, :, xc, ch] * inside
        acc += a @ wb[wt][:, ch].T
        if nprod == 3:
            acc += (alo[img][:, yc][:, :, xc, ch] * inside) @ whi[wt][:, ch].T
    return acc


def epilogue_reference(acc, oy, ox, OW, dcoef=None, bias=None, noise=None, noise_nstride=0, gain=1.0, slope=1.0, clamp=-1.0):
    """Mode-0 epilogue in fp64: v = acc * dcoef[n, o] + noise[n * noise_nstride + oy * OW + ox] + bias[o]; lrelu_slope(v) * gain;
    clamp.  oy / ox: output row / column of each M-space row / column."""
    N = acc.shape[0]
    v = acc.clone()
    if dcoef is not None:
        v = v * dcoef.double()[:, None, None, :]
    if noise is not None:
        idx = torch.arange(N, device=acc.device)[:, None, None] * noise_nstride + oy[None, :, None] * OW + ox[None, None, :]
        v = v + noise.double().flatten()[idx.clamp(0, noise.numel() - 1)][..., None]      # (clipped pixels are not compared)
    if bias is not None:
        v = v + bias.double()
    v = torch.where(v > 0, v, v * slope) * gain
    if clamp >= 0:
        v = v.clamp(-clamp, clamp)
    return v


class Expected(Guarded):
    """A guarded output whose owned elements (`own`) and their fp64 reference (`expect`) _place fills in."""

    def __init__(self, shape, dtype):
        super().__init__(shape, dtype, own=torch.zeros(shape, dtype=torch.bool, device=DEV))
        self.expect = torch.zeros(shape, dtype=torch.float64, device=DEV)


def _place(g, vals, yv, xv, oy, ox, coff, nchw, accumulate=None):
    """Mark the output elements of M-space pixels (yv x xv) as owned and set their reference (+ the prior content when accumulating)."""
    N, Cn = vals.shape[0], vals.shape[-1]
    n = torch.arange(N, device=DEV)[:, None, None, None]
    c = torch.arange(Cn, device=DEV)[None, None, None, :] + coff
    Y, X = oy[yv][None, :, None, None], ox[xv][None, None, :, None]
    v = vals[:, yv][:, :, xv]
    idx = (n, c, Y, X) if nchw else (n, Y, X, c)
    g.own[idx] = True
    g.expect[idx] = v + (accumulate[idx].double() if accumulate is not None else 0.0)


def _seeded(c):
    return torch.Generator(device=DEV).manual_seed(1000 + CASE_IDS.index(c['name']))


def setup_case(c):
    """Operands, epilogue vectors and guarded outputs of a case (the device tensors every descriptor points at)."""
    from next3d_b200 import kernels as K
    g = _seeded(c)
    N, Cin, Cout = c['N'], c['Cin'], c['Cout']
    NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW = _geometry(c)
    taps = _taps(c)
    T = max(t[3] for t in taps) + 1
    a_hi, a_lo = K.split_bf16(torch.randn(NI, AH, AW, Cin, device=DEV, generator=g))
    w_hi, w_lo = K.split_bf16(torch.randn(T, Cout, Cin, device=DEV, generator=g) / math.sqrt(Cin * len(taps)))
    s = dict(c=c, taps=taps, a_hi=a_hi, a_lo=a_lo, w_hi=w_hi, w_lo=w_lo, geo=(NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW))
    if c['epi'] == 'full':
        s.update(dcoef=torch.rand(N, Cout, device=DEV, generator=g) + 0.5, bias=torch.randn(Cout, device=DEV, generator=g) * 0.5,
                 gain=math.sqrt(2), slope=0.2, clamp=2.0)
    elif c['epi'] == 'torgb':
        s.update(dcoef=None, bias=torch.randn(Cout, device=DEV, generator=g), gain=1.0, slope=1.0, clamp=1.5)
    else:
        s.update(dcoef=None, bias=None, gain=1.0, slope=1.0, clamp=-1.0)
    s['noise'], s['noise_nstride'] = None, 0
    if c['noise'] == 'shared':
        s['noise'] = torch.randn(OH, OW, device=DEV, generator=g) * 0.3
    elif c['noise'] == 'sample':
        s['noise'], s['noise_nstride'] = torch.randn(N, OH, OW, device=DEV, generator=g) * 0.3, OH * OW
    s['styles'] = [torch.randn(N, Cout, device=DEV, generator=g) for _ in c['outs']]
    s['outs'] = [(Expected((N, OH, OW, o['cstride']), torch.bfloat16), Expected((N, OH, OW, o['cstride']), torch.bfloat16)) for o in c['outs']]
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
    if c['splits'] > 1:             # second pass: n3d_splitk_epilogue with the full epilogue into fresh guarded outputs
        s.update(dcoef=torch.rand(N, Cout, device=DEV, generator=g) + 0.5, bias=torch.randn(Cout, device=DEV, generator=g) * 0.5,
                 gain=math.sqrt(2), slope=0.2, clamp=2.0)
        per_sample = c['epi_noise'] == 'sample'
        s['noise'] = torch.randn(*((N,) if per_sample else ()), OH, OW, device=DEV, generator=g) * 0.3
        s['noise_nstride'] = OH * OW if per_sample else 0
        s['epi_styles'] = [torch.randn(N, Cout, device=DEV, generator=g) for _ in range(2)]
        s['epi_outs'] = [(Expected((N, OH, OW, cs), torch.bfloat16), Expected((N, OH, OW, cs), torch.bfloat16)) for cs in (Cout, 2 * Cout)]
        s['epi_f32'] = Expected((N, OH, OW, Cout), torch.float32)
    # the reference: accumulators (per split-K slice), then owned elements and expected values of every output
    yv, xv = _valid(s)
    oy = torch.arange(c['MH'], device=DEV) * oy_mul + oy_off
    ox = torch.arange(c['MW'], device=DEV) * ox_mul + ox_off
    s['map'] = (yv, xv, oy, ox)
    _expect(s)
    return s


def _valid(s):
    c = s['c']
    *_, oy_mul, oy_off, ox_mul, ox_off, OH, OW = s['geo']
    yv = torch.nonzero(torch.arange(c['MH'], device=DEV) * oy_mul + oy_off < OH).flatten()
    xv = torch.nonzero(torch.arange(c['MW'], device=DEV) * ox_mul + ox_off < OW).flatten()
    return yv, xv


def _expect(s):
    c, p = s['c'], _plan(s['c'])
    N, MH, MW = c['N'], c['MH'], c['MW']
    NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW = s['geo']
    yv, xv, oy, ox = s['map']
    ref = lambda **kw: conv_reference(s['a_hi'], s['a_lo'], s['w_hi'], s['w_lo'], s['taps'], N, MH, MW, a_img_mul, c['nprod'], **kw)
    epi = lambda acc: epilogue_reference(acc, oy, ox, OW, s['dcoef'], s['bias'], s['noise'], s['noise_nstride'], s['gain'], s['slope'], s['clamp'])
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
        for (hi, lo), sty, (cs, coff) in zip(s['epi_outs'], s['epi_styles'], ((c['Cout'], 0), (2 * c['Cout'], c['Cout']))):
            for t in (hi, lo):
                _place(t, v * sty.double()[:, None, None, :], yv, xv, oy, ox, coff, False)
        _place(s['epi_f32'], v, yv, xv, oy, ox, 0, False)
        return
    acc = ref()
    v = acc if c['mode'] == 1 else epi(acc)
    for (hi, lo), sty, o in zip(s['outs'], s['styles'], c['outs']):
        for t in (hi, lo):
            _place(t, v * (sty.double()[:, None, None, :] if c['mode'] == 0 else 1.0), yv, xv, oy, ox, o['coff'], False)
    if f is not None:
        prior = None
        if f['acc']:                # accumulating output: finite prior content in the owned region
            _place(s['f32'], v, yv, xv, oy, ox, f['coff'], f['nchw'])
            s['f32'].view[s['f32'].own] = torch.randn(int(s['f32'].own.sum()), device=DEV, generator=_seeded(c))
            prior = s['f32'].view.clone()
        _place(s['f32'], v, yv, xv, oy, ox, f['coff'], f['nchw'], prior)
    r = c['rgb']
    if r:
        img = torch.einsum('nyxo,no,co->nyxc', v, s['rgb_s'].double(), s['rgb_w'].double()) + s['rgb_b'].double()
        img = img.clamp(-2.0, 2.0)
        prior = None
        if r['acc']:
            _place(s['rgb'], img, yv, xv, oy, ox, 0, r['nchw'])
            s['rgb'].view[s['rgb'].own] = torch.randn(int(s['rgb'].own.sum()), device=DEV, generator=_seeded(c))
            prior = s['rgb'].view.clone()
        _place(s['rgb'], img, yv, xv, oy, ox, 0, r['nchw'], prior)


def _place_slice(g, k, part, yv, xv, oy, ox):
    """Split-K partial sums of slice k: output [S, N, OH, OW, Cout]."""
    N, Cn = part.shape[0], part.shape[-1]
    n = torch.arange(N, device=DEV)[:, None, None, None]
    cc = torch.arange(Cn, device=DEV)[None, None, None, :]
    idx = (torch.full_like(n, k), n, oy[yv][None, :, None, None], ox[xv][None, None, :, None], cc)
    g.own[idx] = True
    g.expect[idx] = part[:, yv][:, :, xv]


def launch_case(s):
    from next3d_b200 import kernels as K
    c = s['c']
    NI, AH, AW, a_img_mul, oy_mul, oy_off, ox_mul, ox_off, OH, OW = s['geo']
    outs = [K.make_split_out(hi.view, lo.view, sty if c['mode'] == 0 else None, o['cstride'], o['coff'])
            for (hi, lo), sty, o in zip(s['outs'], s['styles'], c['outs'])]
    f = c['f32']
    kw = {}
    if f is not None:
        kw = dict(out_f32=s['f32'].view, f32_cstride=f['cstride'], f32_coff=f['coff'], f32_nchw=f['nchw'], f32_accumulate=f['acc'])
    if c['rgb']:
        r = c['rgb']
        kw['rgb'] = dict(out=s['rgb'].view, weight=s['rgb_w'], style=s['rgb_s'], bias=s['rgb_b'], clamp=2.0, nchw=r['nchw'], accumulate=r['acc'])
    if c['splits'] > 1:
        kw.update(splits=c['splits'], split_stride=s['f32'].view[0].numel())
    mode0 = c['mode'] == 0
    K.conv_gemm(s['a_hi'], s['a_lo'] if c['nprod'] == 3 else None, s['w_hi'], s['w_lo'] if c['nprod'] == 3 else None, s['taps'], c['N'],
                c['MH'], c['MW'], a_img_mul=a_img_mul, nprod=c['nprod'], mode=c['mode'], dcoef=s['dcoef'] if mode0 else None,
                bias=s['bias'] if mode0 else None, noise=s['noise'] if mode0 else None, noise_nstride=s['noise_nstride'] if mode0 else 0,
                gain=s['gain'], slope=s['slope'], clamp=s['clamp'], outs=outs, oy_mul=oy_mul, oy_off=oy_off, ox_mul=ox_mul, ox_off=ox_off,
                OH=OH, OW=OW, **kw)
    if c['splits'] > 1:
        Cout = c['Cout']
        eouts = [K.make_split_out(hi.view, lo.view, sty, cs, coff)
                 for (hi, lo), sty, (cs, coff) in zip(s['epi_outs'], s['epi_styles'], ((Cout, 0), (2 * Cout, Cout)))]
        K.splitk_epilogue(s['f32'].view, s['dcoef'], s['bias'], s['noise'], s['gain'], s['slope'], s['clamp'], outs=eouts,
                          out_f32=s['epi_f32'].view, f32_cstride=Cout, f32_coff=0, noise_nstride=s['noise_nstride'])


def _err(got, g):
    ref = g.expect[g.own]
    return ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item()


def check_case(s):
    """-> {output: range-relative error}; asserts the sentinel and written-element checks."""
    c = s['c']
    errs = {}

    def split_pair(name, hi, lo):
        assert hi.untouched_ok() and lo.untouched_ok(), f'{name}: an element outside the output was written'
        assert hi.written() and lo.written(), f'{name}: an owned element was not written'
        errs[name] = ('split', _err(hi.view[hi.own].double() + lo.view[lo.own].double(), hi))

    def f32(name, g, kind, accumulate=False):
        assert g.untouched_ok(), f'{name}: an element outside the output was written'
        assert accumulate or g.written(), f'{name}: an owned element was not written'
        errs[name] = (kind, _err(g.view[g.own].double(), g))

    for k, (hi, lo) in enumerate(s['outs']):
        split_pair(f'out{k}', hi, lo)
    if s['f32'] is not None:
        f32('f32', s['f32'], 'raw' if c['mode'] == 1 else 'f32', c['f32']['acc'])
    if c['rgb']:
        f32('rgb', s['rgb'], 'rgb', c['rgb']['acc'])
    if c['splits'] > 1:
        for k, (hi, lo) in enumerate(s['epi_outs']):
            split_pair(f'splitk_epilogue.out{k}', hi, lo)
        f32('splitk_epilogue.f32', s['epi_f32'], 'f32')
    return errs


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_conv_gemm_matches_fp64_contract(c):
    s = setup_case(c)
    launch_case(s)
    torch.cuda.synchronize()
    errs = check_case(s)
    bad = {k: (kind, e) for k, (kind, e) in errs.items() if not e < BOUNDS[kind]}
    assert not bad, bad


@pytest.mark.gpu
def test_launched_instance_matches_plan(tmp_path):
    """Every case under torch.profiler: the conv_gemm_kernel<block_n, block_k> it launched (the template arguments are in the
    demangled name) and its grid are the ones `plan` predicts."""
    setups = [setup_case(c) for c in CASES]
    torch.cuda.synchronize()

    def run():
        for s in setups:
            launch_case(s)
        return CASES                        # one conv_gemm_kernel launch per case

    _, events = launched_kernels(run, 'conv_gemm_kernel', tmp_path)
    props = torch.cuda.get_device_properties(0)
    for c, e in zip(CASES, events):
        p = plan(c['N'], c['Cin'], c['Cout'], c['MH'], c['MW'], c['splits'], bool(c['rgb']), sms=props.multi_processor_count,
                 cluster_slots=props.multi_processor_count // 2)
        m = re.search(r'conv_gemm_kernel<(\d+), (\d+)>', e['name'])
        assert m and (int(m.group(1)), int(m.group(2))) == (p['block_n'], p['block_k']), (c['name'], e['name'], p)
        grid = e.get('args', {}).get('grid')
        if grid is not None:
            assert list(grid) == [p['grid'], 1, 1], (c['name'], grid, p)
        cl = e.get('args', {}).get('cluster')
        if cl is not None:
            assert list(cl)[0] == p['cluster'], (c['name'], cl, p)


# ------------------------------------------------------------------------------------------------ alignment (CPU, nothing launched)
def _desc(a, w, N=1, MH=8, MW=16):
    L = lib()
    p = L.ConvGemm()
    p.a_hi, p.a_lo, p.w_hi, p.w_lo = a.data_ptr(), a.data_ptr(), w.data_ptr(), w.data_ptr()
    p.NI, p.AH, p.AW, p.Cin = a.shape
    p.T, p.Cout = w.shape[0], w.shape[1]
    p.N, p.MH, p.MW = N, MH, MW
    p.ntaps = 1
    p.taps[0] = L.ConvTap(0, 0, 0, 0)
    p.nprod = 3
    p.gain, p.slope, p.clamp = 1.0, 1.0, -1.0
    p.oy_mul, p.ox_mul, p.OH, p.OW = 1, 1, MH, MW
    return p


@pytest.mark.parametrize('field', ['out_f32', 'out0.hi', 'out1.lo'])
def test_conv_gemm_refuses_misaligned_outputs(field):
    L = lib()
    a = torch.zeros(1, 8, 16, 16, dtype=torch.bfloat16)
    w = torch.zeros(1, 16, 16, dtype=torch.bfloat16)
    f32 = torch.zeros(1 * 8 * 16 * 16 + 64)
    hi = torch.zeros(1 * 8 * 16 * 16 + 64, dtype=torch.bfloat16)
    p = _desc(a, w)
    if field == 'out_f32':
        p.out_f32, p.f32_cstride = offset_view(f32, 4).data_ptr(), 16
        what = 'out_f32 must be 16-byte aligned'
    else:
        k, part = int(field[3]), field.split('.')[1]
        good, bad = hi.data_ptr(), offset_view(hi, 4).data_ptr()
        p.out[k] = L.SplitOut(bad if part == 'hi' else good, bad if part == 'lo' else good, None, 16, 0)
        what = f'split output {k} (hi / lo) must be 16-byte aligned'
    refused(L.lib.n3d_conv_gemm(C.byref(p), None), what)
    if field == 'out_f32':                 # the transposed-conv entry point shares the check
        p.T = 9
        w9 = torch.zeros(9, 16, 16, dtype=torch.bfloat16)
        p.w_hi = p.w_lo = w9.data_ptr()
        refused(L.lib.n3d_conv_transposed_gemm(C.byref(p), None), what)


def test_conv_gemm_refuses_accumulate_with_split_outputs():
    """The accumulating fp32 store adds the old values into the epilogue's registers before the split outputs are formed from them."""
    L = lib()
    a = torch.zeros(1, 8, 16, 16, dtype=torch.bfloat16)
    w = torch.zeros(1, 16, 16, dtype=torch.bfloat16)
    f32 = torch.zeros(8 * 16 * 16)
    hi = torch.zeros(8 * 16 * 16, dtype=torch.bfloat16)
    p = _desc(a, w)
    p.out_f32, p.f32_cstride, p.f32_accumulate = f32.data_ptr(), 16, 1
    p.out[1] = L.SplitOut(hi.data_ptr(), hi.data_ptr(), None, 16, 0)
    refused(L.lib.n3d_conv_gemm(C.byref(p), None), 'f32_accumulate cannot be combined with split outputs')


def test_conv_gemm_refuses_split_stride_not_multiple_of_4():
    L = lib()
    a = torch.zeros(1, 8, 16, 16, dtype=torch.bfloat16)
    w = torch.zeros(9, 16, 16, dtype=torch.bfloat16)
    f32 = torch.zeros(2 * 8 * 16 * 16 + 64)
    p = _desc(a, w)
    p.mode, p.out_f32, p.f32_cstride, p.splits, p.split_stride = 1, f32.data_ptr(), 16, 2, 8 * 16 * 16 + 2
    refused(L.lib.n3d_conv_gemm(C.byref(p), None), 'split stride that is a multiple of 4')


@pytest.mark.parametrize('entry', ['n3d_splitk_epilogue', 'n3d_fir_up_epilogue'])
@pytest.mark.parametrize('field', ['raw', 'dcoef', 'bias', 'out_f32', 'out0.hi', 'out1.lo', 'out0.style'])
def test_epilogues_refuse_misaligned_pointers(entry, field):
    L = lib()
    N, H, W, Cc = 1, 8, 8, 16
    raw = torch.zeros(N * (H + 1) * (W + 1) * Cc + 64)
    vec = torch.zeros(N * Cc + 64)
    f32 = torch.zeros(N * H * W * Cc + 64)
    bf = torch.zeros(N * H * W * 2 * Cc + 64, dtype=torch.bfloat16)
    ptrs = dict(raw=raw.data_ptr(), dcoef=vec.data_ptr(), bias=vec.data_ptr(), out_f32=f32.data_ptr())
    outs = (L.SplitOut * 2)(L.SplitOut(bf.data_ptr(), bf.data_ptr(), vec.data_ptr(), Cc, 0),
                            L.SplitOut(bf.data_ptr(), bf.data_ptr(), vec.data_ptr(), 2 * Cc, Cc))
    base = {'raw': raw, 'dcoef': vec, 'bias': vec, 'out_f32': f32}
    if field in ptrs:
        if field == 'raw' and entry == 'n3d_splitk_epilogue':
            what = 'multiples of 4'                 # the partial sums' alignment is checked with their stride
        else:
            what = {'raw': 'raw must be 16-byte aligned', 'dcoef': 'dcoef and bias must be 16-byte aligned',
                    'bias': 'dcoef and bias must be 16-byte aligned', 'out_f32': 'out_f32 must be 16-byte aligned'}[field]
        ptrs[field] = offset_view(base[field], 4).data_ptr()
    else:
        k, part = int(field[3]), field.split('.')[1]
        setattr(outs[k], part, offset_view(vec if part == 'style' else bf, 4).data_ptr())
        what = f'split output {k} (hi / lo / style) must be 16-byte aligned'
    if entry == 'n3d_splitk_epilogue':
        rc = L.lib.n3d_splitk_epilogue(ptrs['raw'], 1, N * H * W * Cc, N, H, W, Cc, ptrs['dcoef'], ptrs['bias'], None, 0, 1.0, 0.2, -1.0,
                                       outs, ptrs['out_f32'], Cc, 0, None)
    else:
        rc = L.lib.n3d_fir_up_epilogue(ptrs['raw'], N, H, W, Cc, ptrs['dcoef'], ptrs['bias'], None, 0, 1.0, 0.2, -1.0, outs,
                                       ptrs['out_f32'], Cc, 0, None)
    refused(rc, what)
