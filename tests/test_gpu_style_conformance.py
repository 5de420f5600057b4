"""The kernels that turn a latent into ws, and ws into every layer's modulation, against an fp64 reference over a table of launches
that reaches every launch shape their entry points take:

    n3d_mapping      mapping_kernel       one CTA of 512 threads per latent
    n3d_interp_rows  interp_rows_kernel   one thread per output element, grid-stride
    n3d_styles       styles_kernel        one warp per affine row (a layer's input channel), grid-stride over rows
    n3d_demod        demod_kernel         one warp per output channel of a layer, grid-stride over rows

The references restate the formulas of include/next3d_b200.h (n3d_styles, n3d_demod) and of the MappingNetwork (as oracle.generator.
mapping does, but in fp64) on the device.  demod is evaluated on its own inputs cast to fp64, so that its error is not mixed with the
error of the styles it reads.

Every output is a view into a larger allocation filled with a NaN sentinel: the elements a launch owns must be written (and match),
every other element -- guard bands, the gaps between two layers' blocks -- must keep the sentinel's bits.  The unowned gaps of demod's
inputs hold NaN, so that a read outside a layer's block poisons its result.  Each case is then rerun: the rerun must be bit-identical.
styles, demod and mapping compute image n of a batch in a warp or CTA of its own, so image n must also be bit-identical to a launch of
that image alone.

`plan` mirrors the launch rules in plain Python.  The CPU test checks that the table covers everything in COVERAGE; the profiler test
checks on the GPU that each case ran the kernel and grid the plan predicts.  The engine test checks the real style and dcoef tables of
the tiny and full configurations; the alignment tests at the end need no GPU.
"""
import functools
import math
import re

import numpy as np
import pytest
import torch

from next3d_b200 import config, weights
from tests.helpers import Guarded, RangeErr, cdiv, grid_stride, launched_kernels, lib, offset_view, oracle_widx, range_rel_err, \
    record_errors, refused, rerun_identical

DEV = 'cuda'
SMS = 132                   # SM count the table is planned at (H100 SXM)
WARPS = 8                   # warps per CTA of styles_kernel / demod_kernel (256 threads)
WARP_CAP = SMS * 8 * WARPS  # rows of styles / demod with one warp each: n3d_grid caps the launch at 8 CTAs per SM
FULL_STYLE_ROWS, FULL_DEMOD_ROWS = 29216, 18176             # the full configuration's tables

# Error bounds, each 4x the worst case measured over the table and the engine test on an H100 80GB HBM3 (700 W power limit), which is
# given beside it.  styles, mapping, interp: range-relative, max |got - ref| / max |ref| over a case's output.  demod: relative,
# max |got - ref| / ref over the coefficients (all positive).  N3D_STYLE_ERRORS=<file> appends every measured error to that file as
# JSON lines.
BOUNDS = {
    'styles': 7e-7,         # Worst: 1.7e-7 (engine_full_config_call2_n3)
    'demod': 7.5e-7,        # Worst: 1.8e-7 (demod_n64_cap_plus_1)
    'mapping': 1.4e-6,      # Worst: 3.4e-7 (map_n3_psi0p7_c14)
    'interp': 1e-6,         # Worst: 2.5e-7 (interp_k24_d14336_cubic: the basis rounded to fp32)
}


# ------------------------------------------------------------------------------------------------ the launch rules, mirrored
def rows(c):
    return sum(L[0] for L in c['layers']) if c['kind'] == 'styles' else sum(L[1] for L in c['layers'])


def plan(c, sms=SMS):
    """Kernel, grid, work items and grid-stride passes of a case."""
    k = c['kind']
    if k in ('styles', 'demod'):
        r = rows(c)
        grid = grid_stride(r * 32, sms, 8)
        return dict(kernel=f'{k}_kernel', grid=grid, work=r, passes=cdiv(r, WARPS * grid))
    if k == 'mapping':
        return dict(kernel='mapping_kernel', grid=c['N'], work=c['N'], passes=1)
    work = c['F'] * c['D']
    grid = grid_stride(work, sms, 8)
    return dict(kernel='interp_rows_kernel', grid=grid, work=work, passes=cdiv(work, 256 * grid))


# ------------------------------------------------------------------------------------------------ the case table
def _styles(name, N, num_ws, wdim, layers, gap=0):
    """layers: (Cin, ws index, scale) of each layer; gap: unowned elements before every layer's [N, Cin] block and after the last."""
    return dict(name=name, kind='styles', N=N, num_ws=num_ws, wdim=wdim, layers=layers, gap=gap)


def _demod(name, N, layers, gap=0, styles='randn'):
    """layers: (Cin, Cout) of each layer; gap: NaN / unowned elements before every block of the styles, wsq and dcoef buffers.
    styles: 'randn'; 'tiny' (|s| ~ 1e-7: the 1e-8 epsilon dominates); 'zero' (image 0 of the first layer all zero)."""
    return dict(name=name, kind='demod', N=N, layers=layers, gap=gap, styles=styles)


def _mapping(name, N, psi=1.0, cutoff=None, c_scale=1.0, zscale=1.0, zero_row=False, num_ws=28):
    return dict(name=name, kind='mapping', N=N, psi=psi, cutoff=cutoff, c_scale=c_scale, zscale=zscale, zero_row=zero_row, num_ws=num_ws)


def _interp(name, K, D, F=None, basis='random', w_frames=None):
    """basis 'random' (F rows with exact zeros and negative entries) or the interpolate_ws basis of that kind over K keyframes
    (F = K * w_frames)."""
    return dict(name=name, kind='interp', K=K, D=D, F=F if F is not None else K * w_frames, basis=basis, w_frames=w_frames)


def _layers(total, cin, num_ws, scale=1.0):
    """Layers of `cin` rows (the last one ragged) adding up to `total` rows, cycling through every ws index."""
    return [(min(cin, total - r), (r // cin) % num_ws, scale) for r in range(0, total, cin)]


CASES = [
    # styles: wdim 4 (one lane busy), 68 (17 lanes), 200 (a ragged second pass of the lane loop), 128 and 512 (exact)
    _styles('styles_w4_n1', 1, 3, 4, [(3, 0, 1.0), (33, 2, 0.25), (64, 1, 1.0)], gap=5),
    _styles('styles_w68_n2', 2, 5, 68, [(33, 4, 1.0), (3, 0, 0.5), (100, 2, 1.0)], gap=3),
    _styles('styles_w200_n7', 7, 9, 200, [(3, 8, 1.0), (33, 0, 2.0), (300, 4, 1.0)], gap=1),
    _styles('styles_w128_n2_cap', 2, 14, 128, [(33, i % 14, 1.0 if i % 3 else 0.125) for i in range(WARP_CAP // 33)], gap=2),
    _styles('styles_w512_n7_cap_plus_1', 7, 28, 512, _layers(WARP_CAP - 256, 512, 28) + [(257, 27, 0.5)], gap=4),
    _styles('styles_w512_n64_full', 64, 28, 512, _layers(FULL_STYLE_ROWS, 512, 28, scale=1.0), gap=0),
    # demod: Cin 1 .. 512 below the warp cap, at the full configuration's row count, above the cap at N 64
    _demod('demod_cin1_3_16_n1', 1, [(1, 5), (3, 7), (16, 40)], gap=3),
    _demod('demod_cin31_32_33_n3', 3, [(31, 64), (32, 33), (33, 100)], gap=2),
    _demod('demod_cin512_n3_full', 3, [(512, 512)] * 35 + [(512, 256)], gap=1),
    _demod('demod_n64_cap_plus_1', 64, [(64, 4096), (33, 4353)], gap=1),
    _demod('demod_tiny_styles', 3, [(512, 64), (3, 16)], gap=2, styles='tiny'),
    _demod('demod_zero_row', 3, [(33, 40), (16, 8)], gap=2, styles='zero'),
    # mapping: N up to 1024, psi on both sides of torch.lerp's switch at 0.5 and outside [0, 1], every kind of cutoff
    _mapping('map_n1', 1),
    _mapping('map_n3_psi0p7_c14', 3, psi=0.7, cutoff=14),
    _mapping('map_n133_psi0p5_cm1', 133, psi=0.5, cutoff=-1),
    _mapping('map_n1024_psi0p4999', 1024, psi=0.4999),
    _mapping('map_psi0_c0', 3, psi=0.0, cutoff=0),
    _mapping('map_psi0_c40', 2, psi=0.0, cutoff=40),
    _mapping('map_psim0p5_c1', 3, psi=-0.5, cutoff=1),
    _mapping('map_psi1p5_c27', 3, psi=1.5, cutoff=27),
    _mapping('map_c28_cscale0', 3, psi=0.7, cutoff=28, c_scale=0.0),
    _mapping('map_cm14_zsmall', 3, psi=0.7, cutoff=-14, zscale=1e-3),
    _mapping('map_zlarge_zero_row', 4, psi=0.6, cutoff=14, zscale=1e3, zero_row=True),
    _mapping('map_ws1_cm1', 3, psi=0.7, cutoff=-1, num_ws=1),
    _mapping('map_ws1_none', 2, psi=0.5, num_ws=1),
    # interp_rows: F * D below and above the grid cap, random bases and the interpolation bases of the frame drivers
    _interp('interp_k1_d14336', 1, 14336, F=40),
    _interp('interp_k4_d7', 4, 7, F=9),
    _interp('interp_k24_d1', 24, 1, F=300),
    _interp('interp_k1_d7_cubic', 1, 7, basis='cubic', w_frames=3),
    _interp('interp_k24_d14336_cubic', 24, 14336, basis='cubic', w_frames=2),
    _interp('interp_k4_d14336_linear', 4, 14336, basis='linear', w_frames=8),
]
CASE_IDS = [c['name'] for c in CASES]


def _of(kind, cs):
    return [(c, p) for c, p in cs if c['kind'] == kind]


def _lanes(wdim):
    q = wdim // 4
    return 'fewer than 32' if q < 32 else 'exact' if q % 32 == 0 else 'ragged'


def _rows_class(r):
    return {FULL_STYLE_ROWS: 'full', WARP_CAP: 'cap', WARP_CAP + 1: 'cap + 1'}.get(r, 'below' if r < WARP_CAP else 'above')


COVERAGE = {
    'styles: wdim 4, 68, 128, 512': lambda cs: {c['wdim'] for c, p in _of('styles', cs)} >= {4, 68, 128, 512},
    'styles: fewer than 32 lanes busy, a ragged lane loop, exact multiples': lambda cs: {_lanes(c['wdim']) for c, p in _of('styles', cs)}
        == {'fewer than 32', 'ragged', 'exact'},
    'styles: rows below the warp cap, at it, one over it, and the full configuration\'s':
        lambda cs: {_rows_class(p['work']) for c, p in _of('styles', cs)} >= {'below', 'cap', 'cap + 1', 'full'},
    'styles: N 1, 2, 7, 64': lambda cs: {c['N'] for c, p in _of('styles', cs)} >= {1, 2, 7, 64},
    'styles: ws index 0 and num_ws - 1 in one launch': lambda cs: any({0, c['num_ws'] - 1} <= {L[1] for L in c['layers']} for c, p in _of('styles', cs)),
    'styles: a scale other than 1': lambda cs: any(L[2] != 1.0 for c, p in _of('styles', cs) for L in c['layers']),
    'styles: Cin 3 and 33 blocks with unowned gaps between them':
        lambda cs: any(c['gap'] > 0 and {3, 33} <= {L[0] for L in c['layers']} for c, p in _of('styles', cs)),
    'styles: grid-stride loop taken': lambda cs: any(p['passes'] > 1 for c, p in _of('styles', cs)),
    'demod: Cin 1, 3, 16, 31, 32, 33, 512': lambda cs: {L[0] for c, p in _of('demod', cs) for L in c['layers']} >= {1, 3, 16, 31, 32, 33, 512},
    'demod: rows below and above the warp cap': lambda cs: {p['work'] > WARP_CAP for c, p in _of('demod', cs)} == {False, True},
    'demod: the full configuration\'s rows': lambda cs: any(p['work'] == FULL_DEMOD_ROWS for c, p in _of('demod', cs)),
    'demod: N 1, 3, 64': lambda cs: {c['N'] for c, p in _of('demod', cs)} >= {1, 3, 64},
    'demod: several layers at non-zero soff / ooff bases': lambda cs: any(c['gap'] > 0 and len(c['layers']) > 1 for c, p in _of('demod', cs)),
    'demod: styles so small that the 1e-8 epsilon dominates': lambda cs: any(c['styles'] == 'tiny' for c, p in _of('demod', cs)),
    'demod: an all-zero style row': lambda cs: any(c['styles'] == 'zero' for c, p in _of('demod', cs)),
    'demod: grid-stride loop taken': lambda cs: any(p['passes'] > 1 for c, p in _of('demod', cs)),
    'mapping: N 1, 3, 133, 1024': lambda cs: {c['N'] for c, p in _of('mapping', cs)} >= {1, 3, 133, 1024},
    'mapping: more CTAs than SMs': lambda cs: any(p['grid'] > SMS for c, p in _of('mapping', cs)),
    'mapping: psi 1, 0.7, 0.5, 0.4999 (both formulas of torch.lerp)': lambda cs: {c['psi'] for c, p in _of('mapping', cs)} >= {1.0, 0.7, 0.5, 0.4999},
    'mapping: psi 0, -0.5, 1.5': lambda cs: {c['psi'] for c, p in _of('mapping', cs)} >= {0.0, -0.5, 1.5},
    'mapping: cutoff None, 0, 1, 14, 27, 28, 40, -1, -14 under truncation':
        lambda cs: {c['cutoff'] for c, p in _of('mapping', cs) if c['psi'] != 1} >= {None, 0, 1, 14, 27, 28, 40, -1, -14},
    'mapping: c_scale 1 and 0': lambda cs: {c['c_scale'] for c, p in _of('mapping', cs)} >= {1.0, 0.0},
    'mapping: z scaled by 1e-3 and 1e3': lambda cs: {c['zscale'] for c, p in _of('mapping', cs)} >= {1e-3, 1e3},
    'mapping: an all-zero z row': lambda cs: any(c['zero_row'] for c, p in _of('mapping', cs)),
    'mapping: num_ws 28 and 1': lambda cs: {c['num_ws'] for c, p in _of('mapping', cs)} >= {28, 1},
    'mapping: num_ws 1 with cutoff -1 (no layer truncated) and None (the only layer)':
        lambda cs: {c['cutoff'] for c, p in _of('mapping', cs) if c['num_ws'] == 1 and c['psi'] != 1} >= {-1, None},
    'mapping: psi 0.7 with cutoff 14, as the drivers truncate': lambda cs: any(c['psi'] == 0.7 and c['cutoff'] == 14 for c, p in _of('mapping', cs)),
    'interp: random B at K 1, 4, 24': lambda cs: {c['K'] for c, p in _of('interp', cs) if c['basis'] == 'random'} >= {1, 4, 24},
    'interp: random B at D 1, 7, 14336': lambda cs: {c['D'] for c, p in _of('interp', cs) if c['basis'] == 'random'} >= {1, 7, 14336},
    'interp: interpolate_ws bases at K 1, 4, 24': lambda cs: {c['K'] for c, p in _of('interp', cs) if c['basis'] != 'random'} >= {1, 4, 24},
    'interp: F * D below and above the grid cap': lambda cs: {p['passes'] > 1 for c, p in _of('interp', cs)} == {False, True},
    'interp: B with exact zeros and negative entries': lambda cs: any(c['basis'] == 'random' for c, p in _of('interp', cs)),
    'interp: the cubic and linear bases of interpolate_ws': lambda cs: {c['basis'] for c, p in _of('interp', cs)} >= {'cubic', 'linear'},
    'interp: a cubic basis above the grid cap': lambda cs: any(c['basis'] == 'cubic' and p['passes'] > 1 for c, p in _of('interp', cs)),
}


def case_bytes(c):
    """Device memory of a case: inputs, the guarded output and its fp64 reference."""
    k, N = c['kind'], c.get('N', 1)
    if k == 'styles':
        r = rows(c)
        return N * c['num_ws'] * c['wdim'] * 4 + r * (c['wdim'] + 8) * 4 + 3 * (N * r + c['gap'] * (len(c['layers']) + 1)) * 4 + 8 * N * r
    if k == 'demod':
        w = sum(ci * co for ci, co in c['layers'])
        s = sum(N * ci for ci, co in c['layers'])
        return w * 4 + s * 12 + rows(c) * 40 + N * rows(c) * 12
    if k == 'mapping':
        return N * (512 + 25) * 12 + N * c['num_ws'] * 512 * 12 + 4 * 2 ** 20
    return c['K'] * c['D'] * 12 + c['F'] * c['K'] * 12 + c['F'] * c['D'] * 12


def test_case_table_covers_every_launch_configuration():
    """CPU: the table reaches everything listed in COVERAGE, according to the mirrored launch rules, at <= 512 MB per case."""
    planned = [(c, plan(c)) for c in CASES]
    missing = [k for k, ok in COVERAGE.items() if not ok(planned)]
    assert not missing, missing
    assert len(set(CASE_IDS)) == len(CASE_IDS)
    big = {c['name']: case_bytes(c) / 2 ** 20 for c in CASES if case_bytes(c) > 512 * 2 ** 20}
    assert not big, big


# ------------------------------------------------------------------------------------------------ the fp64 mapping reference
@functools.lru_cache(maxsize=None)
def _mapping_state():
    cfg = config.tiny_config(512)
    return cfg, weights.make_state_dict(cfg, seed=31)


def mapping_params(sd, device):
    """n3d_mapping's parameter dict of a state dict's backbone.mapping."""
    p = 'backbone.mapping'
    names = dict(embed_w='embed.weight', embed_b='embed.bias', fc0_w='fc0.weight', fc0_b='fc0.bias', fc1_w='fc1.weight', fc1_b='fc1.bias',
                 w_avg='w_avg')
    return {k: sd[f'{p}.{v}'].to(device, torch.float32).contiguous() for k, v in names.items()}


def mapping_reference(m, z, c, c_scale, psi, cutoff, num_ws):
    """oracle.generator.mapping in fp64: normalised z and embedded c, two lrelu layers at lr_multiplier 0.01, truncation of
    ws[:, :cutoff] (all layers for None) towards w_avg."""
    d = {k: v.double() for k, v in m.items()}
    x = z.double()
    x = x * (x.square().mean(1, keepdim=True) + 1e-8).rsqrt()
    y = (c.double() * c_scale) @ (d['embed_w'] / math.sqrt(25)).t() + d['embed_b']
    y = y * (y.square().mean(1, keepdim=True) + 1e-8).rsqrt()
    x = torch.cat([x, y], 1)
    for i in (0, 1):
        x = x @ (d[f'fc{i}_w'] * (0.01 / math.sqrt(x.shape[1]))).t() + d[f'fc{i}_b'] * 0.01
        x = torch.where(x > 0, x, 0.2 * x) * math.sqrt(2)
    x = x[:, None].repeat(1, num_ws, 1)
    if psi != 1:
        x[:, :cutoff] = d['w_avg'].lerp(x[:, :cutoff], psi)
    return x


@pytest.mark.parametrize('psi,cutoff', [(1.0, None), (0.7, 14), (0.4999, -1), (0.0, None), (1.5, 27)])
def test_mapping_reference_matches_oracle(psi, cutoff):
    """CPU: the fp64 restatement agrees with the fp32 oracle (oracle.generator.mapping) to fp32 rounding."""
    from oracle import generator as og
    cfg, sd = _mapping_state()
    z, c, _, _ = weights.demo_inputs(cfg, 4, seed=3)
    ref = mapping_reference(mapping_params(sd, 'cpu'), z, c[:, :25], cfg.rendering_kwargs['c_scale'], psi, cutoff, 28)
    assert range_rel_err(og.mapping(sd, cfg, z, c, psi, cutoff), ref) < 2e-6


# ------------------------------------------------------------------------------------------------ outputs and inputs
def _seeded(c):
    return torch.Generator(device=DEV).manual_seed(3000 + CASE_IDS.index(c['name']))


def style_layout(c, N):
    """Base of every layer's [N, Cin] block in the styles output, and the output's size."""
    bases, at = [], c['gap']
    for L in c['layers']:
        bases.append(at)
        at += N * L[0] + c['gap']
    return bases, at


def demod_layout(c, N):
    """Bases of every layer's styles [N, Cin], wsq [Cout, Cin] and dcoef [N, Cout] blocks, and the sizes of the three buffers."""
    g, s, w, o = c['gap'], [], [], []
    ss = ws = os_ = g
    for cin, cout in c['layers']:
        s.append(ss)
        w.append(ws)
        o.append(os_)
        ss, ws, os_ = ss + N * cin + g, ws + cout * cin + g, os_ + N * cout + g
    return s, w, o, (ss, ws, os_)


def _owned(size, blocks):
    own = torch.zeros(size, dtype=torch.bool, device=DEV)
    for b, n in blocks:
        own[b:b + n] = True
    return own


def _i64(parts):
    return torch.cat(parts).to(DEV, torch.int64)


def _i32(parts):
    return torch.cat(parts).to(DEV, torch.int32)


def styles_tables(c, N):
    """row_ooff of a styles case at batch N, and the guarded output."""
    bases, size = style_layout(c, N)
    ooff = _i64([torch.arange(L[0]) + b for L, b in zip(c['layers'], bases)])
    return ooff, Guarded((size,), own=_owned(size, [(b, N * L[0]) for L, b in zip(c['layers'], bases)]))


def demod_inputs(c, N, s_blocks, wsq_blocks):
    """The styles and wsq buffers of a demod case at batch N from each layer's [N, Cin] styles and [Cout, Cin] wsq (NaN in the gaps),
    its row tables and the guarded output."""
    sb, wb, ob, (ssz, wsz, osz) = demod_layout(c, N)
    styles = torch.full((ssz,), float('nan'), device=DEV)
    wsq = torch.full((wsz,), float('nan'), device=DEV)
    for b, t in zip(sb, s_blocks):
        styles[b:b + t.numel()] = t.reshape(-1)
    for b, t in zip(wb, wsq_blocks):
        wsq[b:b + t.numel()] = t.reshape(-1)
    L = c['layers']
    t = dict(styles=styles, wsq=wsq,
             woff=_i64([torch.arange(co) * ci + b for (ci, co), b in zip(L, wb)]),
             cin=_i32([torch.full((co,), ci) for ci, co in L]),
             soff=_i64([torch.full((co,), b) for (ci, co), b in zip(L, sb)]),
             ooff=_i64([torch.arange(co) + b for (ci, co), b in zip(L, ob)]),
             cout=_i32([torch.full((co,), co) for ci, co in L]))
    t['out'] = Guarded((osz,), own=_owned(osz, [(b, N * co) for (ci, co), b in zip(L, ob)]))
    return t


def setup_case(c):
    """Inputs and guarded output of a case (the device tensors every launch points at)."""
    g = _seeded(c)
    rnd = lambda *shape: torch.randn(*shape, device=DEV, generator=g)      # noqa: E731
    k, s = c['kind'], dict(c=c)
    if k == 'styles':
        r = rows(c)
        s['ws'] = rnd(c['N'], c['num_ws'], c['wdim'])
        s['A'] = rnd(r, c['wdim'])
        s['b'] = rnd(r) * 0.5 + 1.0
        s['widx'] = _i32([torch.full((L[0],), L[1]) for L in c['layers']])
        s['scale'] = torch.cat([torch.full((L[0],), L[2]) for L in c['layers']]).to(DEV)
        s['cin'] = _i32([torch.full((L[0],), L[0]) for L in c['layers']])
        s['ooff'], s['out'] = styles_tables(c, c['N'])
    elif k == 'demod':
        N = c['N']
        s['s_blocks'] = [rnd(N, ci) * (1e-7 if c['styles'] == 'tiny' else 1.0) for ci, co in c['layers']]
        if c['styles'] == 'zero':
            s['s_blocks'][0][0] = 0.0
        s['wsq_blocks'] = [rnd(co, ci, 3, 3).square().sum(dim=[2, 3]) for ci, co in c['layers']]
        s.update(demod_inputs(c, N, s['s_blocks'], s['wsq_blocks']))
    elif k == 'mapping':
        N = c['N']
        s['z'] = rnd(N, 512) * c['zscale']
        if c['zero_row']:
            s['z'][N // 2] = 0.0
        s['cc'] = rnd(N, 25)
        s['m'] = mapping_params(_mapping_state()[1], DEV)
        s['out'] = Guarded((N, c['num_ws'], 512))
    else:
        if c['basis'] == 'random':
            B = rnd(c['F'], c['K'])
            B[torch.rand(c['F'], c['K'], device=DEV, generator=g) < 0.3] = 0.0           # exact zeros: skipped by the kernel
        else:
            from next3d_b200 import drivers
            B = drivers.interpolation_basis(c['K'], c['w_frames'], kind=c['basis']).to(DEV, torch.float32)
        s['B'], s['Y'] = B.contiguous(), rnd(c['K'], c['D'])
        s['out'] = Guarded((c['F'], c['D']))
    return s


def launch_case(s):
    from next3d_b200 import kernels as K
    c = s['c']
    k = c['kind']
    if k == 'styles':
        K.styles(s['ws'], s['A'], s['b'], s['widx'], s['scale'], s['ooff'], s['cin'], s['out'].view)
    elif k == 'demod':
        K.demod(s['styles'], s['wsq'], s['woff'], s['cin'], s['soff'], s['ooff'], s['cout'], s['out'].view, c['N'])
    elif k == 'mapping':
        K.mapping(s['z'], s['cc'], c['c_scale'], s['m'], c['psi'], c['cutoff'], c['num_ws'], out=s['out'].view)
    else:
        K.interp_rows(s['B'], s['Y'], out=s['out'].view)


# ------------------------------------------------------------------------------------------------ blocks and references
def style_blocks(c, out, N):
    """Every layer's [N, Cin] block of a styles output."""
    bases, _ = style_layout(c, N)
    return [out[b:b + N * L[0]].view(N, L[0]) for L, b in zip(c['layers'], bases)]


def dcoef_blocks(c, out, N):
    _, _, ob, _ = demod_layout(c, N)
    return [out[b:b + N * co].view(N, co) for (ci, co), b in zip(c['layers'], ob)]


def demod_reference(s_block, wsq):
    """(sum_i s_i^2 wsq[o, i] + 1e-8)^-1/2 in fp64: [N, Cin] styles, [Cout, Cin] wsq -> [N, Cout]."""
    return (s_block.double().square() @ wsq.double().t() + 1e-8).rsqrt()


def rel_err(got, ref):
    """max |got - ref| / ref of positive references; a NaN counts as infinite."""
    e = ((got.double() - ref).abs() / ref).max().item()
    return e if e == e else math.inf


def check_case(s):
    """-> {bound kind: error}; asserts the sentinel and written-element checks first."""
    c = s['c']
    k = c['kind']
    out = s['out']
    assert out.untouched_ok(), f'{c["name"]}: an element outside the output was written'
    assert out.written(), f'{c["name"]}: an owned element was not written'
    if k == 'styles':
        e = RangeErr()
        ws, A, b = s['ws'].double(), s['A'].double(), s['b'].double()
        r0 = 0
        for (cin, wi, scale), got in zip(c['layers'], style_blocks(c, out.view, c['N'])):
            e.add(got, (ws[:, wi] @ A[r0:r0 + cin].t() / math.sqrt(c['wdim']) + b[r0:r0 + cin]) * scale)
            r0 += cin
        return {'styles': e.value()}
    if k == 'demod':
        got = dcoef_blocks(c, out.view, c['N'])
        if c['styles'] == 'zero':      # (0 + 1e-8)^-1/2 = 1e4 up to rsqrtf's 2 ulp
            assert (got[0][0].double() - 1e4).abs().max().item() <= 2 * np.spacing(np.float32(1e4)), got[0][0]
        return {'demod': max(rel_err(d, demod_reference(sb, wq)) for d, sb, wq in zip(got, s['s_blocks'], s['wsq_blocks']))}
    if k == 'mapping':
        ref = mapping_reference(s['m'], s['z'], s['cc'], c['c_scale'], c['psi'], c['cutoff'], c['num_ws'])
        return {'mapping': range_rel_err(out.view, ref)}
    if c['basis'] == 'random':
        ref = s['B'].double() @ s['Y'].double()
    else:
        from next3d_b200 import drivers
        ref = drivers.interpolate_ws(s['Y'].double().view(c['K'], 1, c['D']), c['w_frames'], kind=c['basis']).view(c['F'], c['D']).to(DEV)
    return {'interp': range_rel_err(out.view, ref)}


@pytest.mark.gpu
@pytest.mark.parametrize('c', CASES, ids=CASE_IDS)
def test_kernel_matches_fp64_reference(c):
    s = setup_case(c)
    launch_case(s)
    torch.cuda.synchronize()
    errs = check_case(s)
    record_errors('N3D_STYLE_ERRORS', [{'case': c['name'], 'kind': k, 'err': e, 'bound': BOUNDS[k]} for k, e in errs.items()])
    bad = {k: e for k, e in errs.items() if not e < BOUNDS[k]}
    assert not bad, bad
    assert rerun_identical([s['out']], lambda: launch_case(s)), f'{c["name"]}: a rerun is not bit-identical'


# ------------------------------------------------------------------------------------------------ batch independence
def single_image(s, n):
    """The state of a case that launches image n of s alone (N = 1)."""
    c = s['c']
    k, one = c['kind'], dict(s, c=dict(s['c'], N=1))
    if k == 'styles':
        one['ws'] = s['ws'][n:n + 1].contiguous()
        one['ooff'], one['out'] = styles_tables(c, 1)
    elif k == 'demod':
        one['s_blocks'] = [t[n:n + 1] for t in s['s_blocks']]
        one.update(demod_inputs(c, 1, one['s_blocks'], s['wsq_blocks']))
    else:
        one['z'], one['cc'] = s['z'][n:n + 1].contiguous(), s['cc'][n:n + 1].contiguous()
        one['out'] = Guarded((1, c['num_ws'], 512))
    return one


def _image_rows(s, n):
    """Image n's part of every output block of a case, as one flat tensor."""
    c, v = s['c'], s['out'].view
    if c['kind'] == 'styles':
        return torch.cat([t[n] for t in style_blocks(c, v, c['N'])])
    if c['kind'] == 'demod':
        return torch.cat([t[n] for t in dcoef_blocks(c, v, c['N'])])
    return v[n].reshape(-1)


BATCHED = [c for c in CASES if c['kind'] in ('styles', 'demod', 'mapping') and c['N'] > 1]


@pytest.mark.gpu
@pytest.mark.parametrize('c', BATCHED, ids=[c['name'] for c in BATCHED])
def test_image_does_not_depend_on_batch(c):
    """Image n of a batch of N holds the same bits as a launch of image n alone, for the first, a middle and the last image."""
    s = setup_case(c)
    launch_case(s)
    for n in sorted({0, c['N'] // 2, c['N'] - 1}):
        one = single_image(s, n)
        launch_case(one)
        torch.cuda.synchronize()
        assert one['out'].untouched_ok() and one['out'].written(), (c['name'], n)
        assert torch.equal(_image_rows(s, n).view(torch.int32), _image_rows(one, 0).view(torch.int32)), (c['name'], n)


# ------------------------------------------------------------------------------------------------ launches
@pytest.mark.gpu
def test_launched_kernel_matches_plan(tmp_path):
    """Every case under torch.profiler: the kernel it launched and its grid are the ones `plan` predicts at the device's SM count."""
    pattern = re.compile(r'styles_kernel|demod_kernel|mapping_kernel|interp_rows_kernel')

    def run():
        for c in CASES:
            s = setup_case(c)
            launch_case(s)
            torch.cuda.synchronize()
            del s
        return CASES                        # one launch per case

    _, events = launched_kernels(run, pattern, tmp_path)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for c, e in zip(CASES, events):
        p = plan(c, sms)
        assert pattern.search(e['name']).group(0) == p['kernel'], (c['name'], e['name'], p)
        grid = e.get('args', {}).get('grid')
        if grid is not None:
            assert list(grid) == [p['grid'], 1, 1], (c['name'], grid, p)


# ------------------------------------------------------------------------------------------------ the engine's tables
@pytest.mark.gpu
@pytest.mark.parametrize('factory', [config.tiny_config, config.full_config], ids=['tiny', 'full'])
def test_engine_style_tables_match_fp64(factory):
    """Engine._set_styles at N = 3, 1, 3 (the per-N table cache): every modulated layer's style block against fp64
    fully_connected of the ws the oracle feeds it (times the ToRGB gain), and its dcoef block against fp64 demodulation of those
    styles by the layer's weight."""
    from next3d_b200.engine import Engine
    from oracle import ops as oo
    cfg = factory(512)
    sd = weights.make_state_dict(cfg, seed=41)
    E = Engine(cfg, sd)
    widx = oracle_widx(cfg)
    assert set(widx) == set(E.mod)
    g = torch.Generator(device=DEV).manual_seed(43)
    errs = []
    for call, N in enumerate((3, 1, 3)):
        ws = torch.randn(N, 28, 512, device=DEV, generator=g)
        E._set_styles(ws)
        torch.cuda.synchronize()
        e_s, e_d = RangeErr(), 0.0
        for name, L in E.mod.items():
            got = E._styles[L.sbase * N:(L.sbase + L.cin) * N].view(N, L.cin)
            w = sd[f'{name}.weight'].to(DEV, torch.float64)
            ref = oo.fully_connected(ws[:, widx[name]].double(), sd[f'{name}.affine.weight'].to(DEV, torch.float64),
                                     sd[f'{name}.affine.bias'].to(DEV, torch.float64))
            if L.is_rgb:
                ref = ref / math.sqrt(w.shape[1] * w.shape[2] ** 2)
            e_s.add(got, ref)
            if not L.is_rgb:
                d = E._dcoefs[L.dbase * N:(L.dbase + L.cout) * N].view(N, L.cout)
                e_d = max(e_d, rel_err(d, demod_reference(got, w.square().sum(dim=[2, 3]))))
        case = f'engine_{factory.__name__}_call{call}_n{N}'
        errs += [{'case': case, 'kind': 'styles', 'err': e_s.value(), 'bound': BOUNDS['styles']},
                 {'case': case, 'kind': 'demod', 'err': e_d, 'bound': BOUNDS['demod']}]
    record_errors('N3D_STYLE_ERRORS', errs)
    bad = [e for e in errs if not e['err'] < e['bound']]
    assert not bad, bad


# ------------------------------------------------------------------------------------------------ truncation cutoff
def test_mapping_cutoff_follows_slice_semantics():
    """CPU: kernels.mapping hands n3d_mapping (which truncates layers l < cutoff, or all for cutoff < 0) exactly the layers
    ws[:, :truncation_cutoff] selects, as the reference and the CPU path truncate them."""
    from next3d_b200 import kernels as K
    for num_ws in (1, 14, 28):
        for cutoff in [None, *range(-2 * num_ws - 2, 2 * num_ws + 3)]:
            abi = K.mapping_cutoff(cutoff, num_ws)
            truncated = [l for l in range(num_ws) if abi < 0 or l < abi]
            assert truncated == list(range(num_ws))[:cutoff], (num_ws, cutoff, abi)


@pytest.mark.gpu
@pytest.mark.parametrize('cutoff', [-1, -14])
def test_generator_mapping_negative_cutoff_matches_oracle(cutoff):
    """G.mapping on CUDA truncates the layers ws[:, :cutoff] selects, as oracle.generator.mapping does."""
    from next3d_b200.triplane_next3d import TriPlaneGenerator
    from oracle import generator as og
    cfg, sd = _mapping_state()
    G = TriPlaneGenerator.from_config(cfg, sd, device=DEV)
    z, c, _, _ = weights.demo_inputs(cfg, 3, seed=7)
    got = G.mapping(z.to(DEV), c.to(DEV), truncation_psi=0.7, truncation_cutoff=cutoff)
    ref = og.mapping(sd, cfg, z, c, 0.7, cutoff)
    assert range_rel_err(got.cpu(), ref) < 2e-6


# ------------------------------------------------------------------------------------------------ alignment (CPU, nothing launched)
@pytest.mark.parametrize('field', ['ws', 'affine_w'])
def test_styles_refuses_misaligned_pointers(field):
    L = lib()
    N, num_ws, wdim, r = 1, 2, 8, 4
    t = dict(ws=torch.zeros(N * num_ws * wdim + 64), affine_w=torch.zeros(r * wdim + 64))
    p = {k: v.data_ptr() for k, v in t.items()}
    p[field] = offset_view(t[field], 4).data_ptr()
    b, scale, out = torch.zeros(r), torch.ones(r), torch.zeros(N * r)
    widx, cin, ooff = torch.zeros(r, dtype=torch.int32), torch.full((r,), r, dtype=torch.int32), torch.arange(r)
    refused(L.lib.n3d_styles(p['ws'], N, num_ws, wdim, p['affine_w'], b.data_ptr(), widx.data_ptr(), scale.data_ptr(), ooff.data_ptr(),
                             cin.data_ptr(), out.data_ptr(), r, None), 'n3d_styles: ws and affine_w must be 16-byte aligned')


@pytest.mark.parametrize('field', ['fc0_w', 'fc1_w'])
def test_mapping_refuses_misaligned_pointers(field):
    L = lib()
    N = 1
    m = {k: torch.zeros(v.numel() + 64) for k, v in mapping_params(_mapping_state()[1], 'cpu').items()}
    p = {k: v.data_ptr() for k, v in m.items()}
    p[field] = offset_view(m[field], 4).data_ptr()
    z, c, ws = torch.zeros(N, 512), torch.zeros(N, 25), torch.zeros(N, 28, 512)
    refused(L.lib.n3d_mapping(z.data_ptr(), c.data_ptr(), N, 1.0, p['embed_w'], p['embed_b'], p['fc0_w'], p['fc0_b'], p['fc1_w'], p['fc1_b'],
                              p['w_avg'], 0.7, 14, 28, ws.data_ptr(), None), 'n3d_mapping: fc0_w and fc1_w must be 16-byte aligned')
